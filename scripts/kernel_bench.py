#!/usr/bin/env python
"""Per-kernel device timing (CUDA events, warm-up, L2 flush between timed launches or
back-to-back) of the sm_90a GEMM family on the shapes of the default MLP and of the
hidden=8192 stress config.  Prints one JSON line per case with achieved bytes/s and the
fraction of the HBM bandwidth (measured, from MEASURED_PEAKS.json, else the H100 SXM data sheet)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from shallowspeed_b200.ops import cuda as K  # noqa: E402


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "_fallback": True}   # H100 SXM data sheet


def time_fn(fn, iters, flush=None):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    if flush is None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters
    ts = []
    for _ in range(iters):
        flush.add_(1.0)                      # > L2 sized write
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def time_rotating(fns, iters):
    """Back-to-back launches cycling through `len(fns)` instances of the same op on DISTINCT operand buffers whose total
    size is several times L2: every launch streams its weights from HBM (the previous launches evicted them) and the lines
    it evicts are CLEAN.  The per-iteration "cold" mode above flushes L2 with a read-modify-write pass, i.e. it leaves up to
    50 MB (the H100's L2) of dirty lines whose write-back competes with the timed kernel's reads; this mode is what a real step of a model larger than L2 looks like."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fns[i % len(fns)]()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="default", choices=["default", "stress", "all"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--precision", default="tf32", choices=["tf32", "fp32"])
    ap.add_argument("--k-splits", type=int, default=0,
                    help="also time the experimental split-K variant of fwd / dgrad (-1 = planner's choice, k >= 2 = force)")
    args = ap.parse_args()
    pk = peaks()
    dev = "cuda"
    flush = torch.zeros(128 * 1024 * 1024 // 4, device=dev)   # 128 MB > 50 MB L2
    shapes = []
    if args.shapes in ("default", "all"):
        shapes += [(32, 784, 128), (32, 128, 127), (32, 123, 10), (4, 784, 128), (128, 784, 128)]
    if args.shapes in ("stress", "all"):
        shapes += [(8, 8192, 8192), (32, 8192, 8192), (128, 8192, 8192)]
    for rows, k, n in shapes:
        x = torch.randn(rows, k, device=dev)
        ld = (k + 1 + 7) // 8 * 8
        n_rot = max(1, min(4, int(3 * 50e6 // (n * ld * 4)) + 1)) if n * ld * 4 > 16e6 else 1   # >= 3 x L2 of distinct weights
        Wbs = [torch.randn(n, ld, device=dev) for _ in range(n_rot)]
        Gbs = [torch.zeros(n, ld, device=dev) for _ in range(n_rot)]
        Wb, Gb = Wbs[0], Gbs[0]
        W, b = Wb[:, :k], Wb[:, k]
        y = K.empty_padded(rows, n, dev)
        dz = K.empty_padded(rows, n, dev)
        dz.normal_()
        dx = K.empty_padded(rows, k, dev)
        wbytes = n * k * 4
        pr = args.precision
        cases = {
            "fwd": (lambda: K.linear_fwd(x, W, b, relu=True, out=y, precision=pr), wbytes + rows * (k + n) * 4),
            "dgrad": (lambda: K.linear_dgrad(dz, W, mask=x, out=dx, precision=pr), wbytes + rows * (2 * k + n) * 4),
            "wgrad_write": (lambda: K.linear_wgrad(dz, x, Gb[:, :k], accumulate=False, grad_b=Gb[:, k], precision=pr), wbytes + rows * (k + n) * 4),
            "wgrad_acc": (lambda: K.linear_wgrad(dz, x, Gb[:, :k], accumulate=True, grad_b=Gb[:, k], precision=pr), 2 * wbytes + rows * (k + n) * 4),
        }
        if args.k_splits:
            ks = args.k_splits
            cases["fwd_splitk"] = (lambda: K.linear_fwd(x, W, b, relu=True, out=y, precision=pr, k_splits=ks), cases["fwd"][1])
            cases["dgrad_splitk"] = (lambda: K.linear_dgrad(dz, W, mask=x, out=dx, precision=pr, k_splits=ks), cases["dgrad"][1])
        def rot(name):
            """the same op on each of the rotating weight / gradient buffers"""
            out = []
            for Wr, Gr in zip(Wbs, Gbs):
                Wv, bv = Wr[:, :k], Wr[:, k]
                ks = args.k_splits
                out.append({
                    "fwd": lambda Wv=Wv, bv=bv: K.linear_fwd(x, Wv, bv, relu=True, out=y, precision=pr),
                    "dgrad": lambda Wv=Wv: K.linear_dgrad(dz, Wv, mask=x, out=dx, precision=pr),
                    "wgrad_write": lambda Gr=Gr: K.linear_wgrad(dz, x, Gr[:, :k], accumulate=False, grad_b=Gr[:, k], precision=pr),
                    "wgrad_acc": lambda Gr=Gr: K.linear_wgrad(dz, x, Gr[:, :k], accumulate=True, grad_b=Gr[:, k], precision=pr),
                    "fwd_splitk": lambda Wv=Wv, bv=bv: K.linear_fwd(x, Wv, bv, relu=True, out=y, precision=pr, k_splits=ks),
                    "dgrad_splitk": lambda Wv=Wv: K.linear_dgrad(dz, Wv, mask=x, out=dx, precision=pr, k_splits=ks),
                }[name])
            return out

        for name, (fn, nbytes) in cases.items():
            warm = time_fn(fn, args.iters)
            cold = time_fn(fn, max(10, args.iters // 3), flush=flush)
            flops = 2.0 * rows * k * n
            rec = {"kernel": name, "rows": rows, "in": k, "out": n, "us_back_to_back": round(warm, 2),
                   "us_cold_l2": round(cold, 2), "GBps_cold": round(nbytes / cold / 1e3, 1),
                   "frac_hbm_measured": round(nbytes / cold / 1e3 / pk["hbm_gbs"], 3),
                   "tflops_cold": round(flops / cold / 1e6, 2)}
            if n_rot > 1:
                stream = time_rotating(rot(name), max(12, args.iters))
                rec.update({"us_stream": round(stream, 2), "GBps_stream": round(nbytes / stream / 1e3, 1),
                            "frac_hbm_stream": round(nbytes / stream / 1e3 / pk["hbm_gbs"], 3), "rotating_buffers": n_rot})
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
