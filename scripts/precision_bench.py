#!/usr/bin/env python
"""What bf16 tensor-core products buy: step time of a Trainer in fp32 (3xTF32), tf32 and bf16, alternated block by block
in one process so that all arms see the same card, clocks and neighbours; the loss curves from the same initial weights;
and the chain and grouped-wgrad kernel times from one ``torch.profiler`` run per arm.

    python scripts/precision_bench.py [--steps 200] [--repeats 7] [--warmup 50] [--wide-steps 20] [--train-steps 300]

Workloads (one GPU):
  * reference: 784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches (the chain kernel; the GEMMs are
    narrow and latency-bound);
  * wide: ``bench.py --hidden 4096 --n-layers 8`` (784-4096x7-10), global batch 2048, 4 micro-batches (layer-wise
    tensor-core GEMMs, which dominate the step).
Every block of steps is timed with CUDA events on the engine's stream between two device synchronisations; each line
reports the median block and the spread (min..max) over ``--repeats`` blocks.  The loss curves train the reference model
for ``--train-steps`` steps on the same synthetic data in each arm (``seed_mode="shape"``: the same initial weights) and
report the final loss and the gap to fp32.  The profiler run launches eagerly (``use_graph=False``) and reports the
device time per call of the chain kernel and the grouped weight-gradient kernel.  The first line names the card and its
power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.optimizer_bench import card  # noqa: E402

PRECISIONS = ("fp32", "tf32", "bf16")
WORKLOADS = {"reference": ([784, 128, 127, 126, 125, 124, 123, 10], 128, 4),
             "wide": ([784] + [4096] * 7 + [10], 2048, 4)}
PROFILED = ("mlp_chain_kernel", "tc_wgrad_group_kernel")


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block (reference)")
    p.add_argument("--wide-steps", type=int, default=20, help="steps per timed block (wide)")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--train-steps", type=int, default=300, help="steps of each loss curve (0: none)")
    p.add_argument("--profile-steps", type=int, default=50, help="steps of each profiler run (0: none)")
    p.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    args = p.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("precision_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": limits}), flush=True)
    pool = 8

    def data(sizes, gbs, n):
        x, y = synthetic_mnist(n=n * gbs, n_features=sizes[0], n_classes=sizes[-1])
        return (torch.from_numpy(x).reshape(n, gbs, sizes[0]).to(dev),
                torch.from_numpy(y).reshape(n, gbs, sizes[-1]).to(dev))

    def block(tr, xs, ys, n):
        torch.cuda.synchronize(dev)
        st = torch.cuda.ExternalStream(tr.engine.main_stream(), device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(n):
            tr.step_async(xs[i % pool], ys[i % pool])
        e1.record(st)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    # ---- step time, alternated arms
    for wl in args.workloads:
        sizes, gbs, n_mu = WORKLOADS[wl]
        xs, ys = data(sizes, gbs, pool)
        steps = args.steps if wl == "reference" else args.wide_steps
        trainers = {pr: Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=0.006, device=dev, precision=pr)
                    for pr in PRECISIONS}
        for tr in trainers.values():
            block(tr, xs, ys, args.warmup if wl == "reference" else max(2, args.warmup // 10))
        times = {pr: [] for pr in trainers}
        for _ in range(args.repeats):
            for pr, tr in trainers.items():
                times[pr].append(block(tr, xs, ys, steps))
        base = sorted(times["fp32"])[len(times["fp32"]) // 2]
        for pr, ts in times.items():
            s = sorted(ts)
            eng = trainers[pr].engine
            print(json.dumps({"workload": wl, "sizes": "-".join(map(str, sizes)), "global_batch": gbs,
                              "precision": pr, "ms_per_step": round(s[len(s) // 2], 5), "min": round(s[0], 5),
                              "max": round(s[-1], 5), "vs_fp32": round(s[len(s) // 2] / base, 4), "blocks": len(s),
                              "steps": steps, "chain": bool(eng.uses_chain()),
                              "kernels_per_step": int(eng.kernels_per_step())}), flush=True)
        del trainers, xs, ys
        torch.cuda.empty_cache()

    # ---- loss curves of the reference model from the same initial weights and data
    if args.train_steps > 0:
        sizes, gbs, n_mu = WORKLOADS["reference"]
        x, y = synthetic_mnist(n=args.train_steps * gbs)
        xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
        curves = {}
        for pr in PRECISIONS:
            tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=0.006, device=dev, precision=pr)
            curves[pr] = [float(tr.step(xh[i * gbs:(i + 1) * gbs], yh[i * gbs:(i + 1) * gbs]))
                          for i in range(args.train_steps)]
            del tr
        for pr, c in curves.items():
            gaps = [abs(a - b) for a, b in zip(c, curves["fp32"])]
            print(json.dumps({"curve": pr, "steps": len(c), "first_loss": round(c[0], 6), "final_loss": round(c[-1], 6),
                              "final_gap_to_fp32": round(abs(c[-1] - curves["fp32"][-1]), 7),
                              "max_gap_to_fp32": round(max(gaps), 7),
                              "max_rel_gap_to_fp32": round(max(g / f for g, f in zip(gaps, curves["fp32"])), 6)}),
                  flush=True)

    # ---- kernel times, one profiler run per arm (eager launches)
    if args.profile_steps > 0:
        sizes, gbs, n_mu = WORKLOADS["reference"]
        xs, ys = data(sizes, gbs, pool)
        for pr in PRECISIONS:
            tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=0.006, device=dev, precision=pr,
                         use_graph=False)
            for i in range(20):
                tr.step_async(xs[i % pool], ys[i % pool])
            torch.cuda.synchronize(dev)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(args.profile_steps):
                    tr.step_async(xs[i % pool], ys[i % pool])
                torch.cuda.synchronize(dev)
            for e in prof.key_averages():
                hit = next((k for k in PROFILED if k in e.key), None)
                if hit and e.count:
                    print(json.dumps({"profile": pr, "kernel": hit, "calls_per_step": round(e.count / args.profile_steps, 3),
                                      "us_per_call": round(e.self_device_time_total / e.count, 3)}), flush=True)
            del tr


if __name__ == "__main__":
    main()
