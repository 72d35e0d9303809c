#!/usr/bin/env python
"""Device time per training step of every kernel and copy a ``Trainer`` step launches, from ``torch.profiler``.

    python scripts/step_kernels.py [--sizes 784 128 127 126 125 124 123 10] [--global-batch 128] [--n-mubatches 4]
                                   [--precision fp32] [--momentum 0] [--weight-decay 0] [--steps 300] [--warmup 100]

The engine launches its kernels eagerly here (``use_graph=False``) so that the profiler sees each launch; the steps run
back to back as in ``bench.py`` (inputs already on the device, copied into the engine's staging buffers each step).
After ``--warmup`` untimed steps the profiler records ``--steps`` steps.  One JSON line per kernel or copy: its calls
per step and its device time per step in microseconds, largest first.  The first line names the card and its power
limit.  Tracing slows the host, so take step times from ``bench.py``, not from this script.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REFERENCE = [784, 128, 127, 126, 125, 124, 123, 10]


def card():
    import torch

    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--sizes", type=int, nargs="+", default=REFERENCE)
    p.add_argument("--global-batch", type=int, default=128)
    p.add_argument("--n-mubatches", type=int, default=4)
    p.add_argument("--precision", choices=["fp32", "tf32"], default="fp32")
    p.add_argument("--momentum", type=float, default=0.0)
    p.add_argument("--weight-decay", type=float, default=0.0)
    p.add_argument("--steps", type=int, default=300, help="profiled steps")
    p.add_argument("--warmup", type=int, default=100, help="untimed steps before the profiled ones")
    args = p.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("step_kernels: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock,sm_clock": limits}), flush=True)

    sizes, gbs = args.sizes, args.global_batch
    tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=args.n_mubatches, lr=0.006, precision=args.precision,
                 momentum=args.momentum, weight_decay=args.weight_decay, use_graph=False, device=dev)
    pool = 16
    x, y = synthetic_mnist(n=pool * gbs, n_features=sizes[0], n_classes=sizes[-1])
    xs = torch.from_numpy(x).reshape(pool, gbs, sizes[0]).to(dev)
    ys = torch.from_numpy(y).reshape(pool, gbs, sizes[-1]).to(dev)

    for i in range(args.warmup):
        tr.step_async(xs[i % pool], ys[i % pool])
    torch.cuda.synchronize(dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            tr.step_async(xs[i % pool], ys[i % pool])
        torch.cuda.synchronize(dev)

    rows = [(e.key, e.count, e.self_device_time_total) for e in prof.key_averages() if e.self_device_time_total > 0]
    for key, count, us in sorted(rows, key=lambda r: -r[2]):
        print(json.dumps({"kernel": key, "calls_per_step": round(count / args.steps, 3),
                          "us_per_step": round(us / args.steps, 2)}), flush=True)
    print(json.dumps({"sizes": "-".join(map(str, sizes)), "global_batch": gbs, "n_mubatches": args.n_mubatches,
                      "precision": args.precision, "momentum": args.momentum, "weight_decay": args.weight_decay,
                      "steps": args.steps, "kernels_per_step": int(tr.engine.kernels_per_step()),
                      "total_us_per_step": round(sum(r[2] for r in rows) / args.steps, 2)}), flush=True)


if __name__ == "__main__":
    main()
