#!/usr/bin/env python
"""Cost of the EMA of the weights: step time of plain SGD against plain SGD + EMA, and of momentum 0.9 with weight
decay 5e-4 against the same + EMA, through ``Trainer`` on one GPU, alternated block by block in one process so that
every arm sees the same card, clocks and neighbours.

    python scripts/ema_bench.py [--steps 200] [--repeats 7] [--warmup 50]

Two workloads: the reference model (784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches; latency bound)
and a bandwidth-bound one (--hidden 4096 --n-layers 8, ~104M parameters), where the EMA adds one read and one write of
the EMA buffer per parameter per step, plus a read of the weights on the plain path.  Every block of ``--steps`` steps
is timed with CUDA events on the engine's stream between two device synchronisations; each line reports the median
block and the spread (min..max) over ``--repeats`` blocks.  The first line names the card and its power limit, the
last one the SM clock read right after the timed blocks.
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
MOM = {"momentum": 0.9, "weight_decay": 5e-4}
ARMS = {"plain": {}, "plain+ema": {"ema_decay": 0.999}, "momentum": MOM, "momentum+ema": {**MOM, "ema_decay": 0.999}}


def query(fields):
    import torch

    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader",
                               f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--workloads", nargs="+", default=["reference", "wide"], choices=["reference", "wide"])
    args = p.parse_args()

    import torch

    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.layers import mlp_sizes
    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("ema_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    print(json.dumps({"card": torch.cuda.get_device_name(), "power_limit,max_sm_clock": query("power.limit,clocks.max.sm")}),
          flush=True)

    for wl in args.workloads:
        sizes = REFERENCE if wl == "reference" else mlp_sizes(4096, 8)
        trainers = {arm: Trainer(sizes, global_batch_size=128, n_mubatches=4, lr=0.006, device=dev, **kw)
                    for arm, kw in ARMS.items()}
        pool = 16
        x, y = synthetic_mnist(n=pool * 128)
        xs = torch.from_numpy(x).reshape(pool, 128, 784).to(dev)
        ys = torch.from_numpy(y).reshape(pool, 128, 10).to(dev)

        def block(tr, n):
            torch.cuda.synchronize(dev)
            st = torch.cuda.ExternalStream(tr.engine.main_stream(), device=dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for i in range(n):
                tr.step_async(xs[i % pool], ys[i % pool])
            e1.record(st)
            torch.cuda.synchronize(dev)
            return e0.elapsed_time(e1) / n

        for tr in trainers.values():
            block(tr, args.warmup)
        times = {arm: [] for arm in trainers}
        for _ in range(args.repeats):
            for arm, tr in trainers.items():
                times[arm].append(block(tr, args.steps))
        sm_clock = query("clocks.sm")
        n_params = sum(o * (i + 1) for i, o in zip(sizes[:-1], sizes[1:]))
        for arm, ts in times.items():
            s = sorted(ts)
            print(json.dumps({"workload": wl, "sizes": f"{sizes[0]}-{sizes[1]}x{len(sizes) - 2}-{sizes[-1]}",
                              "params": n_params, "arm": arm, **ARMS[arm], "ms_per_step": round(s[len(s) // 2], 5),
                              "min": round(s[0], 5), "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                              "kernels_per_step": int(trainers[arm].engine.kernels_per_step())}), flush=True)
        print(json.dumps({"workload": wl, "sm_clock_after": sm_clock}), flush=True)
        del trainers
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
