#!/usr/bin/env python
"""Cost of dropout: step time of a Trainer with p = 0 vs one with p = 0.2, alternated block by block in one process so
that both see the same card, clocks and neighbours.

    python scripts/dropout_bench.py [--steps 200] [--repeats 7] [--warmup 50]

Two workloads on one GPU: the reference model (784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches), whose
masks are drawn in the layer-chain kernel's epilogues, and a wide model (--hidden 4096 --n-layers 8), whose masks are
drawn in the layer-wise forward GEMMs' epilogues.  Every block of ``--steps`` steps is timed with CUDA events on the
engine's stream between two device synchronisations; each line reports the median block and the spread (min..max) over
``--repeats`` blocks.  The first line names the card and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.optimizer_bench import card  # noqa: E402

WORKLOADS = {"reference": [784, 128, 127, 126, 125, 124, 123, 10], "wide": [784] + [4096] * 7 + [10]}
ARMS = (0.0, 0.2)

def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    args = p.parse_args()

    import torch

    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("dropout_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": limits}), flush=True)

    for wl in args.workloads:
        sizes = WORKLOADS[wl]
        trainers = {arm: Trainer(sizes, global_batch_size=128, n_mubatches=4, lr=0.006, device=dev, dropout=arm)
                    for arm in ARMS}
        pool = 16
        gen = torch.Generator().manual_seed(0)
        xs = torch.rand(pool, 128, sizes[0], generator=gen).to(dev)
        ys = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (pool, 128), generator=gen), sizes[-1]).float().to(dev)

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
        for arm, ts in times.items():
            s = sorted(ts)
            eng = trainers[arm].engine
            print(json.dumps({"workload": wl, "sizes": "-".join(map(str, sizes)), "dropout": arm,
                              "ms_per_step": round(s[len(s) // 2], 5), "min": round(s[0], 5), "max": round(s[-1], 5),
                              "blocks": len(s), "steps": args.steps, "chain": bool(eng.uses_chain()),
                              "kernels_per_step": int(eng.kernels_per_step()),
                              "final_loss": round(float(trainers[arm].loss()), 6)}), flush=True)
        del trainers
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
