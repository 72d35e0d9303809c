#!/usr/bin/env python
"""Cost of the smooth hidden activations: step time of a Trainer with ReLU against one with GELU, SiLU or tanh, alternated
block by block in one process so that both see the same card, clocks and neighbours.

    python scripts/activation_bench.py [--steps 200] [--repeats 7] [--warmup 50] [--dropout 0 0.2]

Reference model (784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches) on one GPU; the chain kernel's
forward epilogues apply f and store its gate, the backward multiplies by the gate.  For each dropout rate, ReLU and every
smooth activation run as alternated arms; every block of ``--steps`` steps is timed with CUDA events on the engine's
stream between two device synchronisations, and each line reports the median block and the spread (min..max) over
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

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
KINDS = ("relu", "gelu", "silu", "tanh")


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--dropout", type=float, nargs="+", default=[0.0, 0.2], help="drop rates to measure")
    p.add_argument("--activations", nargs="+", default=list(KINDS), choices=list(KINDS))
    args = p.parse_args()

    import torch

    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("activation_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": limits}), flush=True)
    pool = 16
    gen = torch.Generator().manual_seed(0)
    xs = torch.rand(pool, 128, SIZES[0], generator=gen).to(dev)
    ys = torch.nn.functional.one_hot(torch.randint(0, SIZES[-1], (pool, 128), generator=gen), SIZES[-1]).float().to(dev)

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

    for drop in args.dropout:
        trainers = {kind: Trainer(SIZES, global_batch_size=128, n_mubatches=4, lr=0.006, device=dev, dropout=drop,
                                  activation=kind) for kind in args.activations}
        for tr in trainers.values():
            block(tr, args.warmup)
        times = {kind: [] for kind in trainers}
        for _ in range(args.repeats):
            for kind, tr in trainers.items():
                times[kind].append(block(tr, args.steps))
        for kind, ts in times.items():
            s = sorted(ts)
            eng = trainers[kind].engine
            print(json.dumps({"activation": kind, "dropout": drop, "ms_per_step": round(s[len(s) // 2], 5),
                              "min": round(s[0], 5), "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                              "chain": bool(eng.uses_chain()), "kernels_per_step": int(eng.kernels_per_step()),
                              "final_loss": round(float(trainers[kind].loss()), 6)}), flush=True)
        del trainers
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
