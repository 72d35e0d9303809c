#!/usr/bin/env python
"""Cost of residual connections: step time of a Trainer without skips against the same model with ``residual=True``,
alternated block by block in one process so that both arms see the same card, clocks and neighbours.

    python scripts/residual_bench.py [--steps 100] [--repeats 5] [--warmup 20]

Models (one GPU, global batch 128, 4 micro-batches unless noted), each with relu and gelu, in fp32 and bf16:
  (a) 784-128x6-10: the cluster chain kernel;
  (b) 784-32x6-10:  the one-CTA chain kernel;
  (c) 784-2048x6-10, global batch 512: the layer-wise GEMMs with split-K.
Both arms of a model run the same path; a residual ReLU model is gated (its forward stores a gate per hidden element).
Every block of ``--steps`` steps is timed with CUDA events on the engine's stream between two device
synchronisations; each line reports the median block and the spread (min..max) over ``--repeats`` blocks.  The first line
names the card and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.optimizer_bench import card  # noqa: E402

MODELS = {
    "a": ([784] + [128] * 6 + [10], 128),
    "b": ([784] + [32] * 6 + [10], 128),
    "c": ([784] + [2048] * 6 + [10], 512),
}


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=100, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=5, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=20, help="untimed steps per arm before the first block")
    p.add_argument("--models", nargs="+", default=sorted(MODELS), choices=sorted(MODELS))
    p.add_argument("--activations", nargs="+", default=["relu", "gelu"])
    p.add_argument("--precisions", nargs="+", default=["fp32", "bf16"])
    args = p.parse_args()

    import torch

    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("residual_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": limits}), flush=True)
    pool = 8

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

    for key in args.models:
        sizes, gbs = MODELS[key]
        gen = torch.Generator().manual_seed(0)
        xs = torch.rand(pool, gbs, sizes[0], generator=gen).to(dev)
        ys = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (pool, gbs), generator=gen), sizes[-1]).float().to(dev)
        for precision in args.precisions:
            for kind in args.activations:
                trainers = {res: Trainer(sizes, global_batch_size=gbs, n_mubatches=4, lr=0.001, device=dev, activation=kind,
                                         precision=precision, residual=res) for res in (False, True)}
                for tr in trainers.values():
                    block(tr, xs, ys, args.warmup)
                times = {res: [] for res in trainers}
                for _ in range(args.repeats):
                    for res, tr in trainers.items():
                        times[res].append(block(tr, xs, ys, args.steps))
                for res, ts in times.items():
                    s = sorted(ts)
                    eng = trainers[res].engine
                    print(json.dumps({"model": key, "sizes": f"{sizes[0]}-{sizes[1]}x{len(sizes) - 2}-{sizes[-1]}",
                                      "gbs": gbs, "precision": precision, "activation": kind, "residual": res,
                                      "ms_per_step": round(s[len(s) // 2], 5), "min": round(s[0], 5),
                                      "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                                      "chain": bool(eng.uses_chain()), "kernels_per_step": int(eng.kernels_per_step()),
                                      "final_loss": round(float(trainers[res].loss()), 6)}), flush=True)
                del trainers
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
