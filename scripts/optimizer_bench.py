#!/usr/bin/env python
"""Cost of the stateful SGD rule: step time of plain SGD vs ``momentum=0.9, weight_decay=5e-4`` through ``Trainer``,
alternated block by block in one process so that both see the same card, clocks and neighbours.

    python scripts/optimizer_bench.py [--steps 200] [--repeats 7] [--warmup 50]
    torchrun --nproc-per-node N scripts/optimizer_bench.py --gpus N       # data parallel (NCCL all-reduce)

Two workloads: the reference model (784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches; latency bound)
and a bandwidth-bound one (--hidden 4096 --n-layers 8, ~104M parameters), where momentum adds one read and one write of
the momentum buffer and weight decay one read of the weights per parameter per step.  Every block of ``--steps`` steps
is timed with CUDA events on the engine's stream between two device synchronisations; each line reports the median
block and the spread (min..max) over ``--repeats`` blocks.  The first line names the card and its power limit.
With more than one GPU both arms use ``--comm nccl`` (the in-kernel DP reductions keep no optimizer state).
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
ARMS = {"plain": {}, "momentum": {"momentum": 0.9, "weight_decay": 5e-4}}


def card():
    import torch

    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--workloads", nargs="+", default=["reference", "wide"], choices=["reference", "wide"])
    args = p.parse_args()

    import torch
    import torch.distributed as dist

    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.layers import mlp_sizes
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("optimizer_bench: no CUDA device")
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dev = torch.device("cuda", torch.cuda.current_device())
    dp_comm = None
    if args.gpus > 1:
        dist.init_process_group("nccl", rank=rank, world_size=args.gpus, device_id=dev)
        dp_comm, _ = make_torch_comms(ProcessGrid(args.gpus, 1, rank))
    name, limits = card()
    if rank == 0:
        print(json.dumps({"card": name, "power_limit,max_sm_clock": limits, "gpus": args.gpus}), flush=True)

    for wl in args.workloads:
        sizes = REFERENCE if wl == "reference" else mlp_sizes(4096, 8)
        gbs = 128 * args.gpus
        trainers = {arm: Trainer(sizes, global_batch_size=gbs, n_mubatches=4, lr=0.006, dp_comm=dp_comm,
                                 comm_mode="nccl" if args.gpus > 1 else "fused", device=dev, **kw)
                    for arm, kw in ARMS.items()}
        pool = 16
        x, y = synthetic_mnist(n=pool * gbs)
        r = dp_comm.Get_rank() if dp_comm is not None else 0
        xs = torch.from_numpy(x[r::args.gpus].copy()).reshape(pool, 128, 784).to(dev)
        ys = torch.from_numpy(y[r::args.gpus].copy()).reshape(pool, 128, 10).to(dev)

        def block(tr, n):
            torch.cuda.synchronize(dev)
            if dp_comm is not None:
                dist.barrier()
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
        if rank == 0:
            n_params = sum(o * (i + 1) for i, o in zip(sizes[:-1], sizes[1:]))
            for arm, ts in times.items():
                s = sorted(ts)
                print(json.dumps({"workload": wl, "sizes": f"{sizes[0]}-{sizes[1]}x{len(sizes) - 2}-{sizes[-1]}",
                                  "params": n_params, "arm": arm, **ARMS[arm], "ms_per_step": round(s[len(s) // 2], 5),
                                  "min": round(s[0], 5), "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                                  "kernels_per_step": int(trainers[arm].engine.kernels_per_step())}), flush=True)
        del trainers
        torch.cuda.empty_cache()
    if dp_comm is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
