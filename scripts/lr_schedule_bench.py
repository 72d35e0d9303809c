#!/usr/bin/env python
"""Cost of a learning rate that changes every step: step time with a constant rate against a rate that differs from
the previous step's on every step (so the engine rewrites its device ``lr`` slot before every step), through
``Trainer``, alternated block by block in one process so that both arms see the same card, clocks and neighbours.

    python scripts/lr_schedule_bench.py [--steps 200] [--repeats 7] [--warmup 50]
    torchrun --nproc-per-node 8 scripts/lr_schedule_bench.py --gpus 8          # data parallel, --comm fused

Two timings per arm, on the reference model (784-128-127-126-125-124-123-10, 128 rows per replica, 4 micro-batches):
* device: CUDA events on the engine's stream around a block of ``step_async`` calls with device-resident inputs;
* end-to-end: host clock around a block of ``step_pipelined`` calls on pinned host inputs (H2D copy, compute, D2H
  loss of every step), closed by ``flush()``.
Each line reports the median block and the spread (min..max) over ``--repeats`` blocks.  The first line names the card
and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REFERENCE = [784, 128, 127, 126, 125, 124, 123, 10]
LR = 0.006
# "per-step": two rates taken in turn, so no step runs at the rate of the step before it
ARMS = {"constant": None, "per-step": lambda i: LR if i % 2 == 0 else 0.5 * LR}


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
    p.add_argument("--comm", choices=["fused", "nccl", "nvls"], default="fused", help="data-parallel transport")
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=7, help="timed blocks per arm and timing (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    args = p.parse_args()

    import torch
    import torch.distributed as dist

    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import Trainer

    if not torch.cuda.is_available():
        raise SystemExit("lr_schedule_bench: no CUDA device")
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dev = torch.device("cuda", torch.cuda.current_device())
    dp_comm = None
    if args.gpus > 1:
        dist.init_process_group("nccl", rank=rank, world_size=args.gpus, device_id=dev)
        dp_comm, _ = make_torch_comms(ProcessGrid(args.gpus, 1, rank))
    name, limits = card()
    if rank == 0:
        print(json.dumps({"card": name, "power_limit,max_sm_clock": limits, "gpus": args.gpus,
                          "comm": args.comm if args.gpus > 1 else "none"}), flush=True)

    gbs = 128 * args.gpus
    trainers = {arm: Trainer(REFERENCE, global_batch_size=gbs, n_mubatches=4, lr=LR, dp_comm=dp_comm, comm_mode=args.comm,
                             device=dev, lr_schedule=sched)
                for arm, sched in ARMS.items()}
    pool = 16
    x, y = synthetic_mnist(n=pool * gbs)
    r = dp_comm.Get_rank() if dp_comm is not None else 0
    xh = torch.from_numpy(x[r::args.gpus].copy()).reshape(pool, 128, 784).pin_memory()
    yh = torch.from_numpy(y[r::args.gpus].copy()).reshape(pool, 128, 10).pin_memory()
    xd, yd = xh.to(dev), yh.to(dev)

    def sync():
        torch.cuda.synchronize(dev)
        if dp_comm is not None:
            dist.barrier()

    def device_block(tr, n):
        sync()
        st = torch.cuda.ExternalStream(tr.engine.main_stream(), device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(n):
            tr.step_async(xd[i % pool], yd[i % pool])
        e1.record(st)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    def e2e_block(tr, n):
        sync()
        t0 = time.perf_counter()
        for i in range(n):
            tr.step_pipelined(xh[i % pool], yh[i % pool])
        tr.flush()
        torch.cuda.synchronize(dev)
        return 1e3 * (time.perf_counter() - t0) / n

    for tr in trainers.values():
        device_block(tr, args.warmup)
        e2e_block(tr, args.warmup)
    times = {(arm, kind): [] for arm in trainers for kind in ("device", "end_to_end")}
    for _ in range(args.repeats):
        for kind, fn in (("device", device_block), ("end_to_end", e2e_block)):
            for arm, tr in trainers.items():
                times[(arm, kind)].append(fn(tr, args.steps))
    if rank == 0:
        for (arm, kind), ts in times.items():
            s = sorted(ts)
            print(json.dumps({"arm": arm, "timing": kind, "ms_per_step": round(s[len(s) // 2], 5), "min": round(s[0], 5),
                              "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                              "kernels_per_step": int(trainers[arm].engine.kernels_per_step()),
                              "graph_nodes": int(trainers[arm].engine.graph_nodes())}), flush=True)
    del trainers
    if dp_comm is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
