#!/usr/bin/env python
"""Cost of shuffling the training set: the input staging of one step, and the step time of NativeWorker.execute with and
without shuffling.

    python scripts/shuffle_bench.py [--steps 200] [--repeats 3] [--warmup 50] [--profile-steps 50]

Workload: the reference model (784-128-127-126-125-124-123-10, global batch 128, 4 micro-batches, one GPU) on
synthetic MNIST-shaped data (59 500 x 784) resident on the GPU.  Two measurements:

* staging: device time per step of the staging work on the copy stream, from ``torch.profiler`` (CUDA activities) over
  ``--profile-steps`` steps in a run of its own - the two device-to-device ``cudaMemcpy2DAsync`` copies without
  shuffling, the one ``gather_rows_kernel`` launch with it;
* step time: blocks of ``--steps`` steps of ``NativeWorker.execute`` timed with CUDA events on the engine's stream
  between two device synchronisations, the two arms alternated block by block (``--repeats`` blocks each) so that both
  see the same card, clocks and neighbours; each line reports the median block and the spread.

The first line names the card and its power limit.
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
SEED = 20261016


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--steps", type=int, default=200, help="steps per timed block")
    p.add_argument("--repeats", type=int, default=3, help="timed blocks per arm (alternated)")
    p.add_argument("--warmup", type=int, default=50, help="untimed steps per arm before the first block")
    p.add_argument("--profile-steps", type=int, default=50, help="steps traced by torch.profiler per arm")
    args = p.parse_args()

    import torch

    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule

    if not torch.cuda.is_available():
        raise SystemExit("shuffle_bench: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limits = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": limits}), flush=True)

    arms = {}
    for arm in ("plain", "shuffle"):
        model = MLP(SIZES, 0, 1, 128).to(dev)
        opt = SGD(model.parameters(), 0.006, arena=model.arena)
        ds = Dataset(None, 128, 32, synthetic=True, device=dev, shuffle_seed=SEED if arm == "shuffle" else None)
        ds.load(0, 1)
        arms[arm] = (NativeWorker(None, None, model, ds, opt), ds)
    sched = GPipeSchedule(4, 1, 0)
    pos = {arm: 0 for arm in arms}

    def run(arm, n):
        w, ds = arms[arm]
        nb = ds.get_num_batches()
        for _ in range(n):
            i = pos[arm]
            ds.set_epoch(i // nb)
            w.execute(sched, i % nb)
            pos[arm] = i + 1

    def block(arm, n):
        w, _ = arms[arm]
        torch.cuda.synchronize(dev)
        st = torch.cuda.ExternalStream(w.engine_for(sched).main_stream(), device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        run(arm, n)
        e1.record(st)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    for arm in arms:
        run(arm, args.warmup)
    torch.cuda.synchronize(dev)

    # staging device time per step, one traced run per arm
    from torch.profiler import ProfilerActivity, profile

    for arm in arms:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(arm, args.profile_steps)
            torch.cuda.synchronize(dev)
        us, count = 0.0, 0
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            nm = ev.name
            if (arm == "plain" and "Memcpy DtoD" in nm) or (arm == "shuffle" and "gather_rows_kernel" in nm):
                us += ev.time_range.elapsed_us()
                count += 1
        print(json.dumps({"measure": "staging", "arm": arm,
                          "what": "2 x cudaMemcpy2DAsync D2D" if arm == "plain" else "gather_rows_kernel",
                          "launches_per_step": round(count / args.profile_steps, 3),
                          "device_us_per_step": round(us / args.profile_steps, 3), "steps": args.profile_steps}),
              flush=True)

    times = {arm: [] for arm in arms}
    for _ in range(args.repeats):
        for arm in arms:
            times[arm].append(block(arm, args.steps))
    for arm, ts in times.items():
        s = sorted(ts)
        w, _ = arms[arm]
        eng = w.engine_for(sched)
        print(json.dumps({"measure": "step", "arm": arm, "ms_per_step": round(s[len(s) // 2], 5), "min": round(s[0], 5),
                          "max": round(s[-1], 5), "blocks": len(s), "steps": args.steps,
                          "kernels_per_step": int(eng.kernels_per_step()), "graph_nodes": int(eng.graph_nodes()),
                          "loss": round(float(w.batch_loss()), 6)}), flush=True)


if __name__ == "__main__":
    main()
