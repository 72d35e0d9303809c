#!/usr/bin/env python
"""Dump the per-role %globaltimer timeline of the chain kernel (SSB_CHAIN_TIMELINE=1)."""
import os
import sys

os.environ["SSB_CHAIN_TIMELINE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from shallowspeed_b200.dataset import synthetic_mnist
from shallowspeed_b200.parallel.engine import Trainer

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
x, y = synthetic_mnist(n=128 * 4)
xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
tr = Trainer(SIZES, use_graph=False, precision=os.environ.get("PREC", "fp32"))
for i in range(6):
    tr.step_async(xd[(i % 4) * 128:(i % 4 + 1) * 128], yd[(i % 4) * 128:(i % 4 + 1) * 128])
tr.synchronize()
t = tr.engine.chain_timeline()
prod, mma, epi = t[0:256], t[256:512], t[512:768]
t0 = min(v for v in t if v > 0)
rel = lambda v: (v - t0) / 1000.0 if v > 0 else None
print("producer tile issue times (us):", [round(rel(v), 2) for v in prod if v > 0])
print("gemm: (start, accumulator complete) of math warp 1 | publish of the tile written after it")
for g in range(14):
    a, b = mma[2 * g:2 * g + 2]
    e = epi[g + 1]
    if a == 0:
        break
    print(f"gemm {g:2d}: mma {rel(a):7.2f} {rel(b):7.2f} | publish {rel(e) if e else -1:7.2f}")
