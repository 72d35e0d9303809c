"""What the TF32 GEMM path does to operand bits just past the 10-bit mantissa (both operand positions)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from shallowspeed_b200.ops import cuda as K
vals = {"1+2^-11+2^-12": 1 + 2**-11 + 2**-12, "1+2^-11 (tie)": 1 + 2**-11, "1+2^-10+2^-11 (tie)": 1 + 2**-10 + 2**-11,
        "1+2^-12": 1 + 2**-12, "-(1+2^-11+2^-12)": -(1 + 2**-11 + 2**-12), "1+2^-10-2^-23": 1 + 2**-10 - 2**-23}
for name, a in vals.items():
    x = torch.zeros(1, 32, device="cuda"); x[0, 0] = a
    w = torch.zeros(8, 32, device="cuda"); w[0, 0] = 1.0
    y = K.linear_fwd(x, w, None)
    xa = torch.zeros(1, 32, device="cuda"); xa[0, 0] = 1.0
    wa = torch.zeros(8, 32, device="cuda"); wa[0, 0] = a          # same value on the A (weight) operand
    ya = K.linear_fwd(xa, wa, None)
    print(f"{name:22s} a={a!r:22} B-operand -> {float(y[0,0])!r:22} A-operand -> {float(ya[0,0])!r}")
