"""Bit-level model of the bf16 tensor-core products (``--precision bf16``), on the CPU.

The kernels load fp32 operands from shared memory in the m16n8k8 TF32 fragment pattern, round each to bf16 in registers
(``cvt.rn.bf16x2.f32``: round to nearest, ties to even) and feed the pairs to ``mma.sync.m16n8k16.bf16`` with a fixed
permutation of k (csrc/kernels/ptx.cuh: warp_mma_kblock).  The products of two bf16 values are exact in fp32, so against
the fp64 product of the ROUNDED operands the only error left is the fp32 accumulation, which test_gpu_chain bounds by
2^-16 of sum |a'||b'| (the 3xTF32 class).  This file checks the rounding, the permutation and that this oracle tells
bf16 from tf32 and 3xTF32 results of the same data."""
import numpy as np
import torch

from test_precision_model import hi, mm_3xtf32

RTOL_BF16 = 2.0**-16          # accumulation only: the operands are rounded before the oracle sees them
RTOL_FP32 = 2.0**-16          # test_gpu_chain.RTOL["fp32"]: the unrounded operands
ATOL = 1e-30


def rne_bf16(x):
    """bf16(x) as fp32, by bit arithmetic on the fp32 pattern: add 0x7FFF plus the lowest kept bit, cut 16 bits (round
    to nearest, ties to even; overflow goes to inf through the exponent carry).  NaN stays NaN."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(x), np.float32(np.nan), r)


def torch_bf16(x):
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).bfloat16().float().numpy()


def test_rne_matches_torch_bfloat16():
    rng = np.random.default_rng(0)
    with np.errstate(over="ignore"):     # the widest exponents overflow to inf, which is one more case
        x = (rng.standard_normal(200000) * 10.0 ** rng.integers(-40, 39, 200000)).astype(np.float32)
    f32 = np.finfo(np.float32)
    special = np.array([0.0, -0.0, np.inf, -np.inf, f32.max, -f32.max, f32.tiny, -f32.tiny, f32.smallest_subnormal,
                        2.0**-133, 2.0**-134, 3 * 2.0**-134, 1.0, -1.0], dtype=np.float32)
    # ties: the 16 cut bits exactly 0x8000, with the kept lowest bit 0 (stays) and 1 (rounds up)
    base = (rng.integers(0, 2**15, 4000, dtype=np.uint32) << 16) | 0x8000
    ties = np.concatenate([base, base | 0x10000, base | 0x80000000]).view(np.float32)
    subn = rng.integers(1, 2**23, 4000, dtype=np.uint32).view(np.float32)       # every fp32 subnormal pattern class
    for v in (x, special, ties, subn):
        v = v[np.isfinite(v) | np.isinf(v)]
        assert np.array_equal(rne_bf16(v).view(np.uint32), torch_bf16(v).view(np.uint32))
    # overflow: values that round past bf16's largest finite value become inf, as in torch
    assert np.isinf(rne_bf16(np.array([f32.max], dtype=np.float32)))[0]
    assert np.isnan(rne_bf16(np.array([np.nan], dtype=np.float32)))[0]


def k_map(t):
    """Physical k (offset from the k16 step) of logical k (2t, 2t+1, 2t+8, 2t+9) of thread t = lane % 4 (ptx.cuh)."""
    return {2 * t: t, 2 * t + 1: t + 4, 2 * t + 8: 8 + t, 2 * t + 9: 12 + t}


def test_k_map_is_a_bijection_onto_the_16_k_values():
    m = {}
    for t in range(4):
        for logical, physical in k_map(t).items():
            assert logical not in m
            m[logical] = physical
    assert sorted(m) == list(range(16)) and sorted(m.values()) == list(range(16))
    # and it is the TF32 fragment's load pattern at k0 (t, t + 4) and k0 + 8 (8 + t, 12 + t)
    assert all((k_map(t)[2 * t], k_map(t)[2 * t + 1]) == (t, t + 4) for t in range(4))


def mma_kblock_bf16(A, B):
    """One 32-wide k-block of warp_mma_kblock in bf16: A [16, 32], B [8, 32] (n, k), both fp32.  Builds the logical
    m16n8k16 fragments from the physical tiles through k_map for both k16 steps, rounds them with rne_bf16 and returns
    the fp64 sum of the exact products (what the tensor core would return without accumulation error)."""
    D = np.zeros((16, 8))
    for k0 in (0, 16):
        Al = np.zeros((16, 16))
        Bl = np.zeros((16, 8))
        for t in range(4):
            for logical, physical in k_map(t).items():
                Al[:, logical] = rne_bf16(A[:, k0 + physical])
                Bl[logical, :] = rne_bf16(B[:, k0 + physical])
        D += Al @ Bl
    return D


def test_emulated_mma_equals_the_fp64_product_of_the_rounded_operands():
    rng = np.random.default_rng(1)
    for _ in range(20):
        A = rng.standard_normal((16, 32)).astype(np.float32)
        B = rng.standard_normal((8, 32)).astype(np.float32)
        ref = rne_bf16(A).astype(np.float64) @ rne_bf16(B).astype(np.float64).T
        got = mma_kblock_bf16(A, B)
        assert np.allclose(got, ref, rtol=1e-14, atol=0.0)
        # the products are exact in fp32: 8 + 8 significant bits
        pa = rne_bf16(A[:, :1]).astype(np.float64) * rne_bf16(B[:1, :]).astype(np.float64)
        assert np.array_equal(pa.astype(np.float32).astype(np.float64), pa)


def _fp32_kblocks(a, b):
    """sum over 32-wide k-blocks, each block's sum of exact products rounded to fp32 and added in fp32 (the kernels'
    accumulation, with a tensor core that itself adds exactly)"""
    acc = np.zeros((a.shape[0], b.shape[1]), dtype=np.float32)
    for k0 in range(0, a.shape[1], 32):
        acc = acc + (a[:, k0:k0 + 32].astype(np.float64) @ b[k0:k0 + 32].astype(np.float64)).astype(np.float32)
    return acc.astype(np.float64)


def excess(got, ref, bound):
    return float((np.abs(got - ref) / bound).max())


def test_oracle_separates_the_precisions():
    """The bf16 oracle (fp64 product of the bf16-rounded operands, accumulation-only bound) accepts a bf16 evaluation and
    rejects the tf32 and 3xTF32 evaluations of the same data; the fp32 oracle rejects the bf16 evaluation.

    The data keep the margin wide: the rounding errors of the operands partly cancel in a sum of K terms (they grow like
    sqrt(K)) while the accumulation bound grows like K, so the separation shrinks as K grows.  K = 96 (three k-blocks,
    the reference model's narrow layers are 97 to 128 wide) leaves a factor of more than 10 on either side."""
    rng = np.random.default_rng(2)
    M, K, N = 64, 96, 48
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = rng.standard_normal((K, N)).astype(np.float32)
    ar, br = rne_bf16(a), rne_bf16(b)
    ref = ar.astype(np.float64) @ br.astype(np.float64)
    bound = RTOL_BF16 * (np.abs(ar).astype(np.float64) @ np.abs(br).astype(np.float64)) + ATOL
    bf16 = _fp32_kblocks(ar, br)
    tf32 = _fp32_kblocks(hi(a), hi(b))
    x3 = mm_3xtf32(a, b)
    e_bf16, e_tf32, e_3x = excess(bf16, ref, bound), excess(tf32, ref, bound), excess(x3, ref, bound)
    ref32 = a.astype(np.float64) @ b.astype(np.float64)
    e_fp32 = excess(bf16, ref32, RTOL_FP32 * (np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64)) + ATOL)
    print(f"\n[bf16 model] K={K}: bf16 oracle on bf16 {e_bf16:.3g}, on tf32 {e_tf32:.3g}, on 3xtf32 {e_3x:.3g}; "
          f"fp32 oracle on bf16 {e_fp32:.3g}")
    assert e_bf16 <= 1.0 / 10
    assert e_tf32 > 10 and e_3x > 10 and e_fp32 > 10


def test_precision_names_map_to_the_native_codes():
    """One map from a precision name to the code the kernels take (csrc/kernels/precision.h); unknown names raise
    instead of running tf32."""
    import pytest

    from shallowspeed_b200.ops.functional import precision_code

    assert [precision_code(n) for n in ("fp32", "fp32x3", "3xtf32", "tf32", "bf16")] == [1, 1, 1, 0, 2]
    for bad in ("bf-16", "fp16", "BF16", "", None, 2):
        with pytest.raises(ValueError):
            precision_code(bad)
