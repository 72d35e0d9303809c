"""Bit-level model of the fp32-equivalent tensor-core scheme (3xTF32), on the CPU.

The kernels hand the tensor core hi(x) = x with the low 13 mantissa bits cleared (truncation, csrc/kernels/ptx.cuh), so
lo(x) = x - hi(x) is exactly representable in fp32 and has itself <= 13 significant bits (it survives a second truncation
to tf32 with at most a 2^-10 relative loss), and

        a*b  ~=  lo(a)*hi(b) + hi(a)*lo(b) + hi(a)*hi(b)          (the lo*lo term, ~2^-22 relative, is dropped)

This file emulates exactly that arithmetic with integer masks and checks the error levels the GPU tests rely on."""
import numpy as np


def hi(x):
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def lo(x):
    x = x.astype(np.float32)
    return (x - hi(x)).astype(np.float32)


def mm_tf32(a, b):
    """what one kind::tf32 pass computes: truncated operands, exact products, fp32-or-better accumulation"""
    return hi(a).astype(np.float64) @ hi(b).astype(np.float64)


def mm_3xtf32(a, b):
    return mm_tf32(lo(a), b) + mm_tf32(a, lo(b)) + mm_tf32(a, b)


def test_split_is_exact_and_lo_is_small():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(10000) * 10.0 ** rng.integers(-6, 6, 10000)).astype(np.float32)
    assert np.array_equal(hi(x) + lo(x), x)                            # exact decomposition in fp32
    assert np.all(np.abs(lo(x)) <= np.abs(x) * 2.0 ** -10 + 1e-45)     # at most the 13 dropped bits
    assert np.all(np.abs(hi(x)) <= np.abs(x))                          # truncation, never rounds up
    assert np.array_equal(hi(hi(x)), hi(x))


def test_three_pass_scheme_is_fp32_equivalent_single_pass_is_not():
    rng = np.random.default_rng(1)
    a = rng.standard_normal((64, 784)).astype(np.float32)
    b = (rng.standard_normal((784, 128)) / np.sqrt(784)).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    scale = np.abs(ref).max()
    e1 = np.abs(mm_tf32(a, b) - ref).max() / scale
    e3 = np.abs(mm_3xtf32(a, b) - ref).max() / scale
    e32 = np.abs((a @ b).astype(np.float64) - ref).max() / scale       # plain fp32 matmul for comparison
    assert 1e-5 < e1 < 3e-3          # the tolerance class of --precision tf32 (TOL["tf32"] = 3e-3)
    assert e3 < 2e-6                 # well inside TOL["fp32"] = 2e-5 ...
    assert e3 < 20 * max(e32, 1e-8)  # ... and the same order as an fp32 GEMM


def test_dropped_lo_lo_term_is_the_only_systematic_error():
    rng = np.random.default_rng(2)
    a = rng.standard_normal((8, 4096)).astype(np.float32)
    b = rng.standard_normal((4096, 8)).astype(np.float32)
    exact_products = a.astype(np.float64) @ b.astype(np.float64)
    lolo = lo(a).astype(np.float64) @ lo(b).astype(np.float64)
    # the lo parts are truncated once more by the tensor core: that loses at most 2^-10 of a term that is itself 2^-11 small
    resid = exact_products - mm_3xtf32(a, b) - lolo
    assert np.abs(lolo).max() < 1e-4 * np.abs(exact_products).max()
    assert np.abs(resid).max() < 4e-6 * np.abs(exact_products).max()
