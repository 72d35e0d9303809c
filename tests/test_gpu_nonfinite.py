"""NaN and +-Inf through every kernel, per element, against IEEE fp64: the stand-alone GEMMs and their epilogues, split-K,
the loss heads, the update kernels, ``count_correct``, and the one-GPU engine after one step in each launch form.

The class oracle.  Each output element has a class: finite, NaN, +Inf or -Inf (NaN payloads are not compared).  The
class of a product is computed from 0/1 indicators of the operands with fp64 matmuls, which are exact (counts below
2^53), never from an fp64 product over non-finite data: a BLAS may skip zero terms, and ``NaN * 0`` would then vanish.

* a term is NaN when an operand is NaN, or when it is Inf * 0;
* an element is NaN when one of its terms is NaN, or when it has both a +Inf and a -Inf term;
* otherwise it is +-Inf when it has infinite terms of one sign.

The precision's operand model comes first (``operand_class``): bf16 rounds the operands to bf16, so finite values past
the largest bf16 become Inf; tf32 reads the top 19 bits, so a NaN whose payload lies only in the low 13 mantissa bits
(0x7F800001) reads as +-Inf; fp32 (3xTF32) splits x into hi = trunc(x) and lo = x - hi, and lo = Inf - Inf = NaN, so
every term with an infinite operand is NaN.  The fp32 additions of the epilogues (bias, skip, the SGD rules, the bias
column of the weight gradient) are IEEE.  Elementwise steps (activations, masks, gates, the loss heads, the update
rules) are evaluated in fp64 on class representatives, where IEEE arithmetic gives the class directly.

Elements whose class is finite have no term with a non-finite operand.  They are checked either bitwise against the
same launch with every planted operand set to 0 (the stand-alone kernels and the update kernels: the same operands,
the same deterministic order), or, in the engine, with the per-element bounds of test_gpu_chain / test_gpu_bf16
computed from the kernel's own buffers with the non-finite operands set to 0.

The plants: NaN, +Inf, -Inf, NaN with a low-bit payload (0x7F800001, 0xFF800001), Inf against a zero of the other
operand, a +Inf and a -Inf term in one dot product, and in bf16 a finite 3.4e38 that rounds to Inf; at the first and
last row of a 128-row tile and row 129, at k = 31 / 32 / 33 and the last ragged k, either side of a split-K boundary,
and in one micro-batch of several.  Masks (the ReLU mask, the dropout keep) select: a masked-off NaN is +0.  Gates
(the smooth activations' f'(z) and the residual forms) multiply.

The engine grid covers the cluster chain at C = 4 and 2, the one-CTA chain, the k-split first layer (an input plant in
k-block 2, the helper's half), per-micro-batch launches, the layer-wise path, forced split-K and residual models on the
chain and layer-wise paths, with MSE and cross-entropy, ReLU and GELU, with and without dropout, in fp32, tf32 and bf16;
each case reads its launch form back from the engine.  The data-parallel replay (test_gpu_dp_replay's harness, replica 0
of dp 2 under LL and under the one-shot and two-shot flag protocols) plants NaN / +-Inf in the peer's partials, bias
column included, and under LL in the rows it sends back.  Not covered here: the pipeline replay and the multi-GPU
transports.

The CPU tests at the end check the class oracle against numpy's elementwise products, that the engine grid reaches
every launch form, and that the checks reject emulated faults (an fmaxf ReLU, a multiplied mask, a NaN-blind global
max, a NaN row leaking into the next micro-batch, a stale NaN surviving into the next launch) while they accept a
clean emulation.

Measured on an H100 80GB HBM3 (700 W): the H100's mma.sync follows the class oracle (Inf * 0 inside a k-block is NaN, a
+Inf and a -Inf term give NaN, tf32 reads 0x7F800001 as +Inf); the worst err / bound of the finite elements in the
engine is 0.85 (a tf32 dgrad); the file runs in 30 s.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from test_gpu_chain import (ATOL, HEAD_RTOL, RTOL, U, _init_weights, act_dgrad_oracle, act_fwd_oracle, dgrad_oracle,
                            excess, fwd_oracle, head_oracle, rows_update_oracle, tf32_trunc)

FIN, NAN_C, PINF, NINF = 0, 1, 2, 3
NAMES = {FIN: "finite", NAN_C: "NaN", PINF: "+Inf", NINF: "-Inf"}
INF = math.inf
NAN = math.nan


LOWNAN_P = 0x7F800001         # NaN, payload only in the low mantissa bit: +Inf to the tf32 tensor core
LOWNAN_N = 0xFF800001
BIG = 3.4e38                  # finite in fp32, rounds to +Inf in bf16


def _lownan(bits):
    t = torch.tensor([bits], dtype=torch.int64).to(torch.int32)
    return t.view(torch.float32)


def put(t, i, j, v):
    """t[i, j] = v, where v is a float or one of LOWNAN_P / LOWNAN_N (bits)."""
    if isinstance(v, int):
        t[i, j] = _lownan(v).to(t.device)[0]
    else:
        t[i, j] = v


# ================================================================================================== the class oracle
def classes(t):
    """The class of every element of ``t`` (FIN, NAN_C, PINF, NINF) as an int8 tensor on the CPU."""
    t = t.detach().double().cpu()
    c = torch.zeros(t.shape, dtype=torch.int8)
    c[t == INF] = PINF
    c[t == -INF] = NINF
    c[t.isnan()] = NAN_C
    return c


def rep(cls, finite):
    """fp64 representatives: ``finite`` where the class is finite, else NaN / +Inf / -Inf."""
    r = finite.double().clone()
    r[cls == NAN_C] = NAN
    r[cls == PINF] = INF
    r[cls == NINF] = -INF
    return r


def operand_class(t, precision):
    """The operand the products see, as fp64: fp32 / ieee as is, tf32 truncated, bf16 rounded."""
    t = t.detach().float().cpu()
    if precision == "tf32":
        return tf32_trunc(t).double()
    if precision == "bf16":
        return t.bfloat16().double()
    return t.double()


def class_matmul(A, B, precision="ieee", bias=None):
    """The class of every element of A @ B (+ bias, an IEEE fp32 addition) under the precision's operand model (see the
    module docstring), from exact 0/1 matmuls.  A: [n, k], B: [k, m]; ``precision``: "fp32" (3xTF32), "tf32", "bf16"
    or "ieee" (plain IEEE products: the fp32 column sums of the bias gradient)."""
    model = "ieee" if precision == "fp32" else precision
    a, b = operand_class(A, model), operand_class(B, model)
    ones = lambda x: x.double()
    if precision == "fp32":
        # 3xTF32: every term with a non-finite operand is NaN
        nanA, nanB = ~torch.isfinite(a), ~torch.isfinite(b)
        infA = infB = None
    else:
        nanA, nanB = a.isnan(), b.isnan()
        infA, infB = a.isinf(), b.isinf()
    n, k = a.shape
    m = b.shape[1]
    nan_t = ones(nanA) @ torch.ones(k, m, dtype=torch.float64) + torch.ones(n, k, dtype=torch.float64) @ ones(nanB)
    if infA is not None:
        zA, zB = a == 0, b == 0
        nan_t = nan_t + ones(infA) @ ones(zB) + ones(zA) @ ones(infB)
        PA, NA, PB, NB = a > 0, a < 0, b > 0, b < 0          # NaN compares false: not a sign
        pos = (ones(infA & PA) @ ones(PB) + ones(infA & NA) @ ones(NB)
               + ones(PA) @ ones(infB & PB) + ones(NA) @ ones(infB & NB))
        neg = (ones(infA & PA) @ ones(NB) + ones(infA & NA) @ ones(PB)
               + ones(PA) @ ones(infB & NB) + ones(NA) @ ones(infB & PB))
    else:
        pos = neg = torch.zeros(n, m, dtype=torch.float64)
    if bias is not None:
        bb = bias.detach().double().cpu().reshape(1, -1)
        nan_t = nan_t + bb.isnan().double()
        pos = pos + (bb == INF).double()
        neg = neg + (bb == -INF).double()
    c = torch.zeros(n, m, dtype=torch.int8)
    c[pos > 0] = PINF
    c[neg > 0] = NINF
    c[(nan_t > 0) | ((pos > 0) & (neg > 0))] = NAN_C
    return c


def zeroed(t, precision="ieee"):
    """``t`` as fp64 with every operand that is non-finite under the precision's model set to 0 (the finite oracle's
    input: no finite-class element has a term with such an operand)."""
    t = t.detach().double().cpu().clone()
    t[~torch.isfinite(operand_class(t, precision))] = 0.0
    return t


def class_mismatch(got, want):
    """None when every element of ``got`` has the class ``want``, else a description of the first few that do not."""
    gc = classes(got)
    bad = (gc != want).nonzero()
    if bad.numel() == 0:
        return None
    w = [(tuple(i.tolist()), NAMES[int(gc[tuple(i)])], NAMES[int(want[tuple(i)])]) for i in bad[:4]]
    return f"{bad.shape[0]} of {gc.numel()} elements: (index, got, want) {w}"


def assert_classes(got, want, what):
    msg = class_mismatch(got, want)
    assert msg is None, f"{what}: {msg}"


def bitwise_mismatch(got, clean, where):
    """None when ``got`` and ``clean`` have the same bits wherever ``where`` is set."""
    g = got.detach().float().contiguous().cpu().view(torch.int32)
    c = clean.detach().float().contiguous().cpu().view(torch.int32)
    bad = ((g != c) & where).nonzero()
    if bad.numel() == 0:
        return None
    return f"{bad.shape[0]} elements differ from the clean run, first {[tuple(i.tolist()) for i in bad[:4]]}"


def finite_excess(got, ref, bound, want):
    """max err / bound over the elements whose class is finite."""
    f = want == FIN
    if not bool(f.any()):
        return 0.0
    return excess(got.detach().double().cpu()[f], ref[f], bound[f])


def relu_class(c):
    """ReLU of a class: NaN and +Inf stay, -Inf becomes the finite +0."""
    c = c.clone()
    c[c == NINF] = FIN
    return c


def _K():
    from shallowspeed_b200.ops import cuda as K

    return K


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ================================================================================================== stand-alone GEMMs
# (rows, M, K) from test_gpu_gemm.GRID's tile edges: 2 M tiles (row 129), k-blocks 31 / 32 / 33, a ragged last k
GEMM_GRID = [(17, 129, 65), (65, 300, 100), (1, 129, 33), (33, 1000, 777)]
PRECISIONS = ["fp32", "tf32", "bf16"]


def _plants_x(rows, k, precision):
    """(row, col, value) plants of the activation operand: Inf against zeros, a +Inf and a -Inf term in one row,
    low-payload NaNs at the k-block edges and the last k.  None for a single row, which any of them would make
    non-finite as a whole: the other operand's plants reach it there."""
    if rows == 1:
        return []
    last = rows - 1
    p = [(0, 31, NAN), (last, k - 1, LOWNAN_P), (min(1, last), min(32, k - 1), INF), (min(1, last), min(33, k - 1), -INF)]
    if rows > 2:
        p.append((rows // 2, 0, LOWNAN_N))
    if precision == "bf16":
        p.append((last, min(33, k - 1), BIG))
    return p


def _plants_w(m, k, precision):
    """Plants of the weight operand at the first and last row of the first 128-row tile and row 129."""
    p = [(0, min(32, k - 1), -INF), (min(127, m - 1), min(33, k - 1), NAN), (min(128, m - 1), k - 1, INF)]
    if precision == "bf16":
        p.append((min(127, m - 1), 0, -BIG))
    return p


def _planted(shape, gen, plants, scale=1.0, zero_col=None):
    """(planted, clean) CPU tensors: random values, the planted entries non-finite in one and 0 in the other.
    ``zero_col``: every third entry of this column is an exact zero in both (an Inf of the other operand meets them)."""
    t = torch.randn(*shape, generator=gen) * scale
    if zero_col is not None:
        t[1::3, zero_col] = 0.0
    clean = t.clone()
    for i, j, v in plants:
        put(t, i, j, v)
        clean[i, j] = 0.0
    return t, clean


def _cuda_pitched(t, extra=4):
    rows, cols = t.shape
    ld = (cols + 3) // 4 * 4 + extra
    buf = torch.full((rows, ld), NAN)
    buf[:, :cols] = t
    buf = buf.cuda()
    return buf[:, :cols]


def _launch_pair(launch, shapes):
    """Run ``launch(outs, planted=bool)`` on fresh sentinel outputs for the planted and the clean operands."""
    res = []
    for planted in (True, False):
        outs = [torch.full((r, (c + 3) // 4 * 4 + 4), -1234.5, device="cuda")[:, :c] for r, c in shapes]
        launch(outs, planted)
        torch.cuda.synchronize()
        res.append([o.cpu() for o in outs])
    return res


def _check_out(got, clean, want, what, finite_zero=None):
    """Classes as ``want``; finite-class elements bitwise the clean launch, except ``finite_zero`` (ReLU'd -Inf): +0."""
    assert_classes(got, want, what)
    fin = want == FIN
    if finite_zero is not None:
        z = got[finite_zero & fin]
        assert bool((z.view(torch.int32) == 0).all()), f"{what}: a ReLU of -Inf is not +0"
        fin = fin & ~finite_zero
    msg = bitwise_mismatch(got, clean, fin)
    assert msg is None, f"{what}: {msg}"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("rows,m,k", GEMM_GRID)
def test_fwd_epilogues(rows, m, k, precision):
    """FWD with bias, ReLU, GELU and its gate, and the residual skip: classes and clean bits."""
    from shallowspeed_b200.ops import functional as F

    K = _K()
    gen = _gen("nf-fwd", rows, m, k, precision)
    x, x0 = _planted((rows, k), gen, _plants_x(rows, k, precision), zero_col=min(32, k - 1))
    W, W0 = _planted((m, k), gen, _plants_w(m, k, precision), scale=1.0 / math.sqrt(k), zero_col=min(33, k - 1))
    b = torch.randn(m, generator=gen) * 0.5
    b0 = b.clone()
    b[min(2, m - 1)] = -INF                               # a -Inf bias: -Inf, or NaN against a +Inf term
    b0[min(2, m - 1)] = 0.0
    skip = torch.randn(rows, m, generator=gen)
    skip0 = skip.clone()
    skip[rows - 1, 0] = INF
    skip0[rows - 1, 0] = 0.0
    ops = {True: [_cuda_pitched(t) for t in (x, W, skip)] + [b.cuda()],
           False: [_cuda_pitched(t) for t in (x0, W0, skip0)] + [b0.cuda()]}
    cz = class_matmul(x, W.T, precision, bias=b)
    assert bool((cz == NAN_C).any()) and bool((cz == FIN).any())
    if precision != "fp32":
        assert bool((cz == PINF).any()) and bool((cz == NINF).any()), "the plants reach no +-Inf"
    # bias only, no activation
    got, clean = _launch_pair(lambda o, p: K.linear_fwd(ops[p][0], ops[p][1], ops[p][3], relu=False, out=o[0],
                                                        precision=precision), [(rows, m)])
    _check_out(got[0], clean[0], cz, "fwd+bias")
    # ReLU: NaN stays NaN, -Inf gives +0
    got, clean = _launch_pair(lambda o, p: K.linear_fwd(ops[p][0], ops[p][1], ops[p][3], relu=True, out=o[0],
                                                        precision=precision), [(rows, m)])
    _check_out(got[0], clean[0], relu_class(cz), "fwd+relu", finite_zero=cz == NINF)
    # the finite elements of the clean launch within test_gpu_chain's bound
    from test_gpu_residual import operand_model

    op, rtol = operand_model(precision)
    ref, bound = fwd_oracle(op(x0), op(W0), b0, True, rtol)
    assert excess(clean[0], ref, bound) <= 1.0
    # GELU and its gate: the class of f(z) and f'(z) at the class representative
    zr = rep(cz, torch.zeros(rows, m))
    fa, fg = F.activation_ref("gelu", zr)
    got, clean = _launch_pair(lambda o, p: K.linear_fwd(ops[p][0], ops[p][1], ops[p][3], relu=True, out=o[0],
                                                        precision=precision, activation="gelu", gate=o[1]),
                              [(rows, m), (rows, m)])
    fin_z = cz == FIN
    for g, c, f, what in ((got[0], clean[0], fa, "gelu act"), (got[1], clean[1], fg, "gelu gate")):
        want = torch.where(fin_z, torch.zeros_like(cz), classes(f))
        _check_out(g, c, want, what)
    # residual: f(z) + skip, the ReLU gated (act_fwd_any)
    ra, rg = F.activation_ref("relu", zr)
    sk = ops[True][2].cpu().double()
    got, clean = _launch_pair(lambda o, p: K.linear_fwd(ops[p][0], ops[p][1], ops[p][3], relu=True, out=o[0],
                                                        precision=precision, gate=o[1], residual=True, skip=ops[p][2]),
                              [(rows, m), (rows, m)])
    want_a = classes(torch.where(fin_z, torch.zeros(rows, m, dtype=torch.float64), ra)
                     + torch.where(torch.isfinite(sk), torch.zeros_like(sk), sk))
    assert_classes(got[0], want_a, "residual act")
    assert_classes(got[1], torch.where(fin_z, torch.zeros_like(cz), classes(rg)), "residual gate")
    keep = (want_a == FIN) & fin_z & torch.isfinite(sk)
    assert bitwise_mismatch(got[0], clean[0], keep) is None, "residual act: finite elements differ from the clean run"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("rows,m,k", GEMM_GRID)
def test_dgrad_epilogues(rows, m, k, precision):
    """DGRAD with the ReLU mask (select: a masked-off NaN is +0), a gate (multiply) and the residual gpre."""
    K = _K()
    gen = _gen("nf-dgrad", rows, m, k, precision)
    dz, dz0 = _planted((rows, k), gen, _plants_x(rows, k, precision), zero_col=min(32, k - 1))
    W, W0 = _planted((k, m), gen, [(min(31, k - 1), 0, NAN), (k - 1, min(127, m - 1), INF), (min(32, k - 1), min(128, m - 1), -INF)],
                     scale=1.0 / math.sqrt(k))
    mask = torch.randn(rows, m, generator=gen)
    mask.view(-1)[1::7] = -0.0
    mask[0, min(5, m - 1)] = NAN                                     # a NaN mask is off
    gate = torch.randn(rows, m, generator=gen)
    gate.view(-1)[0::5] = 0.0                                        # Inf * a zero gate is NaN
    skip = torch.randn(rows, m, generator=gen)
    skip[0, 0] = -INF
    skip0 = skip.clone()
    skip0[0, 0] = 0.0
    dev = {True: [_cuda_pitched(t) for t in (dz, W, skip)], False: [_cuda_pitched(t) for t in (dz0, W0, skip0)]}
    mk, gt = _cuda_pitched(mask, extra=8), _cuda_pitched(gate)
    cp = class_matmul(dz, W, precision)
    assert bool((cp != FIN).any()) and bool((cp == FIN).any())
    on = mask > 0
    # ReLU mask: select
    got, clean = _launch_pair(lambda o, p: K.linear_dgrad(dev[p][0], dev[p][1], mask=mk, out=o[0], precision=precision),
                              [(rows, m)])
    want = torch.where(on, cp, torch.zeros_like(cp))
    _check_out(got[0], clean[0], want, "dgrad+relu-mask", finite_zero=~on)
    # gate: multiply
    got, clean = _launch_pair(lambda o, p: K.linear_dgrad(dev[p][0], dev[p][1], mask=gt, out=o[0], precision=precision,
                                                          activation="gelu"), [(rows, m)])
    want = classes(rep(cp, torch.ones(rows, m)) * gate.double())
    _check_out(got[0], clean[0], want, "dgrad+gate")
    # residual: gpre = dz @ W + skip, out = gpre * gate
    got, clean = _launch_pair(lambda o, p: K.linear_dgrad(dev[p][0], dev[p][1], mask=gt, out=o[0], precision=precision,
                                                          residual=True, skip=dev[p][2], gpre=o[1]), [(rows, m), (rows, m)])
    pre = rep(cp, torch.ones(rows, m)) + torch.where(torch.isfinite(skip), torch.zeros(rows, m), skip).double()
    _check_out(got[1], clean[1], classes(pre), "residual gpre")
    _check_out(got[0], clean[0], classes(pre * gate.double()), "residual dgrad")


SPLITK = [(100, 1500, 777, 2), (65, 256, 4096, 3)]                 # k-blocks 13 + 12; 43 + 43 + 42


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("rows,m,k,splits", SPLITK)
def test_splitk_boundary(rows, m, k, splits, precision):
    """Forced split-K FWD (bias + ReLU) and DGRAD (mask) with plants either side of every split boundary."""
    K = _K()
    nkb = (k + 31) // 32
    per = (nkb + splits - 1) // splits
    edges = [32 * per * s for s in range(1, splits)]
    gen = _gen("nf-splitk", rows, m, k, precision)
    px = []
    for i, e in enumerate(edges):
        px += [(min(i, rows - 1), e - 1, NAN), (min(i + 3, rows - 1), e, INF), (min(i + 3, rows - 1), e + 1, -INF)]
    x, x0 = _planted((rows, k), gen, px)
    W, W0 = _planted((m, k), gen, [(128, edges[0], INF), (127, edges[0] - 1, -INF)], scale=1.0 / math.sqrt(k))
    b = (torch.randn(m, generator=gen) * 0.5).cuda()
    dx = {True: _cuda_pitched(x), False: _cuda_pitched(x0)}
    dw = {True: _cuda_pitched(W), False: _cuda_pitched(W0)}
    cz = class_matmul(x, W.T, precision, bias=b)
    got, clean = _launch_pair(lambda o, p: K.linear_fwd(dx[p], dw[p], b, relu=True, out=o[0], precision=precision,
                                                        k_splits=splits), [(rows, m)])
    _check_out(got[0], clean[0], relu_class(cz), f"split-K {splits} fwd", finite_zero=cz == NINF)
    # DGRAD: dz [rows, k] @ W' [k, m'] with W' = W.T
    Wt = {p: _cuda_pitched(w.T.contiguous()) for p, w in ((True, W), (False, W0))}
    mask = torch.randn(rows, m, generator=gen)
    mk = _cuda_pitched(mask)
    cp = class_matmul(x, W.T, precision)
    got, clean = _launch_pair(lambda o, p: K.linear_dgrad(dx[p], Wt[p], mask=mk, out=o[0], precision=precision,
                                                          k_splits=splits), [(rows, m)])
    _check_out(got[0], clean[0], torch.where(mask > 0, cp, torch.zeros_like(cp)), f"split-K {splits} dgrad",
               finite_zero=~(mask > 0))


WGRAD = [(33, 65, 129), (128, 200, 300)]                             # rows (the GEMM's K), in, out


def _check_padding(got, clean, n_in, what):
    """Every column past the bias slot has the clean launch's bits.  The 16-byte TMA store of the last chunk reaches
    the columns (in, round_up(in, 4)) and the bias slot: the epilogue stages +0 there, not dZ^T times the zero-filled
    columns of x, which a non-finite dZ would make NaN (Inf * 0) and add into the bias gradient."""
    assert torch.equal(got[:, n_in + 1:].view(torch.int32), clean[:, n_in + 1:].view(torch.int32)), f"{what}: padding changed"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("rows,n_in,out", WGRAD)
def test_wgrad_and_fused_update(rows, n_in, out, precision):
    """WGRAD: the weight and bias-column classes, plain and accumulating; the fused SGD epilogue under the plain rule,
    momentum and the EMA: weight, momentum and EMA non-finite exactly where the rule's fp64 evaluation is."""
    from shallowspeed_b200.ops import functional as F

    K = _K()
    gen = _gen("nf-wgrad", rows, n_in, out, precision)
    dz, dz0 = _planted((rows, out), gen, [(0, 0, NAN), (rows - 1, min(127, out - 1), INF), (rows // 2, min(128, out - 1), LOWNAN_N)])
    x, x0 = _planted((rows, n_in), gen, [(min(1, rows - 1), 31, -INF), (rows - 1, 32, LOWNAN_P)]
                     + ([(2, 33, BIG)] if precision == "bf16" else []), zero_col=40)
    d = {True: (_cuda_pitched(dz), _cuda_pitched(x)), False: (_cuda_pitched(dz0), _cuda_pitched(x0))}
    cw = class_matmul(dz.T, x, precision)
    cb = class_matmul(dz.T, torch.ones(rows, 1), "ieee")
    cg = torch.cat([cw, cb], dim=1)
    assert bool((cg == FIN).any()) and bool((cg != FIN).any())
    ld = (n_in + 1 + 3) // 4 * 4 + 4
    init = torch.randn(out, n_in + 1, generator=gen)
    for accumulate in (False, True):
        outs = {}
        for p in (True, False):
            g = torch.full((out, ld), -1234.5)
            g[:, : n_in + 1] = init
            g = g.cuda()
            K.linear_wgrad(d[p][0], d[p][1], g[:, :n_in], accumulate=accumulate, grad_b=g[:, n_in], precision=precision)
            torch.cuda.synchronize()
            outs[p] = g.cpu()
        _check_out(outs[True][:, : n_in + 1], outs[False][:, : n_in + 1], cg, f"wgrad accumulate={accumulate}")
        _check_padding(outs[True], outs[False], n_in, f"wgrad accumulate={accumulate}")
    lr, mu, alpha = 0.25, 0.9, 0.3
    for rule in ("plain", "momentum", "ema"):
        outs = {}
        for p in (True, False):
            bufs = [torch.full((out, ld), -1234.5) for _ in range(3)]           # W, V, EMA
            g2 = torch.Generator().manual_seed(7)
            for bb in bufs:
                bb[:, : n_in + 1] = torch.randn(out, n_in + 1, generator=g2) * 0.5
            w, v, e = [bb.cuda() for bb in bufs]
            gsc = torch.full((out, ld), -1234.5, device="cuda")
            kw = {}
            if rule == "momentum":
                kw = dict(velocity=v[:, :n_in], momentum=mu)
            elif rule == "ema":
                kw = dict(ema=e[:, :n_in], ema_alpha=alpha)
            K.linear_wgrad(d[p][0], d[p][1], gsc[:, :n_in], grad_b=gsc[:, n_in], weight=w[:, :n_in], lr=lr, fuse_sgd=True,
                           precision=precision, **kw)
            torch.cuda.synchronize()
            outs[p] = (w.cpu(), v.cpu(), e.cpu(), [bb for bb in bufs])
        W0, V0, E0 = [bb[:, : n_in + 1].double() for bb in outs[True][3]]
        grep_ = rep(cg, torch.zeros(out, n_in + 1))
        if rule == "momentum":
            V1 = mu * V0 + grep_
            W1 = W0 - lr * V1
        else:
            V1, W1 = V0, W0 - lr * grep_
        E1 = F.ema_lerp_ref(E0, W1, alpha) if rule == "ema" else E0
        for i, (want, what) in enumerate(((W1, "weight"), (V1, "momentum"), (E1, "ema"))):
            _check_out(outs[True][i][:, : n_in + 1], outs[False][i][:, : n_in + 1], classes(want), f"fused {rule} {what}")
            _check_padding(outs[True][i], outs[False][i], n_in, f"fused {rule} {what}")


# ================================================================================================== update kernels
@pytest.mark.gpu
@pytest.mark.parametrize("n,offset", [(4096, 0), (4099, 0), (4096, 1)], ids=["float4", "odd-tail", "offset-view"])
@pytest.mark.parametrize("rule", ["sgd", "plain", "momentum", "nesterov+wd", "ema"])
def test_update_kernels(rule, n, offset):
    """sgd_ and sgd_momentum_ (float4 body and scalar tail): only the rule's non-finite entries are non-finite, every
    other entry bitwise the clean run."""
    from shallowspeed_b200.ops import functional as F

    K = _K()
    gen = _gen("nf-upd", rule, n, offset)
    g = torch.randn(n + offset, generator=gen)
    g0 = g.clone()
    idx = [offset, offset + 1, offset + 2, offset + n // 2, offset + n - 1, offset + n - 2]
    vals = [NAN, INF, -INF, _lownan(LOWNAN_P)[0].item(), NAN, -INF]
    for i, v in zip(idx, vals):
        g[i] = v
        g0[i] = 0.0
    w = torch.randn(n + offset, generator=gen)
    v = torch.randn(n + offset, generator=gen) * 0.1
    e = torch.randn(n + offset, generator=gen)
    lr, mu, wd, alpha = 0.1, 0.9, 0.01, 0.7
    outs = {}
    for p, gg in ((True, g), (False, g0)):
        W, V, E, G = (t.clone().cuda() for t in (w, v, e, gg))
        sl = slice(offset, offset + n)
        if rule == "sgd":
            K.sgd_step_(W[sl], G[sl], lr)
        elif rule == "plain":
            K.sgd_momentum_step_(W[sl], G[sl], None, lr, 0.0)
        elif rule == "momentum":
            K.sgd_momentum_step_(W[sl], G[sl], V[sl], lr, mu)
        elif rule == "nesterov+wd":
            K.sgd_momentum_step_(W[sl], G[sl], V[sl], lr, mu, weight_decay=wd, nesterov=True)
        else:
            K.sgd_momentum_step_(W[sl], G[sl], V[sl], lr, mu, ema=E[sl], ema_alpha=alpha)
        torch.cuda.synchronize()
        outs[p] = (W.cpu(), V.cpu(), E.cpu())
    gr = g.double()
    w64, v64 = w.double(), v.double()
    gp = gr + (wd * w64 if rule == "nesterov+wd" else 0.0)
    if rule in ("sgd", "plain"):
        V1, W1 = v64, w64 - lr * gp
    else:
        V1 = mu * v64 + gp
        W1 = w64 - lr * ((gp + mu * V1) if rule == "nesterov+wd" else V1)
    E1 = F.ema_lerp_ref(e.double(), W1, alpha) if rule == "ema" else e.double()
    outside = torch.ones(n + offset, dtype=torch.bool)
    outside[offset: offset + n] = False
    for i, (want, what) in enumerate(((W1, "weight"), (V1, "momentum"), (E1, "ema"))):
        wc = classes(want)
        wc[outside] = FIN
        _check_out(outs[True][i], outs[False][i], wc, f"{rule} {what}")


# ================================================================================================== loss heads, argmax
def _head_plants(logits, case):
    z = logits.clone()
    if case == "nan":
        z[3, 2] = NAN
    elif case == "+inf":
        z[0, 9] = INF
    elif case == "-inf":
        z[5, 0] = -INF
        z[7, 4] = -INF
    elif case == "lownan":
        z[-1, -1] = _lownan(LOWNAN_N)[0]
    return z


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nan", "+inf", "-inf", "lownan"])
@pytest.mark.parametrize("loss", ["mse", "cross_entropy"])
def test_loss_head_kernel(loss, case):
    """loss_head_kernel (MSE modes 0-2, cross-entropy 3-4): probs, dlogits and the loss carry the fp64 oracle's classes
    (MSE: one NaN logit poisons the micro-batch through its global max), the finite ones within its bound."""
    K = _K()
    from test_gpu_cross_entropy import ce_head_oracle

    gen = _gen("nf-head", loss, case)
    rows, C = 40, 10
    z = _head_plants(torch.randn(rows, C, generator=gen) * 3.0, case)
    t = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    dz, p, lv = K.loss_head_backward(z.cuda(), t.cuda(), rows, loss=loss)
    pp = K.softmax(z.cuda(), loss=loss)
    torch.cuda.synchronize()
    oracle = head_oracle if loss == "mse" else ce_head_oracle
    (pr, bp), (gr, bg), (lr_, bl) = oracle(z, t, rows, HEAD_RTOL)
    for got, ref, bound, what in ((p, pr, bp, "probs"), (pp, pr, bp, "softmax"), (dz, gr, bg, "dlogits")):
        want = classes(ref)
        assert_classes(got.cpu(), want, f"{loss} {case} {what}")
        assert finite_excess(got, ref, bound, want) <= 1.0, what
    assert_classes(torch.tensor([float(lv)]), classes(torch.tensor([lr_])), f"{loss} {case} loss")
    if loss == "mse" and case == "nan":
        assert bool(p.isnan().all()), "one NaN logit must poison the whole micro-batch (global max)"
    if loss == "mse":
        up = torch.randn(rows, C, generator=gen)
        g2 = K.softmax_grad(up.cuda(), z.cuda())
        from shallowspeed_b200.ops import functional as F

        assert_classes(g2.cpu(), classes(F.softmax_grad_ref(up.double(), z.double())), f"softmax_grad {case}")


@pytest.mark.gpu
def test_count_correct_treats_nan_as_the_maximum():
    """count_correct against torch.argmax (NaN the maximum, the first NaN winning) on rows with NaN, +-Inf and ties."""
    K = _K()
    gen = _gen("nf-argmax")
    rows, C = 300, 10
    pred = torch.randn(rows, C, generator=gen)
    tgt = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    for r in range(0, rows, 3):
        pred[r, (r // 3) % C] = NAN
    for r in range(0, rows, 5):
        pred[r, (r // 5 + 3) % C] = NAN                # rows with two NaNs: the first wins
    for r in range(1, rows, 7):
        pred[r, (r + 1) % C] = INF
    for r in range(2, rows, 11):
        pred[r] = -INF                                  # all -Inf: index 0
    tgt[4] = 0.0
    tgt[4, 7] = NAN                                     # a NaN in the target wins there too
    want = int((pred.argmax(1) == tgt.argmax(1)).sum())
    assert want == int((torch.from_numpy(np.argmax(pred.numpy(), 1)) == tgt.argmax(1)).sum())
    got = int(K.count_correct(pred.cuda(), tgt.cuda()).item())
    assert got == want, (got, want)
    # wide rows: more columns than lanes, NaN in the second pass of a lane
    pred = torch.randn(8, 100, generator=gen)
    tgt = torch.nn.functional.one_hot(torch.arange(8) * 7 + 40, 100).float()
    for r in range(8):
        pred[r, 40 + 7 * r] = NAN
    pred[3, 70] = INF
    assert int(K.count_correct(pred.cuda(), tgt.cuda()).item()) == int((pred.argmax(1) == tgt.argmax(1)).sum()) == 8


# ================================================================================================== the engine
# name -> (sizes, mb_rows, n_mu, env); a "res-" form is a residual model (a skip around every 128 -> 128 layer)
FORMS = {
    "cluster-c4": ([784, 128, 97, 33, 10], 40, 3, {}),
    "cluster-c2": ([100] + [40] * 15 + [10], 24, 2, {}),
    "one-cta": ([33, 32, 31, 17], 100, 2, {}),
    "ksplit-first": ([160, 128, 97, 33, 10], 64, 2, {}),
    "per-micro-batch": ([784, 128, 97, 33, 10], 40, 3, {"SSB_NO_COALESCE": "1"}),
    "layer-wise": ([784, 128, 97, 33, 10], 40, 3, {"SSB_NO_CHAIN": "1"}),
    "splitk-wide": ([784, 512, 256, 10], 64, 2, {"SSB_SPLITK": "2"}),
    "res-chain": ([784, 128, 128, 128, 10], 40, 3, {}),
    "res-per-micro-batch": ([784, 128, 128, 128, 10], 40, 3, {"SSB_NO_COALESCE": "1"}),
    "res-layer-wise": ([784, 128, 128, 128, 10], 40, 3, {"SSB_NO_CHAIN": "1"}),
}
CHAIN_FORMS = {"cluster-c4", "cluster-c2", "one-cta", "ksplit-first", "per-micro-batch", "res-chain",
               "res-per-micro-batch"}


def check_launch_form(form, eng):
    """The engine runs the form the case is named for, read from the engine itself."""
    assert eng.uses_chain() == (form in CHAIN_FORMS), (form, eng.describe())
    if form == "cluster-c4":
        assert eng.chain_cluster() == 4
    elif form == "cluster-c2":
        assert eng.chain_cluster() == 2
    elif form == "one-cta":
        assert eng.chain_cluster() == 1
    elif form == "ksplit-first":
        assert eng.chain_cluster() > 1 and eng.chain_ksplit() == 2, (eng.chain_cluster(), eng.chain_ksplit())
    elif form == "splitk-wide":
        assert "splitk_gemms=0" not in eng.describe(), eng.describe()
    if form in ("per-micro-batch", "res-per-micro-batch"):
        assert not eng.coalesced()
PLANTS = ["input", "weight", "bias"]
# (form, precision, loss, activation, dropout): a covering grid
ENGINE_GRID = [
    ("cluster-c4", "fp32", "mse", "relu", 0.0),
    ("cluster-c4", "tf32", "cross_entropy", "gelu", 0.3),
    ("cluster-c4", "bf16", "mse", "relu", 0.3),
    ("cluster-c2", "tf32", "mse", "relu", 0.0),
    ("cluster-c2", "fp32", "cross_entropy", "relu", 0.3),
    ("one-cta", "bf16", "cross_entropy", "relu", 0.0),
    ("one-cta", "fp32", "mse", "gelu", 0.0),
    ("ksplit-first", "tf32", "mse", "relu", 0.0),
    ("ksplit-first", "bf16", "cross_entropy", "gelu", 0.3),
    ("per-micro-batch", "fp32", "cross_entropy", "relu", 0.0),
    ("per-micro-batch", "tf32", "mse", "gelu", 0.3),
    ("layer-wise", "bf16", "mse", "gelu", 0.0),
    ("layer-wise", "tf32", "cross_entropy", "relu", 0.3),
    ("splitk-wide", "fp32", "mse", "relu", 0.0),
    ("splitk-wide", "tf32", "cross_entropy", "relu", 0.0),
    ("res-chain", "fp32", "mse", "relu", 0.0),
    ("res-chain", "tf32", "cross_entropy", "gelu", 0.3),
    ("res-chain", "bf16", "cross_entropy", "relu", 0.3),
    ("res-per-micro-batch", "fp32", "cross_entropy", "gelu", 0.0),
    ("res-layer-wise", "tf32", "mse", "relu", 0.3),
    ("res-layer-wise", "bf16", "cross_entropy", "gelu", 0.0),
]
SEED = 0x5EED_0F_0DD


def _case_id(c):
    return "-".join(str(v) for v in c)


def _make_trainer(sizes, mb, n_mu, precision, loss, activation, dropout, Ws, bs, residual=False):
    from shallowspeed_b200.parallel.engine import Trainer

    tr = Trainer(sizes, global_batch_size=mb * n_mu, n_mubatches=n_mu, lr=1.0, precision=precision, loss=loss,
                 activation=activation, dropout=dropout, dropout_seed=SEED, residual=residual, device="cuda:0")
    for i, (W, b) in enumerate(zip(Ws, bs)):
        tr.model.arena.weight_view(i).copy_(W)
        tr.model.arena.bias_view(i).copy_(b[None, :])
    return tr


def _snapshot(tr, L, n_mu, gated):
    eng = tr.engine
    s = {}
    for mu in range(n_mu):
        for l in range(1, L + 1):
            s[("act", mu, l)] = eng.act(mu, l).cpu().clone()
            if gated and l < L:
                s[("gate", mu, l)] = eng.gate(mu, l).cpu().clone()
        for l in range(1, L + 1):
            s[("dz", mu, l)] = eng.dz(mu, l).cpu().clone()
        s[("probs", mu)] = eng.probs(mu).cpu().clone()
    return s


def check_engine_layers(s, model, W0, x, t, n_mu, mb, precision, loss, activation, dropout, W1):
    """Every layer of a planted step from the engine's own buffers ``s`` (``_snapshot``): the forward, the head, the
    dgrads and the update carry the class oracle's classes, and their finite elements lie within the fp64 bounds
    computed with the non-finite operands set to 0.  W0: [out, in + 1] blocks before the step, W1 after it.

    A residual layer adds its input to f(z) * keep * s, and every activated layer of a residual model stores its gate,
    ReLU included; the dgrad multiplies by that gate.  The skip gradient the chain keeps in registers is not modelled:
    a residual dgrad's classes are those of (dz @ W) * gate, and its finite elements are left to the bitwise comparison
    with the clean step (test_engine_step_per_layer's isolation check)."""
    from shallowspeed_b200.ops import functional as F
    from test_gpu_cross_entropy import ce_head_oracle
    from test_gpu_residual import operand_model

    op, rtol = operand_model(precision)
    L = len(W0)
    p = dropout
    res_model = any(lin.residual for lin in model.linears)
    sc = F.dropout_scale(p) if p > 0 else 1.0
    res = {}
    dzs_all, acts_all = [[] for _ in range(L)], [[] for _ in range(L)]
    batch = mb * n_mu
    for mu in range(n_mu):
        # the input stays fp32: on the CPU an fp32 -> fp64 conversion quiets a signalling NaN (0x7F800001 becomes
        # 0x7FC00001), which the tf32 operand model would then read as NaN instead of +Inf
        acts = [x[mu * mb:(mu + 1) * mb]] + [s[("act", mu, l)].double() for l in range(1, L + 1)]
        for l in range(1, L + 1):
            W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
            cz = class_matmul(acts[l - 1], W.T, precision, bias=b)
            a0, w0, b0 = zeroed(acts[l - 1], precision), zeroed(W, precision), zeroed(b)
            a0 = a0 if l > 1 else zeroed(acts[0], precision)
            if l < L:
                lin = model.linears[l - 1]
                keep = F.dropout_mask(p, SEED, lin.dropout[2], 0, mu * mb + torch.arange(mb), W.shape[0]) if p > 0 else None
                (ra, ba), gam, _ = act_fwd_oracle(activation, op(a0), op(w0), b0, keep, sc, rtol)
                fa, fg = F.activation_ref(activation, rep(cz, torch.zeros_like(ra)))
                kf = torch.ones_like(ra) if keep is None else keep.double()
                base = torch.where(cz == FIN, ra, torch.where(kf > 0, fa * sc, 0.0))
                fin = cz == FIN
                if lin.residual:
                    skip = acts[l - 1].double()
                    base = base + skip
                    ra = ra + zeroed(skip)
                    ba = ba * (1.0 + U) + U * ra.abs() + ATOL
                    fin = fin & torch.isfinite(skip)
                want = classes(base)
                assert_classes(acts[l], want, f"mu {mu} act{l}")
                res[f"act{l}"] = max(res.get(f"act{l}", 0.0), finite_excess(acts[l], ra, ba, torch.where(fin, want, NAN_C)))
                if activation != "relu" or res_model:
                    # the gate of a kept element is f'(z) * s (finite for a finite z), of a dropped one +0
                    gw = classes(torch.where(kf > 0, fg * sc, 0.0))
                    assert_classes(s[("gate", mu, l)], gw, f"mu {mu} gate{l}")
            else:
                ref, bound = fwd_oracle(op(a0), op(w0), b0, False, rtol)
                assert_classes(acts[L], torch.where(cz == FIN, classes(ref), cz), f"mu {mu} logits")
                res["logits"] = max(res.get("logits", 0.0), finite_excess(acts[L], ref, bound, cz))
        # the head from the kernel's logits
        oracle = head_oracle if loss == "mse" else ce_head_oracle
        tt = t[mu * mb:(mu + 1) * mb]
        (pr, bp), (gr, bg), _ = oracle(acts[L], tt, batch, HEAD_RTOL)
        for got, ref, bound, what in ((s[("probs", mu)], pr, bp, "probs"), (s[("dz", mu, L)], gr, bg, f"dz{L}")):
            want = classes(ref)
            assert_classes(got, want, f"mu {mu} {what}")
            res[what] = max(res.get(what, 0.0), finite_excess(got, ref, bound, want))
        # dgrads from the kernel's dz and the stored act / gate
        dzs = [None] + [s[("dz", mu, l)].double() for l in range(1, L + 1)]
        for l in range(L, 1, -1):
            W = W0[l - 1][:, :-1]
            cp = class_matmul(dzs[l], W, precision)
            d0, w0 = zeroed(dzs[l], precision), zeroed(W, precision)
            gate = s[("gate", mu, l - 1)].double() if activation != "relu" or res_model else None
            if res_model:
                want = classes(rep(cp, torch.ones(cp.shape, dtype=torch.float64)) * gate)
                assert_classes(dzs[l - 1], want, f"mu {mu} dgrad{l}")
                continue
            ref, bound = act_dgrad_oracle(op(d0), op(w0), activation, acts[l - 1], gate, sc, rtol)
            if activation == "relu":
                on = acts[l - 1] > 0
                want = torch.where(on, torch.where(cp == FIN, classes(ref), cp), torch.zeros_like(cp))
            else:
                want = torch.where(cp == FIN, classes(ref), classes(rep(cp, torch.ones_like(ref)) * gate))
            assert_classes(dzs[l - 1], want, f"mu {mu} dgrad{l}")
            res[f"dgrad{l}"] = max(res.get(f"dgrad{l}", 0.0), finite_excess(dzs[l - 1], ref, bound,
                                                                              torch.where(cp == FIN, want, NAN_C)))
        for l in range(1, L + 1):
            dzs_all[l - 1].append(dzs[l])
            acts_all[l - 1].append(acts[l - 1])
    # the update
    for l in range(1, L + 1):
        dz, a = torch.cat(dzs_all[l - 1]), torch.cat(acts_all[l - 1])
        cg = torch.cat([class_matmul(dz.T, a, precision), class_matmul(dz.T, torch.ones(dz.shape[0], 1), "ieee")], 1)
        w_before = W0[l - 1]
        want = classes(w_before - 1.0 * rep(cg, torch.zeros_like(w_before)))
        assert_classes(W1[l - 1], want, f"update{l}")
        fin = (want == FIN) & torch.isfinite(w_before)
        if precision == "bf16":
            from test_gpu_bf16 import _update_oracle

            ref, bound = _update_oracle(zeroed(dz, "bf16"), zeroed(a, "bf16"), zeroed(w_before), 1.0)
        else:
            ref, bound = rows_update_oracle(zeroed(dz), zeroed(a), zeroed(w_before), 1.0, rtol)
        d = W1[l - 1].double() - w_before
        res[f"upd{l}"] = finite_excess(d, ref, bound, torch.where(fin, FIN, NAN_C).to(torch.int8))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


def _blocks(model):
    return [model.arena.block(i)[:, : k + 1].double().cpu().clone() for i, (_, k) in enumerate(model.arena.blocks)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ENGINE_GRID, ids=_case_id)
def test_engine_step_per_layer(case, monkeypatch):
    """One Trainer step per plant (an input row of the last micro-batch, one hidden weight, a last-layer bias at
    +-Inf), every layer checked from the engine's own buffers; for the input plant every other micro-batch (and, under
    cross-entropy, every other row of the planted one) bitwise the clean step."""
    form, precision, loss, activation, dropout = case
    sizes, mb, n_mu, env = FORMS[form]
    residual = form.startswith("res-")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    L, C, rows = len(sizes) - 1, sizes[-1], mb * n_mu
    gen = _gen("nf-engine", case)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen, activation)
    gated = activation != "relu" or residual

    def run(xx, Ws_, bs_):
        tr = _make_trainer(sizes, mb, n_mu, precision, loss, activation, dropout, Ws_, bs_, residual)
        check_launch_form(form, tr.engine)
        assert residual == any(lin.residual for lin in tr.model.linears)
        W0 = _blocks(tr.model)
        lv = float(tr.step(xx.pin_memory(), t.pin_memory()))
        torch.cuda.synchronize()
        return lv, _snapshot(tr, L, n_mu, gated), W0, _blocks(tr.model), tr.model

    l_clean, s_clean, _, _, _ = run(x, Ws, bs)
    assert math.isfinite(l_clean)
    idx = ENGINE_GRID.index(case)
    vals = [NAN, INF, -INF, LOWNAN_P]
    for plant in PLANTS:
        xx, Ws_, bs_ = x.clone(), [w.clone() for w in Ws], [b.clone() for b in bs]
        mu_p, r = n_mu - 1, mb - 1
        if plant == "input":
            K0 = sizes[0]
            put(xx, (n_mu - 1) * mb + r, min(31, K0 - 1), vals[idx % 4])
            put(xx, (n_mu - 1) * mb + r, K0 - 1, vals[(idx + 1) % 4])
            # k-block 2: the helper's half of the k-split first layer (k-blocks kb % 4 in {2, 3})
            put(xx, (n_mu - 1) * mb + r, min(95, K0 - 1), vals[(idx + 2) % 4])
            if precision == "bf16":
                xx[(n_mu - 1) * mb + r, min(33, K0 - 1)] = BIG
        elif plant == "weight":
            lw = min(1, L - 2)                               # a hidden layer's weight (layer 2 where there is one)
            put(Ws_[lw], Ws_[lw].shape[0] - 1, min(32, Ws_[lw].shape[1] - 1), vals[idx % 3])
        else:
            bs_[-1][0] = INF if idx % 2 == 0 else -INF
        lv, s, W0, W1, model = run(xx, Ws_, bs_)
        res = check_engine_layers(s, model, W0, xx, t, n_mu, mb, precision, loss, activation, dropout, W1)
        # the loss: the sum of the heads' losses, NaN in the VM wherever any term is
        from test_gpu_cross_entropy import ce_head_oracle

        oracle = head_oracle if loss == "mse" else ce_head_oracle
        lref = sum(oracle(s[("act", mu, L)].double(), t[mu * mb:(mu + 1) * mb], rows, HEAD_RTOL)[2][0] for mu in range(n_mu))
        assert classes(torch.tensor([lv])) == classes(torch.tensor([lref])), (plant, lv, lref)
        if plant == "input":
            # isolation: the other micro-batches, and under cross-entropy (row-wise throughout) the other rows
            for key, v in s.items():
                other = torch.ones(v.shape, dtype=torch.bool)
                if key[1] == mu_p:
                    if loss != "cross_entropy":
                        continue
                    other[r] = False
                msg = bitwise_mismatch(v, s_clean[key], other)
                assert msg is None, (plant, key, msg)
        print(f"\n[nonfinite] {_case_id(case)} {plant}: loss {lv} " + " ".join(f"{k}={v:.2g}" for k, v in res.items()))


# ---------------------------------------------------------------- the data-parallel replay
# test_gpu_dp_replay's harness: replica 0 of a dp = 2 group, its peer replayed from memory.  The peer's partials carry
# NaN / +-Inf at elements replica 0 owns, bias column included; under LL the peer's phase-C weights (the rows it owns,
# which replica 0 copies) carry them too.  A clean replay with the same data has those entries at 0 (the partials) or
# at their clean values (the copied weights).
DP_CASES = {                                            # name -> (model, protocol, env, mb_rows, n_mu)
    "ll-ref": ("REF", "ll", {"SSB_DP_GATE": "1"}, 16, 4),
    "flag-wide-one-shot": ("WIDE", "one-shot", {"SSB_DP_LL": "0", "SSB_DP_ONE_SHOT": "1"}, 32, 2),
    "flag-wide-two-shot": ("WIDE", "two-shot", {"SSB_DP_LL": "0", "SSB_DP_TWO_SHOT": "1"}, 32, 2),
}


def _dp_plants(owned, k, mine):
    """(row, col, value) plants of one layer's [out, in + 1] block, at elements that are ``mine`` (owned by replica 0)
    or not: the first and the last such element, one in column 32 and one in the bias column (in = k)."""
    sel = owned if mine else ~owned
    pos = sel.nonzero()
    if pos.numel() == 0:
        return []
    out = [(int(pos[0, 0]), int(pos[0, 1]), NAN), (int(pos[-1, 0]), int(pos[-1, 1]), -INF)]
    for col, v in ((min(32, k - 1), INF), (k, INF if mine else NAN)):
        rows = sel[:, col].nonzero()
        if rows.numel():
            out.append((int(rows[rows.numel() // 2, 0]), col, v))
    return out


def _dp_replay(sizes, protocol, env, mb, n_mu, planted, monkeypatch):
    """One step of replica 0 of a dp = 2 group: (W1 blocks, own partials, the peer's buffers, setup, data, epoch)."""
    import gc

    from shallowspeed_b200.pipe import NaiveParallelSchedule
    from test_gpu_chain import _gather, _poison
    from test_gpu_dp_replay import LR, _build_replica, _grad_scale, dp_peer_data, dp_prefill, dp_setup
    from test_gpu_gemm import grad_oracle, rtol_for

    dp, rank = 2, 0
    for kk, v in env.items():
        monkeypatch.setenv(kk, v)
    L, rows = len(sizes) - 1, mb * n_mu
    w, model, ctxs = _build_replica(sizes, dp, rank, mb, n_mu, "fp32", False, monkeypatch)
    sched = NaiveParallelSchedule(n_mu, 1, 0)
    eng = w.engine_for(sched)
    arena = model.arena
    gen = _gen("nf-dp", tuple(sizes), protocol)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        arena.weight_view(i).copy_(W)
        arena.bias_view(i).copy_(b[None, :])
    protos = list(eng.layer_protocols())
    d = dp_setup(ctxs, rank, protocol, sizes, env, arena, protos)
    _poison(eng, model, sizes, rows, True)
    epoch = int(d["me"].epoch[0].item()) + 1
    W0 = [arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(arena.blocks)]
    scale = _grad_scale(sizes, W0, x, t, n_mu, model.batch_size)
    P, Wc = dp_peer_data(d, gen, arena.blocks, scale, W0, LR)
    plants = []
    for i, (_, k) in enumerate(arena.blocks):
        pa = _dp_plants(d["owned"][i], k, True)
        pc = _dp_plants(d["owned"][i], k, False) if d["ll"] else []
        plants.append((pa, pc))
        for r_, c_, v in pa:
            P[1][i][r_, c_] = v if planted else 0.0
        for r_, c_, v in pc:
            if planted:
                Wc[1][i][r_, c_] = v
    torch.cuda.synchronize()
    dp_prefill(d, P, Wc, epoch)
    torch.cuda.synchronize()
    w.step_from(sched, x.pin_memory(), t.pin_memory())
    eng.synchronize()
    torch.cuda.synchronize()
    act = [x.double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L)]
    dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
    own = [grad_oracle(dz[i + 1], act[i], rtol_for("fp32", rows))[0] for i in range(L)]
    W1 = [arena.block(i)[:, : k + 1].cpu().clone() for i, (_, k) in enumerate(arena.blocks)]
    peer = d["bufs"][1]
    bufs = {name: getattr(peer, name).cpu().clone() for name in ("W", "stage", "arrive", "done", "llA", "llC")
            if getattr(peer, name) is not None}
    out = dict(W0=W0, W1=W1, own=own, P=P, Wc=Wc, bufs=bufs, owners=[o.clone() for o in d["owners"]],
               owned=[o.clone() for o in d["owned"]], plants=plants, epoch=epoch, ll=d["ll"], protos=protos,
               offsets=[int(o) for o in arena.offsets], lds=[int(v) for v in arena.lds], blocks=list(arena.blocks),
               tiles=d.get("tiles"))
    eng.synchronize()
    del eng, w, d
    gc.collect()
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(DP_CASES))
def test_dp_replay_carries_the_peer_classes(case, monkeypatch):
    """The owned updates carry the class of W0 - lr * (own + peer) with the peer's non-finite partials, bias column
    included; under LL the copied rows carry the peer's non-finite phase-C bits and the phase-C lines sent to the peer
    carry the new weights bit for bit; every other weight and every outbound line, tile and flag is bitwise the clean
    replay."""
    import test_gpu_dp_replay as R

    name, protocol, env, mb, n_mu = DP_CASES[case]
    sizes = getattr(R, name)
    clean = _dp_replay(sizes, protocol, env, mb, n_mu, False, monkeypatch)
    got = _dp_replay(sizes, protocol, env, mb, n_mu, True, monkeypatch)
    assert (got["protos"] == [R._C().DP_PROTO_LL] * len(got["blocks"])) == got["ll"], got["protos"]
    n_nf = 0
    for i, (o, k) in enumerate(got["blocks"]):
        owned, owners = got["owned"][i], got["owners"][i]
        tot = got["own"][i] + got["P"][1][i].double()
        want = classes(got["W0"][i] - R.LR * tot)
        if got["ll"]:
            peer_rows = owners == 1
            want[peer_rows] = classes(got["Wc"][1][i].double())[peer_rows]
        else:
            want[~owned] = FIN
        assert_classes(got["W1"][i], want, f"layer {i + 1}: weights")
        n_nf += int((want != FIN).sum())
        msg = bitwise_mismatch(got["W1"][i], clean["W1"][i], want == FIN)
        assert msg is None, f"layer {i + 1}: finite weights: {msg}"
        if got["ll"]:
            pm = owners == 1
            assert torch.equal(got["W1"][i][pm].view(torch.int32), got["Wc"][1][i][pm].view(torch.int32)), \
                f"layer {i + 1}: copied rows differ from the peer's phase-C lines"
    assert n_nf >= 2 * len(got["blocks"]), "the plants reached too few weights"
    every = lambda t: torch.ones(t.shape, dtype=torch.bool)
    if got["ll"]:
        # phase A (my partials to the peer) bitwise the clean replay; phase C (my new rows) bit for bit my weights
        msg = bitwise_mismatch(got["bufs"]["llA"], clean["bufs"]["llA"], every(got["bufs"]["llA"]))
        assert msg is None, f"phase-A lines: {msg}"
        mine = R.ll_messages(got["tiles"], 2, 0, got["epoch"] & 1)
        R.check_lines(got["bufs"]["llC"], mine[("C", 1)], got["W1"], None, got["epoch"], "phase C to 1")
        R.check_only(got["bufs"]["llC"], mine[("C", 1)], got["epoch"], "llC of 1")
        zc, cc = got["bufs"]["llC"], clean["bufs"]["llC"]
        diff = (zc != cc).any(1)
        vals = torch.cat([zc[diff, 0], zc[diff, 2]]).view(torch.float32)
        assert bool((~torch.isfinite(vals)).any()), "no non-finite weight reached a phase-C line"
    else:
        for nm in ("stage", "arrive", "done"):
            msg = bitwise_mismatch(got["bufs"][nm], clean["bufs"][nm], every(got["bufs"][nm]))
            assert msg is None, f"{nm} of the peer: {msg}"
        # two-shot tiles I own are published into the peer's weights: my new weights, bit for bit, non-finite included
        Wp, Wpc = got["bufs"]["W"], clean["bufs"]["W"]
        published = 0
        for i, (o, k) in enumerate(got["blocks"]):
            off, ld = got["offsets"][i], got["lds"][i]
            blk, blkc = Wp[off: off + o * ld].view(o, ld)[:, : k + 1], Wpc[off: off + o * ld].view(o, ld)[:, : k + 1]
            pm = got["owners"][i] == 0
            if got["protos"][i] == R._C().DP_PROTO_TWO_SHOT:
                assert torch.equal(blk[pm].view(torch.int32), got["W1"][i][pm].view(torch.int32)), f"layer {i + 1}"
                published += int((~torch.isfinite(blk[pm])).sum())
            assert torch.equal(blk[~pm].view(torch.int32), blkc[~pm].view(torch.int32)), f"layer {i + 1}: peer rows"
        if protocol == "two-shot":
            assert published > 0, "no non-finite weight was published to the peer"


# ---------------------------------------------------------------- engine level: the VM, inference, stale state
VM_SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
# every launch form: name -> (sizes, env); the chain forms at 32-row micro-batches
VM_FORMS = {
    "cluster-c4": (VM_SIZES, {}),
    "cluster-c2": ([100] + [40] * 15 + [10], {}),
    "one-cta": ([33, 32, 31, 17], {}),
    "ksplit-first": ([160, 128, 97, 33, 10], {}),
    "per-micro-batch": (VM_SIZES, {"SSB_NO_COALESCE": "1"}),
    "layer-wise": (VM_SIZES, {"SSB_NO_CHAIN": "1"}),
    "splitk-wide": ([784, 512, 256, 10], {"SSB_SPLITK": "2"}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(VM_FORMS))
def test_nan_hidden_weight_gives_a_nan_loss_like_the_vm(form, monkeypatch):
    """A NaN in one hidden weight: the loss of step 0 is NaN, as in the Python VM, and after the step the weights are
    non-finite exactly where the VM's are, in every launch form."""
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule, Worker

    sizes, env = VM_FORMS[form]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    x, y = synthetic_mnist(n=128, n_features=sizes[0], n_classes=sizes[-1])
    out = {}
    for dev in ("cpu", "cuda"):
        model = MLP(sizes, 0, 1, 128).to(dev)
        params = list(model.parameters())
        with torch.no_grad():
            params[2].data[5, 17] = NAN                     # layer 2's weight
        opt = SGD(model.parameters(), 0.05, arena=model.arena)
        ds = Dataset(None, 128, 32, device=dev)
        ds.local_batch_size = 128
        ds.from_arrays(x, y)
        w = Worker(None, None, model, ds, opt) if dev == "cpu" else NativeWorker(None, None, model, ds, opt)
        w.execute(GPipeSchedule(4, 1, 0), 0)
        if dev == "cuda":
            check_launch_form(form, w.engine_for(GPipeSchedule(4, 1, 0)))
        loss = w.batch_loss()
        if dev == "cuda":
            w.sync_to_model()
        out[dev] = (loss, [p.data.detach().cpu().clone() for p in model.parameters()])
    assert math.isnan(out["cpu"][0]), "the VM's loss is NaN"
    assert math.isnan(out["cuda"][0]), f"{form}: the engine reports a finite loss {out['cuda'][0]} for a NaN weight"
    for i, (pc, pg) in enumerate(zip(out["cpu"][1], out["cuda"][1])):
        assert torch.equal(torch.isfinite(pc), torch.isfinite(pg)), f"{form}: parameter {i}: non-finite elsewhere than the VM's"
        assert torch.equal(classes(pc), classes(pg)), f"{form}: parameter {i}: other classes than the VM's"


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["coalesced", "per-micro-batch", "layer-wise", "splitk-wide"])
def test_no_state_carries_a_nan_into_the_next_launch(form, monkeypatch):
    """Inference of a NaN input, then of a clean one: the second call is bitwise what a fresh engine returns (no split-K
    workspace, cluster scratch or loss slot keeps a value from the first).  Training the same way: a step whose input
    holds NaN, then the weights restored and a clean step, against a fresh engine's clean step."""
    from shallowspeed_b200.pipe import InferenceSchedule

    env = {"coalesced": {}, "per-micro-batch": {"SSB_NO_COALESCE": "1"}, "layer-wise": {"SSB_NO_CHAIN": "1"},
           "splitk-wide": {"SSB_SPLITK": "2"}}[form]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sizes = [784, 512, 256, 10] if form == "splitk-wide" else [784, 128, 97, 33, 10]
    mb, n_mu = 40, 3
    rows = mb * n_mu
    gen = _gen("nf-stale", form)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, 10, (rows,), generator=gen), 10).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen)
    xn = x.clone()
    xn[::7, 5] = NAN
    xn[3, 100] = INF
    sched = InferenceSchedule(n_mu, 1, 0)

    def infer(tr, xx):
        eng = tr.worker.engine_for(sched)
        tr.worker.step_from(sched, xx.pin_memory(), t.pin_memory())
        eng.synchronize()
        torch.cuda.synchronize()
        return [eng.probs(mu).cpu().clone() for mu in range(n_mu)], [eng.act(mu, len(sizes) - 1).cpu().clone() for mu in range(n_mu)]

    used = _make_trainer(sizes, mb, n_mu, "fp32", "mse", "relu", 0.0, Ws, bs)
    first = infer(used, xn)
    assert all(bool(p.isnan().any()) for p in first[0][:1] + first[0][-1:])
    second = infer(used, x)
    fresh = infer(_make_trainer(sizes, mb, n_mu, "fp32", "mse", "relu", 0.0, Ws, bs), x)
    for a, b in zip(second[0] + second[1], fresh[0] + fresh[1]):
        assert bitwise_mismatch(a, b, torch.ones(a.shape, dtype=torch.bool)) is None, f"{form}: inference kept state"
    # training: a NaN step, the weights put back, then a clean step
    tr = _make_trainer(sizes, mb, n_mu, "fp32", "mse", "relu", 0.0, Ws, bs)
    l_nan = float(tr.step(xn.pin_memory(), t.pin_memory()))
    assert math.isnan(l_nan)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        tr.model.arena.weight_view(i).copy_(W)
        tr.model.arena.bias_view(i).copy_(b[None, :])
    l2 = float(tr.step(x.pin_memory(), t.pin_memory()))
    ref = _make_trainer(sizes, mb, n_mu, "fp32", "mse", "relu", 0.0, Ws, bs)
    l_ref = float(ref.step(x.pin_memory(), t.pin_memory()))
    torch.cuda.synchronize()
    assert l2 == l_ref, (l2, l_ref)
    for a, b in zip(_blocks(tr.model), _blocks(ref.model)):
        assert torch.equal(a.float().view(torch.int32), b.float().view(torch.int32)), f"{form}: training kept state"


@pytest.mark.gpu
def test_relu_kernels_keep_nan_and_zero_the_rest():
    """The stand-alone ReLU (relu_fwd_kernel) and the mask kernel on every class: NaN stays, -Inf / -0 / negatives
    give +0, +Inf and positives pass; the mask selects, so a masked-off NaN or Inf gradient is +0, as relu_grad_ref."""
    from shallowspeed_b200.ops import functional as F

    K = _K()
    z = torch.tensor([[NAN, INF, -INF, -0.0, 0.0, -1.5, 2.5, _lownan(LOWNAN_N)[0].item()]])
    y = K.relu(z.cuda()).cpu()
    want = F.relu_ref(z)
    assert torch.equal(classes(y), classes(want))
    fin = torch.isfinite(want)
    want = torch.where(z > 0, z, 0.0)                      # -0 gives +0 (relu_ref's clamp_min keeps -0)
    assert torch.equal(y[fin].view(torch.int32), want[fin].view(torch.int32)), y
    g = torch.tensor([[NAN, INF, -INF, NAN, 1.0, -2.0, 3.0, NAN]])
    got = K.relu_grad(g.cuda(), z.cuda() > 0).cpu()
    ref = F.relu_grad_ref(g, z > 0)
    assert torch.equal(classes(got), classes(ref))
    assert torch.equal(got[torch.isfinite(ref)].view(torch.int32), ref[torch.isfinite(ref)].view(torch.int32))
    assert bool((ref[~(z > 0)].view(torch.int32) == 0).all())


# ================================================================================================== CPU side
@pytest.mark.parametrize("precision", ["ieee", "fp32", "tf32", "bf16"])
def test_class_oracle_matches_elementwise_products(precision):
    """class_matmul against numpy: every term a[i, k] * b[k, j] formed elementwise in fp64 (on the precision's operands,
    fp32 with an infinite operand made NaN), then summed without a BLAS."""
    g = np.random.default_rng(zlib.crc32(precision.encode()))
    for trial in range(30):
        n, k, m = g.integers(1, 7, size=3)
        A = g.standard_normal((n, k)).astype(np.float32)
        B = g.standard_normal((k, m)).astype(np.float32)
        A[g.random((n, k)) < 0.2] = 0.0
        B[g.random((k, m)) < 0.2] = 0.0
        specials = np.array([np.nan, np.inf, -np.inf, _lownan(LOWNAN_P)[0].item(), _lownan(LOWNAN_N)[0].item(), BIG, -BIG],
                            dtype=np.float32)
        for M in (A, B):
            sel = g.random(M.shape) < 0.15
            M[sel] = g.choice(specials, size=int(sel.sum()))
        bias = g.standard_normal(m).astype(np.float32)
        if trial % 3 == 0:
            bias[g.integers(0, m)] = g.choice([np.nan, np.inf, -np.inf])
        oa = operand_class(torch.from_numpy(A), "ieee" if precision == "fp32" else precision).numpy()
        ob = operand_class(torch.from_numpy(B), "ieee" if precision == "fp32" else precision).numpy()
        with np.errstate(invalid="ignore", over="ignore"):
            terms = oa[:, :, None] * ob[None, :, :]                         # [n, k, m]
            if precision == "fp32":
                bad = ~np.isfinite(oa)[:, :, None] | ~np.isfinite(ob)[None, :, :]
                terms = np.where(bad, np.nan, terms)
            # sum the non-finite parts exactly: finite terms replaced by 0 cannot change the class (no overflow here)
            nf = np.where(np.isfinite(terms), 0.0, terms)
            want = nf.sum(axis=1) + np.where(np.isfinite(bias), 0.0, bias).astype(np.float64)[None, :]
        got = class_matmul(torch.from_numpy(A), torch.from_numpy(B), precision, bias=torch.from_numpy(bias))
        assert torch.equal(got, classes(torch.from_numpy(want))), (precision, trial, A, B, bias)


def test_class_oracle_hand_cases():
    A = torch.tensor([[INF, 1.0], [INF, -1.0], [NAN, 0.0], [INF, 0.0], [0.0, 2.0]])
    B = torch.tensor([[0.0, 1.0], [1.0, 1.0]])
    c = class_matmul(A, B, "ieee")
    assert c.tolist() == [[NAN_C, PINF], [NAN_C, PINF], [NAN_C, NAN_C], [NAN_C, PINF], [FIN, FIN]]
    c = class_matmul(torch.tensor([[INF, INF]]), torch.tensor([[1.0], [-1.0]]), "tf32")
    assert c.tolist() == [[NAN_C]]                                   # a +Inf and a -Inf term
    lown = _lownan(LOWNAN_P)
    assert class_matmul(lown.view(1, 1), torch.tensor([[2.0]]), "tf32").tolist() == [[PINF]]
    assert class_matmul(lown.view(1, 1), torch.tensor([[2.0]]), "bf16").tolist() == [[NAN_C]]
    assert class_matmul(torch.tensor([[INF]]), torch.tensor([[2.0]]), "fp32").tolist() == [[NAN_C]]
    assert class_matmul(torch.tensor([[BIG]]), torch.tensor([[-1.0]]), "bf16").tolist() == [[NINF]]
    assert class_matmul(torch.tensor([[BIG]]), torch.tensor([[-1.0]]), "tf32").tolist() == [[FIN]]


def test_engine_grid_reaches_every_branch():
    forms = {c[0] for c in ENGINE_GRID}
    assert forms == set(FORMS)
    for col, values in ((1, PRECISIONS), (2, ["mse", "cross_entropy"]), (3, ["relu", "gelu"]), (4, [0.0, 0.3])):
        assert {c[col] for c in ENGINE_GRID} == set(values)
    for prec in PRECISIONS:
        assert {c[2] for c in ENGINE_GRID if c[1] == prec} == {"mse", "cross_entropy"}
    # the cluster sizes and the k-split the forms are named for
    from shallowspeed_b200 import _C

    layers = lambda s: list(zip(s[:-1], s[1:]))
    assert _C.chain_cluster_size(layers(FORMS["cluster-c4"][0]), True, True, True, True, False, False) == 4
    assert _C.chain_cluster_size(layers(FORMS["cluster-c2"][0]), True, True, True, True, False, False) == 2
    assert _C.chain_cluster_size(layers(FORMS["one-cta"][0]), True, True, True, True, False, False) == 1
    assert _C.chain_cluster_size(layers(FORMS["ksplit-first"][0]), True, True, True, True, False, False) > 1
    assert (FORMS["ksplit-first"][0][0] + 31) // 32 > 4                # more than 4 k-blocks in layer 1: the k-split
    assert max(FORMS["splitk-wide"][0][1:-1]) > 128                    # wider than the chain: layer-wise, split-K forced


# ---------------------------------------------------------------- the checks reject emulated faults
def _emulated_fwd(x, W, b, relu):
    """A kernel's FWD emulated on the CPU with the class oracle's semantics: relu(x @ W.T + b) per element."""
    terms = x.double()[:, None, :] * W.double()[None, :, :]
    z = terms.sum(-1) + b.double()
    return relu(z).float()


def test_checks_reject_emulated_faults():
    x = torch.randn(5, 40)
    W = torch.randn(7, 40)
    b = torch.randn(7)
    x[1, 3] = NAN
    x[2, 31] = -INF
    W[4, 32] = 0.0
    cz = class_matmul(x, W.T, "ieee", bias=b)
    want = relu_class(cz)
    good = _emulated_fwd(x, W, b, lambda z: torch.where(z <= 0, torch.zeros_like(z), z))
    assert class_mismatch(good, want) is None
    fmaxf = _emulated_fwd(x, W, b, lambda z: torch.fmax(z, torch.zeros_like(z)))         # NaN read as 0
    assert class_mismatch(fmaxf, want) is not None
    # a mask applied by multiplying: NaN * 0 = NaN where the select gives +0
    g = torch.tensor([[NAN, 1.0, INF], [2.0, -INF, 3.0]])
    act = torch.tensor([[0.0, 1.0, -0.0], [1.0, 0.0, 2.0]])
    from shallowspeed_b200.ops import functional as F

    want = classes(F.relu_grad_ref(g, act > 0))
    assert class_mismatch(torch.where(act > 0, g, 0.0), want) is None
    assert class_mismatch(g * (act > 0), want) is not None
    # a NaN-blind global max: only the NaN row becomes NaN
    z = torch.randn(6, 10)
    z[2, 3] = NAN
    t = torch.nn.functional.one_hot(torch.arange(6) % 10, 10).float()
    (p, _), _, _ = head_oracle(z, t, 6, HEAD_RTOL)
    m = z.nan_to_num(nan=-INF).max()                                    # fmaxf over the batch skips the NaN
    e = torch.exp(z.double() - m.double())
    blind = e / (e.sum(1, keepdim=True) + 1e-7)
    assert class_mismatch(F.softmax_ref(z.double()), classes(p)) is None
    assert class_mismatch(blind, classes(p)) is not None
    # a NaN row leaking into the next micro-batch, and a stale NaN in the next launch: the bitwise isolation checks
    clean = torch.randn(2, 8, 4)
    planted = clean.clone()
    planted[1, 3, 0] = NAN
    leak = planted.clone()
    leak[0, 0, 1] = NAN
    mb0 = torch.ones(8, 4, dtype=torch.bool)
    assert bitwise_mismatch(planted[0], clean[0], mb0) is None
    assert bitwise_mismatch(leak[0], clean[0], mb0) is not None
    fresh = torch.randn(8, 4)
    stale = fresh.clone()
    stale[5, 2] = NAN
    assert bitwise_mismatch(fresh.clone(), fresh, mb0) is None
    assert bitwise_mismatch(stale, fresh, mb0) is not None
    # and the class check sees a stale NaN where the oracle says finite
    assert class_mismatch(stale, classes(fresh)) is not None
