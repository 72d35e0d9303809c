"""The layer-wise tensor-core GEMMs (``csrc/kernels/tc_gemm.cu``) against a per-element fp64 oracle at every tile edge:
FWD, DGRAD and WGRAD stand-alone, split-K, the fused SGD epilogue with and without momentum / weight decay, and the
engine at wide shapes, where every layer runs on these kernels.

The bounds are test_gpu_chain's, ``|got - ref| <= rtol * (|A| @ |B|) + ATOL``, with three additions:
* K > 4096: one more fp32 rounding per 32-wide k-block sum and per split partial, ``(ceil(K/32) + splits) * 2^-24``
  (``rtol_for``); RTOL's own derivation covers K <= 4096.
* the bias gradient is an fp32 sum over the rows in order, in both precisions: one rounding per row (``grad_oracle``).
* the stateful SGD rule carries the gradient's bound through each of its steps (``sgd_oracle``).

Worst err / bound, measured on an H100 80GB HBM3 (700 W): fp32 0.05 for FWD / DGRAD, 0.01 for split-K, 0.47 for WGRAD
and 0.5 for the engine's updates (the fp32 rounding of the stored weight, at most 2^-24 of it against 2^-23 in the
bound); tf32 0.97 for WGRAD and 0.93 for the fused update with one row, 0.96 for the engine's updates and 0.91 for its
10-term dgrad.  These come near 1 by the bound's own derivation: with one product per element (or few non-zero ones,
behind a ReLU) nothing averages out, and two operands truncated to 10 mantissa bits reach almost 2^-9 of the product.

The residual form (``tc_gemm_res_kernel``) runs through ``ops.cuda``'s ``residual=`` / ``skip=`` / ``gpre=`` at every
tile edge and split count, in fp32, tf32 and bf16, with a nil feature where the result is the skip up to one rounding.

Every input's padding columns hold NaN and every output's padding a finite sentinel, so a kernel that reads or writes
past the end of a row fails.  The CPU tests at the end check that the grid reaches every branch of the host planner,
and that the oracles reject a set of plausible kernel faults while they accept the exact result and an fp32 one.
"""
import math
import re
import zlib

import pytest
import torch

from test_gpu_chain import (ATOL, FAR_BIASES, FP32_ULP, HEAD_RTOL, LR, RTOL, _gather, _init_weights, _n_mu, _poison,
                            _selftest_data, act_dgrad_oracle, act_fwd_oracle, dgrad_oracle, excess, fwd_oracle,
                            head_oracle, update_oracle)

U = 2.0**-24                  # unit roundoff of fp32
SENTINEL = -1234.5            # output padding: finite and non-zero, so x + (-0.0) keeps its bits
NAN = float("nan")
MU, WD = 0.9, 1e-2
SGD_LR = 0.25
WORST = {}                    # (kernel, precision) -> worst err / bound of the session, printed at the end (-s)


def _note(key, res, what):
    v = max(res.values()) if res else 0.0
    if v > WORST.get(key, (0.0, ""))[0] or key not in WORST:
        WORST[key] = (v, what)
    print(f"\n[gemm] {key[0]} {key[1]} {what}: max err/bound {v:.3g} ("
          + " ".join(f"{k}={x:.2g}" for k, x in res.items()) + ")")
    bad = {k: x for k, x in res.items() if not x <= 1.0}
    assert not bad, (what, bad)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for (kernel, precision), (v, what) in sorted(WORST.items()):
        print(f"[gemm] worst err/bound {kernel:>12} {precision}: {v:.3g} at {what}")


def rtol_for(precision, k, splits=1):
    """RTOL, plus one fp32 rounding per k-block sum and per split partial for K > 4096 (RTOL's derivation stops there)."""
    r = RTOL[precision]
    if k > 4096:
        r += (math.ceil(k / 32) + splits) * U
    return r


def grad_oracle(dz, x, rtol):
    """The [out, in + 1] gradient block ``[dz.T @ x | colsum(dz)]`` in fp64 and its bound.  The bias column is summed
    over the rows in order in fp32 (no TF32 in either precision): one rounding per row, on top of rtol."""
    dz, x = dz.double(), x.double()
    g = torch.cat([dz.T @ x, dz.sum(0)[:, None]], dim=1)
    mag = torch.cat([dz.abs().T @ x.abs(), dz.abs().sum(0)[:, None]], dim=1)
    bound = rtol * mag + ATOL
    bound[:, -1] += dz.shape[0] * U * mag[:, -1]
    return g, bound


def sgd_oracle(g, g_bound, W0, V0, lr, mu, wd, nesterov):
    """One step of the stateful rule (torch.optim.SGD, dampening 0) in fp64, from a gradient and its bound:

        g' = g + wd * w ;  v = mu * v + g' ;  d = nesterov ? g' + mu * v : v ;  w -= lr * d

    Each step carries the bound of its operands (rtol * mag of the GEMM) and adds one fp32 rounding per operation,
    FP32_ULP of the magnitude of its product and its result (fp32 mu, wd and lr are roundings of the same size).
    Returns (W1, bound, V1, bound)."""
    W0, V0 = W0.double(), V0.double()
    gp = g + wd * W0
    e_gp = g_bound + FP32_ULP * (wd * W0.abs() + gp.abs())
    v = mu * V0 + gp
    e_v = e_gp + FP32_ULP * (mu * V0.abs() + v.abs())
    if nesterov:
        d = gp + mu * v
        e_d = e_gp + mu * e_v + FP32_ULP * (mu * v.abs() + d.abs())
    else:
        d, e_d = v, e_v
    W1 = W0 - lr * d
    return W1, lr * e_d + FP32_ULP * (lr * d.abs() + W1.abs()), v, e_v


def _K():
    from shallowspeed_b200.ops import cuda as K

    return K


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _ld(cols, extra=4):
    return (cols + 3) // 4 * 4 + extra


def _pitched(rows, cols, gen, scale=1.0, extra=4, fill=NAN):
    """(buffer, view): a [rows, cols] view of a [rows, round_up(cols, 4) + extra] CUDA buffer with random values and
    ``fill`` in the padding.  The view is TMA-legal, so ``as_tma`` hands the kernels this very memory."""
    buf = torch.full((rows, _ld(cols, extra)), fill)
    buf[:, :cols] = torch.randn(rows, cols, generator=gen) * scale
    buf = buf.cuda()
    view = buf[:, :cols]
    assert _K().tma_ready(view)
    return buf, view


def _out(rows, cols, extra=4):
    buf = torch.full((rows, _ld(cols, extra)), SENTINEL, device="cuda")
    return buf, buf[:, :cols]


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _mask_values(rows, cols, gen):
    """A ReLU mask with exact 0.0, -0.0 and negatives, all of which mean 'off'."""
    m = torch.randn(rows, cols, generator=gen)
    m.view(-1)[0::5] = 0.0
    m.view(-1)[1::5] = -0.0
    return m


# ================================================================================================== FWD / DGRAD
# (rows, M, K): FWD writes [rows, M] from K inputs, DGRAD [rows, M] from K outputs.  rows picks block_n (16 / 32 / 48 /
# 64) and the N tiles, M the 128-row M tiles, K the k-blocks and the ring (stages = min(6, k-blocks)).
GRID = [
    (1, 129, 7),          # K below one k-block; block_n 16; 2 M tiles, the last ragged
    (15, 300, 32),        # one full k-block
    (16, 64, 33),         # two k-blocks, the second 1 wide
    (17, 1000, 65),       # block_n 32; 3 stages
    (33, 129, 100),       # block_n 48; 4 stages
    (48, 33, 150),        # 5 stages
    (63, 300, 777),       # block_n 64 with one ragged N tile; many ring wraps from here on
    (64, 129, 4096),
    (65, 1000, 200),      # 2 N tiles, the last 1 row
    (100, 300, 4096),
    (129, 129, 8192),     # K > 4096: rtol_for's extra term
    (300, 1000, 777),     # 5 N tiles x 8 M tiles, both ragged
    (300, 16, 31),
]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("rows,m,k", GRID)
def test_fwd_per_element(rows, m, k, precision):
    K = _K()
    gen = _gen("fwd", rows, m, k)
    _, x = _pitched(rows, k, gen)
    wbuf, _ = _pitched(m, k + 1, gen, scale=1.0 / math.sqrt(k))      # the arena block: W | bias column | NaN
    wbuf[:, k] = torch.randn(m, generator=gen).cuda() * 0.5
    W, b = wbuf[:, :k], wbuf[:, k]
    xc, Wc, bc = x.cpu(), W.cpu(), b.cpu()
    rtol = rtol_for(precision, k)
    res = {}
    for relu in (False, True):
        for bias in (None, b):
            ybuf, y = _out(rows, m)
            K.linear_fwd(x, W, bias, relu=relu, out=y, precision=precision)
            torch.cuda.synchronize()
            ref, bound = fwd_oracle(xc, Wc, bc if bias is not None else torch.zeros(m), relu, rtol)
            res[f"relu{int(relu)}bias{int(bias is not None)}"] = excess(y, ref, bound)
            assert bool((ybuf[:, m:] == SENTINEL).all()), "FWD wrote into the output's padding"
    _note(("fwd", precision), res, f"rows={rows} m={m} k={k}")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("rows,m,k", GRID)
def test_dgrad_per_element(rows, m, k, precision):
    K = _K()
    gen = _gen("dgrad", rows, m, k)
    _, dz = _pitched(rows, k, gen)
    _, W = _pitched(k, m, gen, scale=1.0 / math.sqrt(k))
    mbuf = torch.full((rows, _ld(m, 8)), NAN)                        # a pitch unlike dX's
    mbuf[:, :m] = _mask_values(rows, m, gen)
    mask = mbuf.cuda()[:, :m]
    dzc, Wc, mc = dz.cpu(), W.cpu(), mask.cpu()
    rtol = rtol_for(precision, k)
    res = {}
    for use_mask in (False, True):
        dxbuf, dx = _out(rows, m)
        assert dx.stride(0) != mask.stride(0)
        K.linear_dgrad(dz, W, mask=mask if use_mask else None, out=dx, precision=precision)
        torch.cuda.synchronize()
        ref, bound = dgrad_oracle(dzc, Wc, mc if use_mask else torch.ones(rows, m), rtol)
        res[f"mask{int(use_mask)}"] = excess(dx, ref, bound)
        assert bool((dxbuf[:, m:] == SENTINEL).all()), "DGRAD wrote into the output's padding"
    _note(("dgrad", precision), res, f"rows={rows} m={m} k={k}")


# ---------------------------------------------------------------- the activated and dropout variants
# every forward variant gemm_configure registers: ReLU + dropout (tc_gemm_drop_kernel) and each smooth kind with and
# without dropout (tc_gemm_gate_kernel); the launch's rows are samples (row_base + n) * dp + rank of the masks
FWD_VARIANTS = [("relu", True)] + [(k, d) for k in ("gelu", "silu", "tanh") for d in (False, True)]
DROP = (0.3, 0x1234_5678_9ABC_DEF0, 6, 9, 5, 3, 2)            # p, seed, layer, step, row_base, dp, rank


def _variant(kind, drop):
    return f"{kind}{'+drop' if drop else ''}"


def _keep(rows, m):
    from shallowspeed_b200.ops import functional as F

    p, seed, layer, step, row_base, dp, rank = DROP
    return F.dropout_mask(p, seed, layer, step, (row_base + torch.arange(rows)) * dp + rank, m), F.dropout_scale(p)


def _fwd_inputs(tag, rows, m, k):
    """x, the arena block's W and bias (features 0..3 with FAR_BIASES: the tails of f and f')."""
    gen = _gen(tag, rows, m, k)
    _, x = _pitched(rows, k, gen)
    wbuf, _ = _pitched(m, k + 1, gen, scale=1.0 / math.sqrt(k))
    bias = torch.randn(m, generator=gen) * 0.5
    bias[: min(4, m)] = torch.tensor(FAR_BIASES[: min(4, m)])
    wbuf[:, k] = bias.cuda()
    return x, wbuf[:, :k], wbuf[:, k]


def _check_fwd_variant(kind, drop, y, ybuf, gbuf, x, W, b, rtol, res, tag):
    """act and gate of one activated forward launch against act_fwd_oracle; dropped elements +0 bitwise; the padding of
    y and of the gate buffer keeps its sentinel."""
    rows, m = y.shape
    keep, s = _keep(rows, m) if drop else (None, 1.0)
    (ra, ba), gam, _ = act_fwd_oracle(kind, x.cpu(), W.cpu(), b.cpu(), keep, s, rtol)
    res[tag + "-act"] = excess(y, ra, ba)
    got = [y.cpu()]
    if gam is not None:
        res[tag + "-gate"] = excess(gbuf[:, :m], *gam)
        got.append(gbuf[:, :m].cpu())
    if keep is not None:
        for t in got:
            assert bool((t[~keep].view(torch.int32) == 0).all()), f"{tag}: a dropped element is not +0"
    assert bool((ybuf[:, m:] == SENTINEL).all()), f"{tag}: FWD wrote into the output's padding"
    assert bool((gbuf[:, m:] == SENTINEL).all()), f"{tag}: FWD wrote into the gate's padding"
    if gam is None:
        assert bool((gbuf == SENTINEL).all()), f"{tag}: a ReLU launch wrote a gate"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("rows,m,k", GRID)
def test_fwd_activation_and_dropout_per_element(rows, m, k, precision):
    K = _K()
    x, W, b = _fwd_inputs("fwd-act", rows, m, k)
    rtol = rtol_for(precision, k)
    for kind, drop in FWD_VARIANTS:
        res = {}
        ybuf, y = _out(rows, m)
        gbuf, gate = _out(rows, m)
        K.linear_fwd(x, W, b, relu=True, out=y, precision=precision, activation=kind,
                     gate=gate if kind != "relu" else None, dropout=DROP if drop else None)
        torch.cuda.synchronize()
        _check_fwd_variant(kind, drop, y, ybuf, gbuf, x, W, b, rtol, res, _variant(kind, drop))
        _note((f"fwd-{_variant(kind, drop)}", precision), res, f"rows={rows} m={m} k={k}")


def _gate_values(rows, cols, gen):
    """A gate: any sign (GELU and SiLU have negative derivatives), exact zeros where dropout dropped."""
    g = torch.randn(rows, cols, generator=gen) * 0.7
    g.view(-1)[0::7] = 0.0
    return g


def _dgrad_inputs(tag, rows, m, k):
    gen = _gen(tag, rows, m, k)
    _, dz = _pitched(rows, k, gen)
    _, W = _pitched(k, m, gen, scale=1.0 / math.sqrt(k))
    masks = []
    for fill in (_mask_values, _gate_values):
        mbuf = torch.full((rows, _ld(m, 8)), NAN)                  # a pitch unlike dX's
        mbuf[:, :m] = fill(rows, m, gen)
        masks.append(mbuf.cuda()[:, :m])
    return dz, W, masks


def _dgrad_variant(K, dz, W, mask, gate, variant, y, precision, k_splits=0):
    if variant == "relu+drop":
        K.linear_dgrad(dz, W, mask=mask, out=y, precision=precision, k_splits=k_splits, dropout=DROP)
    else:
        K.linear_dgrad(dz, W, mask=gate, out=y, precision=precision, k_splits=k_splits, activation="gelu")


def _dgrad_variant_oracle(variant, dz, W, mask, gate, rtol):
    if variant == "relu+drop":
        return act_dgrad_oracle(dz.cpu(), W.cpu(), "relu", mask.cpu(), None, _keep(1, 1)[1], rtol)
    return act_dgrad_oracle(dz.cpu(), W.cpu(), "gelu", None, gate.cpu(), 1.0, rtol)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("rows,m,k", GRID)
def test_dgrad_gate_and_dropout_per_element(rows, m, k, precision):
    """DGRAD through ReLU + dropout (the stored output as the mask, times s where it passes, exactly 0 elsewhere) and
    through a gate (times the gate), each mask with a pitch of its own and NaN in its padding."""
    K = _K()
    dz, W, (mask, gate) = _dgrad_inputs("dgrad-act", rows, m, k)
    rtol = rtol_for(precision, k)
    for variant in ("relu+drop", "gate"):
        dxbuf, dx = _out(rows, m)
        _dgrad_variant(K, dz, W, mask, gate, variant, dx, precision)
        torch.cuda.synchronize()
        ref, bound = _dgrad_variant_oracle(variant, dz, W, mask, gate, rtol)
        if variant == "relu+drop":
            assert bool((dx.cpu()[mask.cpu() <= 0] == 0).all()), "a masked element is not 0"
        assert bool((dxbuf[:, m:] == SENTINEL).all()), "DGRAD wrote into the output's padding"
        _note((f"dgrad-{variant}", precision), {variant: excess(dx, ref, bound)}, f"rows={rows} m={m} k={k}")


@pytest.mark.gpu
def test_linear_fwd_refuses_a_gate_with_another_pitch():
    """The gated epilogue writes the gate with y's row pitch: a gate of another pitch is refused before any launch."""
    K = _K()
    x, W, b = _fwd_inputs("refuse-gate", 16, 40, 33)
    ybuf, y = _out(16, 40)
    gbuf, gate = _out(16, 40, extra=8)
    assert gate.stride(0) != y.stride(0)
    with pytest.raises(RuntimeError, match="row pitch"):
        K.linear_fwd(x, W, b, relu=True, out=y, activation="gelu", gate=gate)
    with pytest.raises(RuntimeError, match="relu"):
        K.linear_fwd(x, W, b, relu=False, out=y, dropout=DROP)
    torch.cuda.synchronize()
    assert bool((ybuf == SENTINEL).all()) and bool((gbuf == SENTINEL).all())


# ================================================================================================== split-K
# (rows, M, K, forced split counts that leave no split empty).  Every shape has >= 2 M tiles and >= 2 N tiles.
SPLITK_CASES = [
    (100, 1500, 777, (2, 3, 5)),          # 25 k-blocks: 13+12, 9+9+7, 5x5 (8 would leave one empty); planner 3
    (130, 300, 1819, (2, 3, 5, 6, 8)),    # 57 k-blocks: 29+28, 19x3, 12x4+9, 10x5+7, 8x7+1; planner 7
    (65, 256, 4096, (2, 3, 5, 8)),        # 128 k-blocks: 64x2, 43+43+42, 26x4+24, 16x8; planner 8
]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mode", ["fwd", "dgrad"])
@pytest.mark.parametrize("rows,m,k,forced", SPLITK_CASES, ids=[f"rows{c[0]}-m{c[1]}-k{c[2]}" for c in SPLITK_CASES])
def test_splitk_per_element_and_deterministic(rows, m, k, forced, mode, precision):
    """FWD (bias + ReLU) and DGRAD (mask) with forced split counts and the planner's: each within the oracle's bound
    (plain and split-K need not agree bit for bit), and three launches bit-identical (the partials are added in a fixed
    split order)."""
    from shallowspeed_b200 import _C

    K = _K()
    gen = _gen("splitk", mode, rows, m, k)
    if mode == "fwd":
        _, a = _pitched(rows, k, gen)
        wbuf, _ = _pitched(m, k + 1, gen, scale=1.0 / math.sqrt(k))
        wbuf[:, k] = torch.randn(m, generator=gen).cuda() * 0.5
        W, b = wbuf[:, :k], wbuf[:, k]
        oracle = lambda rtol: fwd_oracle(a.cpu(), W.cpu(), b.cpu(), True, rtol)
        launch = lambda y, ks: K.linear_fwd(a, W, b, relu=True, out=y, precision=precision, k_splits=ks)
    else:
        _, a = _pitched(rows, k, gen)
        _, W = _pitched(k, m, gen, scale=1.0 / math.sqrt(k))
        mbuf = torch.full((rows, _ld(m, 8)), NAN)
        mbuf[:, :m] = _mask_values(rows, m, gen)
        mask = mbuf.cuda()[:, :m]
        oracle = lambda rtol: dgrad_oracle(a.cpu(), W.cpu(), mask.cpu(), rtol)
        launch = lambda y, ks: K.linear_dgrad(a, W, mask=mask, out=y, precision=precision, k_splits=ks)
    planner = _C.splitk_plan(m, rows, k, torch.cuda.get_device_properties(0).multi_processor_count, 0)[0]
    assert planner >= 2
    res = {}
    for ks in (0,) + tuple(forced) + (-1,):
        splits = planner if ks == -1 else max(ks, 1)
        ref, bound = oracle(rtol_for(precision, k, splits))
        outs = []
        for _ in range(3):
            ybuf, y = _out(rows, m)
            launch(y, ks)
            torch.cuda.synchronize()
            assert bool((ybuf[:, m:] == SENTINEL).all()), f"k_splits={ks} wrote into the output's padding"
            outs.append(_bits(y))
        res[f"ks{ks if ks >= 0 else 'auto'}"] = excess(outs[0].view(torch.float32), ref, bound)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), f"k_splits={ks} is not deterministic"
    _note((f"splitk-{mode}", precision), res, f"rows={rows} m={m} k={k} planner={planner}")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mode", ["fwd", "dgrad"])
@pytest.mark.parametrize("rows,m,k,forced", SPLITK_CASES, ids=[f"rows{c[0]}-m{c[1]}-k{c[2]}" for c in SPLITK_CASES])
def test_splitk_activation_and_dropout_per_element(rows, m, k, forced, mode, precision):
    """The split-K instantiations of the activated and dropout variants (FWD: every FWD_VARIANTS entry; DGRAD: ReLU +
    dropout and the gate) at the first forced split count and the planner's, per element, and two launches bit-identical."""
    K = _K()
    res = {}
    for ks in (forced[0], -1):
        if mode == "fwd":
            x, W, b = _fwd_inputs("splitk-act", rows, m, k)
            for kind, drop in FWD_VARIANTS:
                outs = []
                for _ in range(2):
                    ybuf, y = _out(rows, m)
                    gbuf, gate = _out(rows, m)
                    K.linear_fwd(x, W, b, relu=True, out=y, precision=precision, k_splits=ks, activation=kind,
                                 gate=gate if kind != "relu" else None, dropout=DROP if drop else None)
                    torch.cuda.synchronize()
                    outs.append((_bits(ybuf), _bits(gbuf)))
                tag = f"ks{ks if ks >= 0 else 'auto'}-{_variant(kind, drop)}"
                _check_fwd_variant(kind, drop, y, ybuf, gbuf, x, W, b, rtol_for(precision, k, 8), res, tag)
                assert all(torch.equal(u, v) for u, v in zip(*outs)), f"{tag} is not deterministic"
        else:
            dz, W, (mask, gate) = _dgrad_inputs("splitk-act", rows, m, k)
            for variant in ("relu+drop", "gate"):
                outs = []
                for _ in range(2):
                    dxbuf, dx = _out(rows, m)
                    _dgrad_variant(K, dz, W, mask, gate, variant, dx, precision, k_splits=ks)
                    torch.cuda.synchronize()
                    outs.append(_bits(dxbuf))
                tag = f"ks{ks if ks >= 0 else 'auto'}-{variant}"
                res[tag] = excess(dx, *_dgrad_variant_oracle(variant, dz, W, mask, gate, rtol_for(precision, k, 8)))
                assert torch.equal(outs[0], outs[1]), f"{tag} is not deterministic"
                assert bool((dxbuf[:, m:] == SENTINEL).all()), f"{tag} wrote into the output's padding"
    _note((f"splitk-{mode}-act", precision), res, f"rows={rows} m={m} k={k}")


# ================================================================================================== WGRAD
# in = the N of this GEMM: block_n 32 (in <= 32) or 64, the last column tile full or ragged, in % 4 != 0 (the TMA store
# clips at 16 bytes).  rows = its K.  out = its M: 129 and 300 give a ragged second M tile.
WGRAD_IN = [1, 4, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 777]
WGRAD_ROWS = [1, 2, 31, 33, 128, 512]


def _wgrad_out(n_in):
    return (129, 300, 33)[WGRAD_IN.index(n_in) % 3]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("n_in", WGRAD_IN)
def test_wgrad_per_element_and_padding(n_in, precision):
    """Every rows x accumulate x bias-gradient target (none, a separate vector, the arena column).  Padding contract
    (tc_gemm.cu, the WGRAD epilogue): columns at or beyond round_up(in, 4) keep their bits; columns in
    [in, round_up(in, 4)) keep their value or, for a plain store, become zero; column `in` holds the bias gradient when
    that is where db points."""
    K = _K()
    out = _wgrad_out(n_in)
    r4 = (n_in + 3) // 4 * 4
    ld = _ld(n_in + 1)
    res = {}
    for rows in WGRAD_ROWS:
        gen = _gen("wgrad", n_in, rows, precision)
        _, dz = _pitched(rows, out, gen)
        _, x = _pitched(rows, n_in, gen)
        g, gb = grad_oracle(dz.cpu(), x.cpu(), rtol_for(precision, rows))
        for accumulate in (False, True):
            for db_mode in ("none", "separate", "arena"):
                gbuf = torch.full((out, ld), SENTINEL)
                if accumulate:
                    gbuf[:, : n_in + 1] = torch.randn(out, n_in + 1, generator=gen)
                gbuf = gbuf.cuda()
                sep = torch.randn(out, generator=gen).cuda()
                g0, sep0 = gbuf.cpu(), sep.cpu()
                db = {"none": None, "separate": sep, "arena": gbuf[:, n_in]}[db_mode]
                K.linear_wgrad(dz, x, gbuf[:, :n_in], accumulate=accumulate, grad_b=db, precision=precision)
                torch.cuda.synchronize()
                g1 = gbuf.cpu()
                tag = f"rows{rows}{'acc' if accumulate else ''}-{db_mode}"
                ref, bound = g[:, :n_in], gb[:, :n_in]
                if accumulate:
                    ref = ref + g0[:, :n_in].double()
                    bound = bound + FP32_ULP * ref.abs()
                res[tag] = excess(g1[:, :n_in], ref, bound)
                if db_mode != "none":
                    b_prev = (g0[:, n_in] if db_mode == "arena" else sep0).double()
                    ref_b, bound_b = g[:, n_in], gb[:, n_in]
                    if accumulate:
                        ref_b = ref_b + b_prev
                        bound_b = bound_b + FP32_ULP * ref_b.abs()
                    got_b = g1[:, n_in] if db_mode == "arena" else sep.cpu()
                    res[tag + "-db"] = excess(got_b, ref_b, bound_b)
                # the padding contract
                bias_col = n_in if db_mode == "arena" else None
                for c in range(n_in, ld):
                    if c == bias_col:
                        continue
                    same = torch.equal(_bits(g1[:, c]), _bits(g0[:, c]))
                    if c < r4 and not accumulate:
                        ok = bool(((g1[:, c] == g0[:, c]) | (g1[:, c] == 0.0)).all())
                    else:
                        ok = same
                    assert ok, f"{tag}: padding column {c} of in={n_in} (ld {ld}) changed"
    _note(("wgrad", precision), res, f"in={n_in} out={out}")


# ================================================================================================== fused SGD
SGD_RULES = {"plain": (0.0, 0.0, False), "momentum": (MU, 0.0, False), "nesterov": (MU, 0.0, True),
             "weight-decay": (0.0, WD, False), "momentum+wd": (MU, WD, False), "nesterov+wd": (MU, WD, True)}
SGD_SHAPES = [(32, 127, 126), (1, 5, 300), (33, 65, 129), (128, 777, 200), (512, 64, 33), (2, 4, 1000)]   # rows, in, out


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("rule", list(SGD_RULES))
def test_fused_sgd_per_element(rule, precision):
    """W, V and the bias column per element from random non-zero W and V; G bit-untouched (dW never reaches memory);
    padding of W and V bit-untouched."""
    K = _K()
    mu, wd, nesterov = SGD_RULES[rule]
    res = {}
    for rows, n_in, out in SGD_SHAPES:
        gen = _gen("sgd", rule, rows, n_in, out)
        _, dz = _pitched(rows, out, gen)
        _, x = _pitched(rows, n_in, gen)
        ld = _ld(n_in + 1)
        bufs = []
        for scale in (0.5, 0.1, None):                              # W, V, G
            b = torch.full((out, ld), SENTINEL)
            if scale is not None:
                b[:, : n_in + 1] = torch.randn(out, n_in + 1, generator=gen) * scale
            bufs.append(b.cuda())
        wbuf, vbuf, gbuf = bufs
        w0, v0, g0 = wbuf.cpu(), vbuf.cpu(), gbuf.cpu()
        K.linear_wgrad(dz, x, gbuf[:, :n_in], grad_b=gbuf[:, n_in], weight=wbuf[:, :n_in], lr=SGD_LR, fuse_sgd=True,
                       precision=precision, velocity=vbuf[:, :n_in] if mu > 0 else None, momentum=mu,
                       weight_decay=wd, nesterov=nesterov)
        torch.cuda.synchronize()
        g, gb = grad_oracle(dz.cpu(), x.cpu(), rtol_for(precision, rows))
        v_in = v0[:, : n_in + 1] if mu > 0 else torch.zeros(out, n_in + 1)
        W1, bW, V1, bV = sgd_oracle(g, gb, w0[:, : n_in + 1], v_in, SGD_LR, mu, wd, nesterov)
        w1, v1 = wbuf.cpu(), vbuf.cpu()
        tag = f"r{rows}i{n_in}o{out}"
        res[tag + "-W"] = excess(w1[:, :n_in], W1[:, :n_in], bW[:, :n_in])
        res[tag + "-b"] = excess(w1[:, n_in], W1[:, n_in], bW[:, n_in])
        if mu > 0:
            res[tag + "-V"] = excess(v1[:, : n_in + 1], V1, bV)
        assert torch.equal(_bits(gbuf), _bits(g0)), f"{tag}: the fused update wrote into G"
        assert torch.equal(_bits(w1[:, n_in + 1:]), _bits(w0[:, n_in + 1:])), f"{tag}: W's padding changed"
        assert torch.equal(_bits(v1), _bits(v0)) if mu == 0 else torch.equal(_bits(v1[:, n_in + 1:]), _bits(v0[:, n_in + 1:]))
    _note(("fused-sgd", precision), res, rule)


@pytest.mark.gpu
def test_fused_sgd_refuses_a_bias_gradient_outside_the_block():
    """The fused update writes the bias at db's offset from G, taken in W and V: anything but G's own bias column would
    be a write through an unrelated offset.  The plan refuses it before any launch."""
    K = _K()
    gen = _gen("refuse")
    _, dz = _pitched(8, 33, gen)
    _, x = _pitched(8, 20, gen)
    ld = _ld(21)
    wbuf, vbuf, gbuf = (torch.zeros(33, ld, device="cuda") for _ in range(3))
    separate = torch.zeros(33, device="cuda")
    w0 = wbuf.clone()
    for kw in ({}, dict(velocity=vbuf[:, :20], momentum=MU)):
        for db in (separate, gbuf[:, 19], wbuf[:, 20]):
            with pytest.raises(RuntimeError, match="bias column"):
                K.linear_wgrad(dz, x, gbuf[:, :20], grad_b=db, weight=wbuf[:, :20], lr=0.1, fuse_sgd=True, **kw)
    torch.cuda.synchronize()
    assert torch.equal(wbuf, w0) and int(torch.count_nonzero(gbuf)) == 0 and int(torch.count_nonzero(vbuf)) == 0


# ================================================================================================== the engine
WIDE = {"4096-2048-2048": [4096, 2048, 2048, 10],    # 8 splits on every forward GEMM and on the dgrad
        "1000-1500-777": [1000, 1500, 777, 10]}      # 4 / 5 / 3 forward splits, 3 dgrad splits; in = 777 for WGRAD
FORMS = {"coalesced": (), "per-micro-batch": ("SSB_NO_COALESCE",)}
ENGINE_CASES = [(s, mb, f, sk, "fp32", False) for s in WIDE for mb in (32, 128) for f in FORMS for sk in (0, 1)]
ENGINE_CASES += [(s, 128, "coalesced", 1, "tf32", False) for s in WIDE]
ENGINE_CASES += [("1000-1500-777", 32, f, 1, "fp32", True) for f in FORMS]


def _engine_run(shape, mb_rows, form, splitk, precision, momentum, monkeypatch):
    """Two steps with split-K, one without; each step checked layer by layer from the engine's buffers against the
    weights (and momentum) snapshot taken just before it.  Step 2 runs on new inputs, so an output that a split-K tile
    failed to rewrite (a counter not re-armed) still holds step 1's value and fails the forward oracle."""
    from shallowspeed_b200.parallel.engine import Trainer

    sizes = WIDE[shape]
    monkeypatch.setenv("SSB_SPLITK", str(splitk))
    for k in FORMS[form]:
        monkeypatch.setenv(k, "1")
    L, C, n_mu = len(sizes) - 1, sizes[-1], _n_mu(mb_rows)
    rows = mb_rows * n_mu
    steps = 2 if splitk else 1
    gen = _gen("engine", shape, mb_rows, form, splitk, precision, momentum)
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(steps)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float() for _ in range(steps)]
    Ws, bs = _init_weights(sizes, xs[0], n_mu, gen)
    opt = dict(momentum=MU, weight_decay=WD, nesterov=True) if momentum else {}
    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=LR, precision=precision, **opt)
    model, eng = tr.model, tr.engine
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
        if momentum:
            o, k = model.arena.blocks[i]
            model.arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen).cuda() * 1e-3
    assert not eng.uses_chain()
    assert eng.coalesced() == (form == "coalesced")
    n_split = int(re.search(r"splitk_gemms=(\d+)", eng.describe()).group(1))
    assert (n_split > 0) if splitk else (n_split == 0), eng.describe()
    _poison(eng, model, sizes, rows, True)
    res = {}
    for step in range(steps):
        s = f"s{step + 1}."
        W0 = [model.arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
        if momentum:
            V0 = [model.arena.momentum_block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
        loss = float(tr.step(xs[step].pin_memory(), ts[step].pin_memory()))
        torch.cuda.synchronize()
        act = [xs[step].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L):
            frac = float((act[l] > 0).double().mean())
            assert 0.05 <= frac <= 0.95, f"step {step + 1} layer {l}: {frac:.3f} of the activations are positive"
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"step {step + 1}: dz[{l}] is all zero"
            ref, bound = fwd_oracle(act[l - 1], W0[l - 1][:, :-1], W0[l - 1][:, -1], l < L,
                                    rtol_for(precision, sizes[l - 1]))
            res[s + f"fwd{l}"] = excess(act[l], ref, bound)
        loss_ref = loss_bound = 0.0
        for mu in range(n_mu):
            r = slice(mu * mb_rows, (mu + 1) * mb_rows)
            (_, _), (g, bg), (lv, bl) = head_oracle(act[L][r], ts[step][r], rows, HEAD_RTOL)
            res[s + "dzL"] = max(res.get(s + "dzL", 0.0), excess(dz[L][r], g, bg))
            loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
        res[s + "loss"] = abs(loss - loss_ref) / loss_bound if math.isfinite(loss) else math.inf
        for l in range(L, 1, -1):
            ref, bound = dgrad_oracle(dz[l], W0[l - 1][:, :-1], act[l - 1], rtol_for(precision, sizes[l]))
            res[s + f"dgrad{l}"] = excess(dz[l - 1], ref, bound)
        for i in range(L):
            W1 = model.arena.block(i)[:, : sizes[i] + 1].double().cpu()
            rtol = rtol_for(precision, rows)
            if momentum:
                g, gb = grad_oracle(dz[i + 1], act[i], rtol)
                Wr, bW, Vr, bV = sgd_oracle(g, gb, W0[i], V0[i], LR, MU, WD, True)
                res[s + f"upd{i + 1}"] = excess(W1, Wr, bW)
                V1 = model.arena.momentum_block(i)[:, : sizes[i] + 1].double().cpu()
                res[s + f"mom{i + 1}"] = excess(V1, Vr, bV)
            else:
                ref, bound = update_oracle(dz[i + 1], act[i], W0[i], LR, rtol)
                res[s + f"upd{i + 1}"] = excess(W1 - W0[i], ref, bound)
    kind = "engine-mom" if momentum else "engine"
    _note((kind, precision), res, f"{shape} mb_rows={mb_rows} n_mu={n_mu} {form} splitk={splitk} ({n_split} GEMMs)")


@pytest.mark.gpu
@pytest.mark.parametrize("shape,mb_rows,form,splitk,precision,momentum", ENGINE_CASES)
def test_engine_wide_layers_per_layer(shape, mb_rows, form, splitk, precision, momentum, monkeypatch):
    _engine_run(shape, mb_rows, form, splitk, precision, momentum, monkeypatch)


# ================================================================================================== CPU side
def _block_n(mode, n):
    if mode == "wgrad":
        return 64 if n >= 64 else (n + 31) // 32 * 32
    return 64 if n >= 64 else (n + 15) // 16 * 16


def _plan(mode, m, n, k):
    """Mirror of tc_gemm.cu's plain planning (gemm_plan_*, finish_plan): (block_n, stages, num_kb, grid.x, grid.y)."""
    bn = _block_n(mode, n)
    num_kb = -(-k // 32)
    epi = bn * 512 if mode == "wgrad" else 0
    stages = max(1, min(6, (200 * 1024 - epi) // (128 * 128 + bn * 128), num_kb))
    return bn, stages, num_kb, -(-m // 128), -(-n // bn)


def _engine_gemms(sizes, mb_rows, form):
    """(mode, M, N, K) of every GEMM the layer-wise engine plans for one training step."""
    rows = mb_rows * _n_mu(mb_rows) if form == "coalesced" else mb_rows
    out = []
    for l, (i, o) in enumerate(zip(sizes[:-1], sizes[1:])):
        out.append(("fwd", o, rows, i))
        if l > 0:
            out.append(("dgrad", i, rows, o))
        out.append(("wgrad", o, i, rows))
    return out


def test_grid_reaches_every_planner_branch():
    from shallowspeed_b200 import _C

    sms = 132
    gemms = [(mode, m, rows, k) for rows, m, k in GRID for mode in ("fwd", "dgrad")]
    gemms += [("wgrad", _wgrad_out(i), i, r) for i in WGRAD_IN for r in WGRAD_ROWS]
    gemms += [("wgrad", o, i, r) for r, i, o in SGD_SHAPES]
    splits = [(m, rows, k, ks) for rows, m, k, forced in SPLITK_CASES for ks in forced + (0,)]
    engine_splits = []
    for shape, mb, form, splitk, _, _ in ENGINE_CASES:
        for g in _engine_gemms(WIDE[shape], mb, form):
            gemms.append(g)
            if splitk and g[0] != "wgrad" and _C.splitk_plan(g[1], g[2], g[3], sms, 0)[0] >= 2:
                engine_splits.append((g[1], g[2], g[3], 0))
    assert engine_splits
    seen = {"bn": set(), "wbn": set(), "stages": set(), "wrap": False, "gx": False, "gy": False, "in%4": False,
            "wragged": False}
    for mode, m, n, k in gemms:
        bn, stages, num_kb, gx, gy = _plan(mode, m, n, k)
        seen["wbn" if mode == "wgrad" else "bn"].add(bn)
        seen["stages"].add(stages)
        seen["wrap"] |= num_kb > stages
        seen["gx"] |= gx >= 2
        seen["gy"] |= gy >= 2
        if mode == "wgrad":
            seen["in%4"] |= n % 4 != 0
            seen["wragged"] |= gy >= 2 and n % bn != 0
    assert seen["bn"] == {16, 32, 48, 64} and seen["wbn"] == {32, 64}
    assert seen["stages"] == {1, 2, 3, 4, 5, 6} and seen["wrap"]
    assert seen["gx"] and seen["gy"] and seen["in%4"] and seen["wragged"]
    counts, uneven, both = set(), False, False
    for m, n, k, force in splits + engine_splits:
        got, per, grid_z, stages, _smem, err = _C.splitk_plan(m, n, k, sms, force)
        assert err == "" and got == grid_z >= 2, (m, n, k, force)
        counts.add(got)
        uneven |= per * got != -(-k // 32)
        bn, _, _, gx, gy = _plan("fwd", m, n, k)
        both |= gx >= 2 and gy >= 2
        assert stages == max(2, min(6, 100 * 1024 // (128 * 128 + bn * 128), per))     # gemm_plan_enable_splitk
    assert counts >= set(range(2, 9)) and uneven and both
    # the split counts the engine cases are chosen for (132 SMs, 128 rows)
    want = {(2048, 128, 4096): 8, (2048, 128, 2048): 8, (1500, 128, 1000): 4, (777, 128, 1500): 5, (10, 128, 777): 3,
            (1500, 128, 777): 3}
    for (m, n, k), ks in want.items():
        assert _C.splitk_plan(m, n, k, sms, 0)[0] == ks, (m, n, k)
    # a forced count that would leave a split empty is refused on the host
    assert "empty split" in _C.splitk_plan(1500, 100, 777, sms, 8)[5]


def test_oracles_reject_injected_faults():
    """Each fault is applied to an exact fp64 result; its oracle must reject it and accept the exact result and an fp32
    evaluation of the same operation."""
    rtol = RTOL["fp32"]
    # ---- split-K: 777 = 3 splits of 9, 9 and 7 k-blocks; one partial dropped or counted twice
    x, W, b = _selftest_data(seed=2, rows=64, k=777, n=300)
    ref, bound = fwd_oracle(x, W, b, False, rtol)
    edges = [0, 288, 576, 777]
    parts = [x[:, lo:hi].double() @ W[:, lo:hi].double().T for lo, hi in zip(edges[:-1], edges[1:])]
    exact = sum(parts) + b.double()
    assert excess(exact, ref, bound) <= 1.0 and excess(x @ W.T + b, ref, bound) <= 1.0
    assert excess(exact - parts[2], ref, bound) > 1.0
    assert excess(exact + parts[2], ref, bound) > 1.0
    # ---- the bias missing on the last M tile only (output features 256..299)
    nob = exact.clone()
    nob[:, 256:] -= b[256:].double()
    assert excess(nob, ref, bound) > 1.0
    # ---- a stale output: the previous step's, same inputs, weights before one SGD step of lr = LR
    g = torch.Generator().manual_seed(3)
    dz_prev = torch.randn(64, 300, generator=g) * 1e-3
    d, _ = update_oracle(dz_prev, x, torch.cat([W, b[:, None]], 1), LR, rtol)
    W2, b2 = W.double() + d[:, :-1], b.double() + d[:, -1]
    ref2, bound2 = fwd_oracle(x, W2, b2, True, rtol)
    assert excess(ref2, ref2, bound2) <= 1.0 and excess((x.double() @ W2.T + b2).float().clamp_min(0), ref2, bound2) <= 1.0
    assert excess(exact.clamp_min(0.0), ref2, bound2) > 1.0

    # ---- the mask read with dX's pitch instead of its own
    rows, m, k = 33, 130, 97
    dz = torch.randn(rows, k, generator=g)
    Wd = torch.randn(k, m, generator=g) / math.sqrt(k)
    mbuf = torch.full((rows, _ld(m, 8)), NAN)
    mbuf[:, :m] = _mask_values(rows, m, g)
    mask = mbuf[:, :m]
    dref, dbound = dgrad_oracle(dz, Wd, mask, rtol)
    assert excess(dref, dref, dbound) <= 1.0 and excess((dz @ Wd) * (mask > 0), dref, dbound) <= 1.0
    flat, ld_dx = mbuf.reshape(-1), _ld(m)
    wrong = torch.stack([flat[r * ld_dx: r * ld_dx + m] for r in range(rows)])
    assert excess((dz.double() @ Wd.double()) * (wrong > 0), dref, dbound) > 1.0

    # ---- the stateful rule: Nesterov's mu * v dropped, weight decay skipped on the bias column, V not written back
    rows, n_in, out = 64, 128, 97
    dzs = torch.randn(rows, out, generator=g) * 0.1
    xs = torch.randn(rows, n_in, generator=g)
    W0 = torch.randn(out, n_in + 1, generator=g) * 0.5
    V0 = torch.randn(out, n_in + 1, generator=g) * 0.1
    gr, gb = grad_oracle(dzs, xs, rtol)
    W1, bW, V1, bV = sgd_oracle(gr, gb, W0, V0, SGD_LR, MU, WD, True)
    assert excess(W1, W1, bW) <= 1.0 and excess(V1, V1, bV) <= 1.0
    # fp32 all the way (torch's rule on an fp32 gradient): accepted
    g32 = torch.cat([dzs.T @ xs, dzs.sum(0)[:, None]], 1)
    gp32 = g32 + WD * W0
    v32 = MU * V0 + gp32
    w32 = W0 - SGD_LR * (gp32 + MU * v32)
    assert excess(w32, W1, bW) <= 1.0 and excess(v32, V1, bV) <= 1.0
    W0d, V0d = W0.double(), V0.double()
    gp = gr + WD * W0d
    v = MU * V0d + gp
    assert excess(W0d - SGD_LR * gp, W1, bW) > 1.0                                  # no mu * v
    gp_nb = gp.clone()
    gp_nb[:, -1] = gr[:, -1]
    v_nb = MU * V0d + gp_nb
    w_nb = W0d - SGD_LR * (gp_nb + MU * v_nb)
    assert excess(w_nb[:, -1], W1[:, -1], bW[:, -1]) > 1.0                         # no decay on the bias
    assert excess(v_nb[:, -1], V1[:, -1], bV[:, -1]) > 1.0
    assert excess(V0d, V1, bV) > 1.0                                                # V not written back
    assert excess(W0d - SGD_LR * (gp + MU * v), W1, bW) <= 1.0


# ================================================================================================== the residual form
# tc_gemm_res_kernel through ops.cuda's residual=True: FWD out = skip + f(z) * keep * s (every activation gated, ReLU's
# gate 1[z > 0] * keep * s), DGRAD gpre = dz W + skip, out = gpre * mask (the mask: the previous layer's gate).  skip,
# gpre and the mask each have a row pitch unlike out's.  bf16 through test_gpu_bf16's operand model.  The last feature
# of every shape is nil (FWD: zero weight row and bias, so f(0) = 0; DGRAD: zero weight column), where the result is the
# skip itself up to one rounding: a skip rounded or truncated like an operand fails there.
RES_PRECISIONS = ["fp32", "tf32", "bf16"]
RES_FWD_VARIANTS = [("relu", False)] + FWD_VARIANTS


def _res_ops(precision, k, splits=1):
    """(operand model, rtol) of a product of K = k in this precision (test_gpu_bf16 for bf16)."""
    if precision == "bf16":
        from test_gpu_bf16 import bf, rtol_bf16

        return bf, rtol_bf16(k, splits)
    return (lambda t: t.double().cpu()), rtol_for(precision, k, splits)


def _res_fwd_inputs(tag, rows, m, k):
    x, W, b = _fwd_inputs(tag, rows, m, k)
    W[m - 1] = 0.0                                          # the nil output feature
    b[m - 1] = 0.0
    _, skip = _pitched(rows, m, _gen(tag, "skip", rows, m, k), extra=12)
    assert skip.stride(0) != _out(1, m)[1].stride(0)
    return x, W, b, skip


def _check_res_fwd(kind, drop, skip, y, ybuf, gbuf, x, W, b, op, rtol, res, tag):
    rows, m = y.shape
    keep, s = _keep(rows, m) if drop else (None, 1.0)
    (ra, ba), gam, z = act_fwd_oracle(kind, op(x), op(W), b.cpu(), keep, s, rtol)
    sk = skip.cpu().double() if skip is not None else torch.zeros(rows, m, dtype=torch.float64)
    ref = sk + ra
    res[tag + "-out"] = excess(y, ref, ba * (1.0 + U) + U * ref.abs() + ATOL)
    res[tag + "-skip"] = excess(y[:, m - 1], sk[:, m - 1], U * sk[:, m - 1].abs() + ATOL)
    g = gbuf[:, :m].cpu()
    if kind == "relu":
        e = fwd_oracle(op(x), op(W), b.cpu(), False, rtol)[1]
        want = (z > 0).double() * s * (1.0 if keep is None else keep.double())
        sure = z.abs() > e
        assert torch.equal(g.double()[sure], want[sure]), f"{tag}: a ReLU gate is not 1[z > 0] * keep * s"
        assert bool(((g == 0) | (g == s)).all()), f"{tag}: a ReLU gate is neither 0 nor s"
    else:
        res[tag + "-gate"] = excess(g, *gam)
    if keep is not None:
        want = skip.cpu()[~keep] if skip is not None else torch.zeros(int((~keep).sum()))
        assert torch.equal(y.cpu()[~keep].view(torch.int32), want.view(torch.int32)), f"{tag}: a dropped output is not the skip"
        assert bool((g[~keep].view(torch.int32) == 0).all()), f"{tag}: a dropped gate is not +0"
    assert bool((ybuf[:, m:] == SENTINEL).all()), f"{tag}: FWD wrote into the output's padding"
    assert bool((gbuf[:, m:] == SENTINEL).all()), f"{tag}: FWD wrote into the gate's padding"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", RES_PRECISIONS)
@pytest.mark.parametrize("rows,m,k", GRID)
def test_fwd_residual_per_element(rows, m, k, precision):
    """Every activation with and without dropout, with a skip and without one; without one the output equals the gated
    non-residual launch's (a smooth kind) or the plain ReLU / dropout launch's."""
    K = _K()
    x, W, b, skip = _res_fwd_inputs("fwd-res", rows, m, k)
    op, rtol = _res_ops(precision, k)
    for kind, drop in RES_FWD_VARIANTS:
        res = {}
        for with_skip in (True, False):
            ybuf, y = _out(rows, m)
            gbuf, gate = _out(rows, m)
            K.linear_fwd(x, W, b, relu=True, out=y, precision=precision, activation=kind, gate=gate,
                         dropout=DROP if drop else None, residual=True, skip=skip if with_skip else None)
            torch.cuda.synchronize()
            tag = f"{_variant(kind, drop)}-skip{int(with_skip)}"
            _check_res_fwd(kind, drop, skip if with_skip else None, y, ybuf, gbuf, x, W, b, op, rtol, res, tag)
        pbuf, plain = _out(rows, m)
        K.linear_fwd(x, W, b, relu=True, out=plain, precision=precision, activation=kind, dropout=DROP if drop else None,
                     gate=_out(rows, m)[1] if kind != "relu" else None)
        torch.cuda.synchronize()
        assert torch.equal(y.cpu(), plain.cpu()), f"{_variant(kind, drop)}: skip=None differs from the plain launch"
        _note((f"fwd-res-{_variant(kind, drop)}", precision), res, f"rows={rows} m={m} k={k}")


def _check_res_dgrad(dz, W, mask, skip, gpre, dx, dxbuf, gpbuf, op, rtol, res, tag):
    rows, m = dx.shape
    prod = op(dz) @ op(W)
    sk = skip.cpu().double() if skip is not None else torch.zeros_like(prod)
    pre = prod + sk
    pre_b = rtol * (op(dz).abs() @ op(W).abs()) + U * (prod.abs() + sk.abs()) + ATOL
    mk = mask.cpu().double() if mask is not None else torch.ones_like(pre)
    res[tag + "-out"] = excess(dx, pre * mk, pre_b * mk.abs() + U * (pre * mk).abs() + ATOL)
    res[tag + "-skip"] = excess(dx[:, m - 1], (sk * mk)[:, m - 1], 2.0 * U * (sk * mk)[:, m - 1].abs() + ATOL)
    if gpre is not None:
        res[tag + "-gpre"] = excess(gpre, pre, pre_b)
        g = gpre.cpu()
        want = (g * mask.cpu()) if mask is not None else g
        assert torch.equal(dx.cpu().view(torch.int32), want.view(torch.int32)), f"{tag}: out is not fp32(gpre * mask)"
        assert bool((gpbuf[:, m:] == SENTINEL).all()), f"{tag}: DGRAD wrote into gpre's padding"
    else:
        assert bool((gpbuf == SENTINEL).all()), f"{tag}: DGRAD wrote a gpre it was not given"
    assert bool((dxbuf[:, m:] == SENTINEL).all()), f"{tag}: DGRAD wrote into the output's padding"


def _res_dgrad_inputs(tag, rows, m, k):
    dz, W, (_, gate) = _dgrad_inputs(tag, rows, m, k)
    W[:, m - 1] = 0.0                                       # the nil input feature
    _, skip = _pitched(rows, m, _gen(tag, "skip", rows, m, k), scale=0.5, extra=12)
    return dz, W, gate, skip


@pytest.mark.gpu
@pytest.mark.parametrize("precision", RES_PRECISIONS)
@pytest.mark.parametrize("rows,m,k", GRID)
def test_dgrad_residual_per_element(rows, m, k, precision):
    """Every combination of skip, gpre and mask present or null."""
    K = _K()
    dz, W, gate, skip = _res_dgrad_inputs("dgrad-res", rows, m, k)
    op, rtol = _res_ops(precision, k)
    res = {}
    for has_skip in (True, False):
        for has_gpre in (True, False):
            for has_mask in (True, False):
                dxbuf, dx = _out(rows, m)
                gpbuf, gp = _out(rows, m, extra=16)
                assert len({dx.stride(0), gp.stride(0), gate.stride(0), skip.stride(0)}) == 4
                K.linear_dgrad(dz, W, mask=gate if has_mask else None, out=dx, precision=precision, residual=True,
                               skip=skip if has_skip else None, gpre=gp if has_gpre else None)
                torch.cuda.synchronize()
                tag = f"skip{int(has_skip)}gpre{int(has_gpre)}mask{int(has_mask)}"
                _check_res_dgrad(dz, W, gate if has_mask else None, skip if has_skip else None, gp if has_gpre else None,
                                 dx, dxbuf, gpbuf, op, rtol, res, tag)
    _note(("dgrad-res", precision), res, f"rows={rows} m={m} k={k}")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", RES_PRECISIONS)
@pytest.mark.parametrize("mode", ["fwd", "dgrad"])
@pytest.mark.parametrize("rows,m,k,forced", SPLITK_CASES, ids=[f"rows{c[0]}-m{c[1]}-k{c[2]}" for c in SPLITK_CASES])
def test_splitk_residual_per_element_and_deterministic(rows, m, k, forced, mode, precision):
    """The split-K instantiations of the residual form at every forced split count and the planner's, per element, two
    launches bit-identical.  FWD: ReLU and GELU with dropout in turn; DGRAD: skip, gpre and the mask."""
    K = _K()
    res = {}
    for i, ks in enumerate(tuple(forced) + (-1,)):
        op, rtol = _res_ops(precision, k, 8)
        tag = f"ks{ks if ks >= 0 else 'auto'}"
        outs = []
        for _ in range(2):
            if mode == "fwd":
                x, W, b, skip = _res_fwd_inputs("splitk-res", rows, m, k)
                kind, drop = (("relu", False), ("gelu", True))[i % 2]
                ybuf, y = _out(rows, m)
                gbuf, gate = _out(rows, m)
                K.linear_fwd(x, W, b, relu=True, out=y, precision=precision, k_splits=ks, activation=kind, gate=gate,
                             dropout=DROP if drop else None, residual=True, skip=skip)
                torch.cuda.synchronize()
                outs.append((_bits(ybuf), _bits(gbuf)))
            else:
                dz, W, gate, skip = _res_dgrad_inputs("splitk-res", rows, m, k)
                dxbuf, dx = _out(rows, m)
                gpbuf, gp = _out(rows, m, extra=16)
                K.linear_dgrad(dz, W, mask=gate, out=dx, precision=precision, k_splits=ks, residual=True, skip=skip, gpre=gp)
                torch.cuda.synchronize()
                outs.append((_bits(dxbuf), _bits(gpbuf)))
        if mode == "fwd":
            _check_res_fwd(kind, drop, skip, y, ybuf, gbuf, x, W, b, op, rtol, res, f"{tag}-{_variant(kind, drop)}")
        else:
            _check_res_dgrad(dz, W, gate, skip, gp, dx, dxbuf, gpbuf, op, rtol, res, tag)
        assert all(torch.equal(u, v) for u, v in zip(*outs)), f"{tag} is not deterministic"
    _note((f"splitk-{mode}-res", precision), res, f"rows={rows} m={m} k={k}")


@pytest.mark.gpu
def test_residual_arguments_default_to_the_plain_launch_bit_for_bit():
    """residual=False, skip=None and gpre=None are the launches of before: the same bits as the bindings called without
    the residual arguments, on one shape per mode; and the bindings refuse residual arguments they cannot honour."""
    from shallowspeed_b200 import _C

    K = _K()
    x, W, b, skip = _res_fwd_inputs("res-defaults", 65, 129, 100)
    outs = []
    for call in range(3):
        ybuf, y = _out(65, 129)
        gbuf, gate = _out(65, 129)
        if call == 0:
            K.linear_fwd(x, W, b, relu=True, out=y, activation="gelu", gate=gate, dropout=DROP)
        elif call == 1:
            K.linear_fwd(x, W, b, relu=True, out=y, activation="gelu", gate=gate, dropout=DROP, residual=False, skip=None)
        else:
            bias, bstride = K._bias_arg(b, 129)
            _C.linear_fwd(x, W, bias, bstride, True, y, 1, 0, 1, gate, DROP)
        torch.cuda.synchronize()
        outs.append((_bits(ybuf), _bits(gbuf)))
    assert all(torch.equal(u, v) for o in outs[1:] for u, v in zip(outs[0], o))
    dz, Wd, gate, gskip = _res_dgrad_inputs("res-defaults", 65, 129, 100)
    outs = []
    for call in range(3):
        dxbuf, dx = _out(65, 129)
        if call == 0:
            K.linear_dgrad(dz, Wd, mask=gate, out=dx, activation="gelu")
        elif call == 1:
            K.linear_dgrad(dz, Wd, mask=gate, out=dx, activation="gelu", residual=False, skip=None, gpre=None)
        else:
            _C.linear_dgrad(dz, Wd, gate, dx, 1, 0, 1, None)
        torch.cuda.synchronize()
        outs.append(_bits(dxbuf))
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    _, y = _out(65, 129)
    _, gp = _out(65, 129)
    with pytest.raises(RuntimeError, match="needs residual"):
        K.linear_fwd(x, W, b, relu=True, out=y, skip=skip)
    with pytest.raises(RuntimeError, match="need residual"):
        K.linear_dgrad(dz, Wd, mask=gate, out=dx, skip=gskip)
    with pytest.raises(RuntimeError, match="need residual"):
        K.linear_dgrad(dz, Wd, mask=gate, out=dx, gpre=gp)
    with pytest.raises(RuntimeError, match="dropout"):
        K.linear_dgrad(dz, Wd, mask=gate, out=dx, residual=True, dropout=DROP)
    with pytest.raises(RuntimeError, match="skip shape"):
        K.linear_fwd(x, W, b, relu=True, out=y, residual=True, skip=skip[:, :128])
    with pytest.raises(RuntimeError, match="gpre shape"):
        K.linear_dgrad(dz, Wd, mask=gate, out=dx, residual=True, gpre=gp[:64])
    with pytest.raises(RuntimeError, match="row pitch"):
        K.linear_fwd(x, W, b, relu=True, out=y, residual=True, gate=_out(65, 129, extra=8)[1])
    with pytest.raises(RuntimeError, match="fp32"):
        K.linear_fwd(x, W, b, relu=True, out=y, residual=True, skip=skip.double())
    with pytest.raises(RuntimeError, match="only a smooth activation or a residual layer"):
        K.linear_fwd(x, W, b, relu=True, out=y, gate=_out(65, 129)[1])


def test_residual_oracles_reject_a_rounded_skip():
    """At a nil feature the bound is one rounding of the skip: the exact skip passes, the skip rounded to bf16 or
    truncated to tf32 (as a product's operand would be) fails, and so does a skip gradient added after the mask."""
    from test_gpu_bf16 import bf
    from test_gpu_chain import tf32_trunc

    g = torch.Generator().manual_seed(4)
    skip = torch.randn(64, 8, generator=g)
    sk = skip.double()
    bound = U * sk.abs() + ATOL
    assert excess(skip, sk, bound) <= 1.0
    assert excess(bf(skip), sk, bound) > 1.0
    assert excess(tf32_trunc(skip), sk, bound) > 1.0
    mk = torch.rand(64, 8, generator=g).double() + 0.5
    assert excess((skip.double() * mk).float(), sk * mk, 2.0 * U * (sk * mk).abs() + ATOL) <= 1.0
    assert excess(sk * 0.0 + sk, sk * mk, 2.0 * U * (sk * mk).abs() + ATOL) > 1.0
