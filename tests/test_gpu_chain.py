"""The layer-chain kernel (``csrc/kernels/mlp_chain.cu``) against a per-layer fp64 oracle, at every micro-batch size,
width, depth and class count it accepts, and the layer-wise fallback at the shapes the chain refuses.

One training step runs through ``Trainer``; every layer is then checked on its own, in fp64, from the engine's own
buffers: the forward product of layer l from the kernel's act[l-1], the loss head from the kernel's logits, the dgrad of
layer l from the kernel's dz[l] and the mask of its act[l-1], the SGD update from the kernel's dz and act.  Errors
cannot cascade and ReLU sign flips cannot blur the comparison, so the bounds are per element:

    |got - ref| <= rtol * (|A| @ |B|) + ATOL            (bias as one more column of A with a 1 in B)

The CPU tests at the end check that the grid reaches every branch the kernel chooses by shape, and that the comparison
helpers reject a set of plausible kernel faults while accepting a correct result.
"""
import math

import pytest
import torch

# ------------------------------------------------------------------------------------------------------------------
# Error bounds.  Operands are split into TF32 by truncation (ptx.cuh: tf32_hi_bits; the tensor core truncates lo as
# well), and every 32-wide k-block is summed in a fresh fp32 accumulator.
# * fp32 (3xTF32): hi*hi + hi*lo + lo*hi.  Truncating lo loses < 2^-20 of each operand and lo*lo < 2^-20 of the
#   product, so one product is off by < 3 * 2^-20 of |a||b|; the fp32 sums over the k-blocks add ~(K/32) * 2^-24 in
#   the worst case.  2^-16 is about 4x the sum of both at K = 4096.
# * tf32: one truncated pass, < 2^-10 per operand, so < 2^-9 of |a||b| per product.  This is the worst case, not an
#   estimate: with few terms (a 2-row weight gradient) nothing averages out and the error comes close to it.
# * the loss head is plain fp32 (expf, one sum of <= 32 terms, one division) in both precisions: the relative error
#   of a probability is < 2^-18 for logits that span < 80; 2^-16 is the bound for every quantity derived from it.
# Worst err / bound over the grid, measured on an H100 80GB HBM3 (400 W): fp32 0.09 for the products, 0.49 for the
# update (its fp32 storage rounding); tf32 0.91 (the update at 2 rows), 0.81 for the products; loss head 0.09.
RTOL = {"fp32": 2.0**-16, "tf32": 2.0**-9}
HEAD_RTOL = 2.0**-16
# sums of flushed / underflowed subnormal products (<= 4096 terms of < 2^-126 each) and exact zeros
ATOL = 1e-30
LR = 1.0                      # large enough that the update stands well above the fp32 rounding of the weights
LOGIT_SPREAD = 20.0           # within a micro-batch: far rows depend on the +1e-7 of the global-max softmax
FP32_ULP = 2.0**-23

BASE = [784, 128, 97, 33, 10]
MB_GRID = [1, 8, 16, 24, 32, 40, 48, 64, 80, 100, 112, 128]
SHAPES = {
    "loss-head-only": [784, 10],                       # L = 1: no dgrad GEMM
    "tiny": [7, 5, 3],                                  # fan-in below one k-block
    "straddle-c17": [33, 32, 31, 17],                   # k-block edges; C = 17 runs the slow loss head
    "full-c16": [784, 128, 128, 16],                    # full-width layers; C = 16 is the fast-path edge
    "c32-k4096": [4096, 96, 64, 32],                    # C = 32 (the maximum); many ring wraps
    "depth16": [100] + [40] * 15 + [10],                # kChainMaxLayers
}
FALLBACKS = {
    "depth17": [100] + [40] * 16 + [10],                # more layers than the chain plan holds
    "too-wide": [784, 129, 10],                         # a layer wider than one M tile
    "c33": [784, 64, 33],                               # more classes than the fused loss head takes
}


def _n_mu(mb_rows):
    return 1 if mb_rows == 128 else 2


# ================================================================================================== oracle helpers
def excess(got, ref, bound):
    """max |got - ref| / bound over all elements (inf if ``got`` holds a non-finite value)."""
    got = got.double().cpu()
    if not bool(torch.isfinite(got).all()):
        return math.inf
    if got.numel() == 0:
        return 0.0
    return float(((got - ref).abs() / bound).max())


def fwd_oracle(x, W, b, relu, rtol):
    """relu?(x @ W.T + b) in fp64 and its per-element bound."""
    x, W, b = x.double(), W.double(), b.double()
    z = x @ W.T + b
    mag = x.abs() @ W.abs().T + b.abs()
    return (z.clamp_min(0.0) if relu else z), rtol * mag + ATOL


def dgrad_oracle(dz, W, act_prev, rtol):
    """(dz @ W) * (act_prev > 0) in fp64 (the mask from the activation the kernel stored) and its bound."""
    dz, W = dz.double(), W.double()
    return (dz @ W) * (act_prev > 0), rtol * (dz.abs() @ W.abs()) + ATOL


def head_oracle(z, t, batch, rtol):
    """Loss head of ONE micro-batch on the kernel's logits ``z``: (probs, dz, loss) in fp64 through the reference
    contract (``ops.functional``: shift by the micro-batch's global max, +1e-7) and their bounds.  The bounds carry a
    relative error ``rtol`` of every probability through the MSE gradient and the softmax Jacobian to first order."""
    from shallowspeed_b200.ops import functional as F

    z, t = z.double(), t.double()
    p = F.softmax_ref(z)
    dp = F.mse_loss_grad_ref(p, t, batch)
    dz = F.softmax_grad_ref(dp, z)
    loss = float(F.mse_loss_ref(p, t, batch))
    sens = p * (dp.abs() + 2.0 * p / batch)                    # |d(p * dp)| per unit relative error of p
    g_sum = (p * dp).sum(1, keepdim=True).abs()
    b_dz = rtol * (sens + p * g_sum + p * sens.sum(1, keepdim=True)) + ATOL
    b_loss = rtol * float(((t - p) ** 2 + 2.0 * (t - p).abs() * p).sum()) / batch + ATOL
    return (p, rtol * p + ATOL), (dz, b_dz), (loss, b_loss)


def update_oracle(dz, a_prev, W0, lr, rtol):
    """SGD step of one layer over all rows: ``-lr * [dz.T @ a_prev | sum(dz)]`` and its bound, plus one fp32 ulp of
    the weights for the rounding of the stored result.  ``W0`` is the [out, in + 1] block before the step."""
    dz, a_prev, W0 = dz.double(), a_prev.double(), W0.double()
    d = -lr * torch.cat([dz.T @ a_prev, dz.sum(0)[:, None]], dim=1)
    mag = lr * torch.cat([dz.abs().T @ a_prev.abs(), dz.abs().sum(0)[:, None]], dim=1)
    return d, rtol * mag + FP32_ULP * (W0.abs() + d.abs()) + ATOL


def tf32_trunc(x):
    """The single-pass TF32 operand of the kernels: fp32 with the low 13 mantissa bits cut."""
    return (x.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


# ================================================================================================== activated layers
# The forward epilogue of an activated layer computes z in fp32 (the GEMM), then a = f(z) and the gate g = f'(z) with the
# device formulas of ptx.cuh: act_fwd, then, under dropout, keep ? (a * s, g * s) : (0, 0).  Against the fp64 reference
# f(z_ref) * s, with z_ref and e_z = rtol * mag + ATOL from fwd_oracle, the error of a kept element is at most
#   (a) s * e_z * sup |f'| over [z_ref - e_z, z_ref + e_z]   (z carried through f; sup |f'| <= |f'(z_ref)| + e_z * M2)
#   (b) s * B(z): the rounding of the device formula itself, for any fp32 z in that interval
#   (c) U * s * |f|: the one rounding of "* s"
# and the same for g with f' and f'' in place of f and f'.  M1, M2, M3 = sup |f'|, |f''|, |f'''| over the reals.
#
# (b), by operation, with U = 2^-24: a product or a sum adds U of its result, a correctly rounded division the same,
# and erff, expf and tanhf add 2 ulp <= 4U of theirs (the CUDA Math API's maximum ulp errors; no fast-math).  An input
# error carries through the operation's derivative.  First order in U (the dropped U^2 terms are below 1e-6 of these):
#   GELU  c = 0.5 (1 + erff(z * fl(1/sqrt2))): 2U of the product, carried through erf' (at most (2/sqrt(pi)) u e^-u^2
#         * 2U < U), 4U of erff, U * 2c of the sum:        |dc| <= 2.5U + U c (absolute: the 1 + erf cancellation)
#         a = z c:                                          |da| <= U |z| (2.5 + 2c)
#         g = c + z (expf(-0.5 z z) * fl(1/sqrt(2 pi))): U z^2 / 2 of the exponent carried through exp, 4U of expf, U
#         of the constant, 3U of the products, U of the sum: |dg| <= U (2.5 + c + |g| + |z| phi(z) (7 + z^2 / 2))
#   SiLU  s = 1 / (1 + expf(-z)): 4U of expf, U of the sum, U of the division: |ds| <= 6U s, and, since 1 is a
#         rounding candidate of both the sum and the quotient, |ds| <= (2 + 4U)(1 - s) as well (s rounds to 1 once
#         e^-z < U: the error is then e^-z, not 6U); q = 1 - s: |dq| <= |ds| + U q
#         a = z s:                                          |da| <= |z| |ds| + U |a|
#         g = s (1 + z q): r = z q, |dr| <= |z| |dq| + U |z| q ; w = 1 + r, |dw| <= |dr| + U |w|
#                                                           |dg| <= |w| |ds| + s |dw| + U |g|
#   tanh  t = tanhf(z), |dt| <= 4U |t| ;  a = t:             |da| <= 4U |t|
#         g = 1 - t t:                                      |dg| <= 9U t^2 + U |g| (1 - t^2 cancels: absolute)
# Each magnitude is taken at its supremum over [z_ref - e_z, z_ref + e_z] (|z| + e_z, sigma and Phi at the upper end,
# |f| + e_z M1, ...).  ATOL (1e-30) covers what the first-order terms do not: expf overflowing to inf below z = -88.72
# (SiLU's s = 0 where sigma(z) < 3e-39) and subnormal intermediates, all below 1e-36 in absolute terms.
# These terms are absolute errors of order |z| * 2^-24 where f or f' is small against |z| (GELU below z = -5, tanh' above
# |z| = 8): the tests accept that tail cancellation; act_fwd does not change.
ACT_LIP = {"gelu": (1.13, 0.80, 0.78), "silu": (1.10, 0.50, 0.31), "tanh": (1.0, 0.77, 2.0)}   # M1, M2, M3, rounded up
U = 2.0**-24
_SQRT2 = math.sqrt(2.0)


def act_ref(kind, z):
    """(f, f', f'') of a smooth activation in fp64 (GELU through erfc, so that its left tail keeps its digits)."""
    z = z.double()
    if kind == "gelu":
        Phi = 0.5 * torch.special.erfc(-z / _SQRT2)
        phi = torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)
        return z * Phi, Phi + z * phi, phi * (2.0 - z * z)
    if kind == "silu":
        s, q = torch.sigmoid(z), torch.sigmoid(-z)
        return z * s, s * (1.0 + z * q), s * q * (2.0 - z * torch.tanh(0.5 * z))
    t, sech2 = torch.tanh(z), 1.0 / torch.cosh(z) ** 2
    return t, sech2, -2.0 * t * sech2


def act_rounding_bound(kind, z, e):
    """Bound (b) on |f_dev(y) - f(y)| and |f'_dev(y) - f'(y)| for every fp32 y within ``e`` of ``z`` (see above)."""
    z, e = z.double(), torch.as_tensor(e, dtype=torch.float64)
    M1, M2, _ = ACT_LIP[kind]
    f, f1, _ = act_ref(kind, z)
    lo, hi = z - e, z + e
    Z = z.abs() + e
    A, G = f.abs() + e * M1, f1.abs() + e * M2
    if kind == "gelu":
        C = 0.5 * torch.special.erfc(-hi / _SQRT2)
        zmin = (z.abs() - e).clamp_min(0.0)
        tail = torch.exp(-0.5 * zmin * zmin) / math.sqrt(2.0 * math.pi) * Z * (7.0 + 0.5 * Z * Z)
        return U * Z * (2.5 + 2.0 * C), U * (2.5 + C + G + tail)
    if kind == "silu":
        S, Q = torch.sigmoid(hi), torch.sigmoid(-lo)
        ds = torch.minimum(6.0 * U * S, (2.0 + 4.0 * U) * Q)
        dq = ds + U * Q
        Wm = 1.0 + Z * Q
        dw = Z * dq + U * Z * Q + U * Wm
        return Z * ds + U * A, Wm * ds + S * dw + U * G
    T = torch.maximum(torch.tanh(lo).abs(), torch.tanh(hi).abs())
    return 4.0 * U * T, 9.0 * U * T * T + U * G


def act_fwd_oracle(kind, a_prev, W, b, keep, s, rtol):
    """An activated layer from the kernel's own input: ((act, bound), (gate, bound) or None, z_ref) in fp64.  ``keep``:
    the dropout mask (None: no dropout), ``s``: the fp32 scale the kernel multiplies by.  Dropped elements have the
    reference 0 and the bound ATOL; the caller checks them bitwise."""
    z, e = fwd_oracle(a_prev, W, b, False, rtol)
    keep_f = torch.ones_like(z) if keep is None else keep.to(z.device).double()
    if kind == "relu":
        a = z.clamp_min(0.0)
        return (a * s * keep_f, (s * e + U * s * a) * keep_f + ATOL), None, z
    M1, M2, M3 = ACT_LIP[kind]
    f, f1, f2 = act_ref(kind, z)
    Ba, Bg = act_rounding_bound(kind, z, e)
    ba = s * (e * (f1.abs() + e * M2) + Ba) + U * s * (f.abs() + e * M1)
    bg = s * (e * (f2.abs() + e * M3) + Bg) + U * s * (f1.abs() + e * M2)
    return (f * s * keep_f, ba * keep_f + ATOL), (f1 * s * keep_f, bg * keep_f + ATOL), z


def act_dgrad_oracle(dz, W, kind, act_prev, gate_prev, s, rtol):
    """dgrad through an activated layer, from the kernel's own stored mask: (dz @ W) * gate_prev for a smooth kind,
    (dz @ W) * (act_prev > 0) * s for ReLU (s = 1 without dropout), and its bound.  One more rounding, of the multiply."""
    dz, W = dz.double(), W.double()
    m = gate_prev.double() if kind != "relu" else (act_prev > 0).double() * s
    ref = (dz @ W) * m
    return ref, rtol * (dz.abs() @ W.abs()) * m.abs() + U * ref.abs() + ATOL


def rows_update_oracle(dz, a_prev, W0, lr, rtol):
    """update_oracle plus the bias column's fp32 sum over the rows in order (one rounding per row, as test_gpu_gemm's
    grad_oracle): the engines sum up to 1024 rows, past RTOL's margin for it in fp32."""
    d, bound = update_oracle(dz, a_prev, W0, lr, rtol)
    bound[:, -1] += dz.shape[0] * U * lr * dz.double().abs().sum(0)
    return d, bound


WORST = {}                    # (kernel, activation, dropout, precision) -> (worst err / bound, its check and case)


def note_worst(key, res, what):
    for k, v in res.items():
        if v > WORST.get(key, (-1.0, ""))[0]:
            WORST[key] = (v, f"{k} at {what}")


@pytest.fixture(scope="module", autouse=True)
def worst_table():
    yield
    print()
    for (kernel, kind, drop, precision), (v, what) in sorted(WORST.items()):
        print(f"[worst] {kernel:>10} {kind:>4} {'drop' if drop else 'nodrop':>6} {precision}: {v:.3g} ({what})")


def check_layers(eng, model, W0, x, n_mu, mb, precision, lr, samples_of, step=0, check_update=True):
    """Every layer of the step that just ran, per micro-batch and per element, from the engine's own buffers against
    fp64: act (and the gate) of every activated layer through act_fwd_oracle, with the masks of
    ``ops.functional.dropout_mask`` and dropped elements exactly 0; every dgrad through act_dgrad_oracle from the stored
    act / gate; the update through rows_update_oracle.  ``samples_of(mu)``: the global sample index of every row of
    micro-batch mu; ``x``: the stage input of the step; ``W0``: the flat weight arena before the step.  bf16 products
    are checked from the rounded operands (test_gpu_residual.operand_model).  Returns {check: max err / bound}."""
    from shallowspeed_b200.ops import functional as F
    from test_gpu_residual import operand_model

    kind, p = model.activation, model.dropout
    op, rtol = operand_model(precision)
    s = F.dropout_scale(p) if p > 0 else 1.0
    L = len(model.linears)
    res, n_dropped, tails = {}, 0, [0, 0]
    upd_dz = [[] for _ in range(L)]
    upd_a = [[] for _ in range(L)]
    blocks = []
    for lin in model.linears:
        blk = W0[model.arena.offsets[lin.block_index]:][: lin.out_dims * model.arena.lds[lin.block_index]]
        blocks.append(blk.view(lin.out_dims, -1)[:, : lin.in_dims + 1].double().cpu())

    def put(k, v):
        res[k] = max(res.get(k, 0.0), v)

    for mu in range(n_mu):
        samples = samples_of(mu)
        # act[0] of the engine is the staging set of the NEXT step; the step's input is x itself
        acts = [x[mu * mb:(mu + 1) * mb].double()] + [eng.act(mu, l).double().cpu() for l in range(1, L + 1)]
        raw = [None] + [eng.act(mu, l).cpu() for l in range(1, L + 1)]
        dzs = [eng.dz(mu, l).double().cpu() for l in range(L + 1)]
        gates = [None] * (L + 1)
        for l, lin in enumerate(model.linears, start=1):
            W, b = blocks[l - 1][:, :-1], blocks[l - 1][:, -1]
            if lin.activation is not None:
                keep = F.dropout_mask(p, model.dropout_seed, lin.dropout[2], step, samples, lin.out_dims) if p > 0 else None
                (ra, ba), gam, z = act_fwd_oracle(kind, op(acts[l - 1]), op(W), b, keep, s, rtol)
                put(f"act{l}", excess(acts[l], ra, ba))
                tails[0] += int((z.abs() > 4).sum())
                tails[1] += int((z.abs() > 9).sum())
                if kind != "relu":
                    gates[l] = eng.gate(mu, l).cpu()
                    put(f"gate{l}", excess(gates[l], *gam))
                if keep is not None:
                    assert int((~keep).sum()) > 0, (mu, l)
                    n_dropped += int((~keep & ((z > 0) if kind == "relu" else (z != 0))).sum())
                    dropped = [raw[l][~keep]] + ([gates[l][~keep]] if gates[l] is not None else [])
                    for t in dropped:
                        assert bool((t.view(torch.int32) == 0).all()), f"mu {mu} layer {l}: a dropped element is not +0"
            else:
                ref, bound = fwd_oracle(op(acts[l - 1]), op(W), b, False, rtol)
                put(f"fwd{l}", excess(acts[l], ref, bound))
            if l >= 2:
                prev = model.linears[l - 2]
                if prev.activation is None:
                    ref, bound = dgrad_oracle(op(dzs[l]), op(W), torch.ones_like(acts[l - 1]), rtol)
                else:
                    ref, bound = act_dgrad_oracle(op(dzs[l]), op(W), kind, acts[l - 1], gates[l - 1], s, rtol)
                    if kind == "relu":
                        assert bool((dzs[l - 1][acts[l - 1] == 0] == 0).all()), (mu, l)
                put(f"dgrad{l}", excess(dzs[l - 1], ref, bound))
            upd_dz[l - 1].append(dzs[l])
            upd_a[l - 1].append(acts[l - 1])
    if p > 0:
        assert n_dropped > 0                     # the masks removed live units: the checks above are not vacuous
    if check_update:
        W1 = model.arena.weights.detach().double().cpu()
        for l, lin in enumerate(model.linears, start=1):
            o, ld = lin.out_dims, model.arena.lds[lin.block_index]
            off = model.arena.offsets[lin.block_index]
            d = (W1[off:off + o * ld] - W0[off:off + o * ld].double().cpu()).view(o, ld)[:, : lin.in_dims + 1]
            if precision == "bf16":
                from test_gpu_bf16 import _update_oracle

                ref, bound = _update_oracle(torch.cat(upd_dz[l - 1]), torch.cat(upd_a[l - 1]), blocks[l - 1], lr)
            else:
                ref, bound = rows_update_oracle(torch.cat(upd_dz[l - 1]), torch.cat(upd_a[l - 1]), blocks[l - 1], lr,
                                                rtol)
            put(f"upd{l}", excess(d, ref, bound))
    kernel = "chain" if eng.uses_chain() else "layer-wise"
    note_worst((kernel, kind, p > 0, precision), res, f"L={L} n_mu={n_mu} mb={mb} step={step}")
    worst = max(res, key=res.get)
    print(f"\n[layers] {kernel} {kind} p={p} {precision} n_mu={n_mu} mb={mb}: max err/bound {res[worst]:.3g} ({worst}); "
          f"|z|>4: {tails[0]}, |z|>9: {tails[1]}; " + " ".join(f"{k}={v:.2g}" for k, v in res.items()))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


# ================================================================================================== GPU side
FAR_BIASES = (12.0, -12.0, 6.0, -6.0)    # features 0..3 of every hidden layer: the tails of f and f' (|z| > 9 and > 4)


def _init_weights(sizes, x, n_mu, gen, activation="relu", far=False):
    """He-scaled weights and non-zero biases (a zero bias would hide a kernel that drops it), with the last layer scaled
    so that the logits of the widest micro-batch span LOGIT_SPREAD through the hidden activation ``activation``.
    ``far``: the first features of every hidden layer get FAR_BIASES."""
    from shallowspeed_b200.ops import functional as F

    Ws, bs = [], []
    for i, o in zip(sizes[:-1], sizes[1:]):
        Ws.append(torch.randn(o, i, generator=gen, dtype=torch.float64) * math.sqrt(2.0 / i))
        bs.append(torch.randn(o, generator=gen, dtype=torch.float64) * 0.1)
    if far:
        for b in bs[:-1]:
            n = min(len(FAR_BIASES), b.numel())
            b[:n] = torch.tensor(FAR_BIASES[:n], dtype=torch.float64)
    a = x.double()
    for l, (W, b) in enumerate(zip(Ws, bs)):
        a = a @ W.T + b
        if l < len(Ws) - 1:
            a = F.activation_ref(activation, a)[0]
    spread = max(float(z.max() - z.min()) for z in a.chunk(n_mu))
    s = LOGIT_SPREAD / spread
    Ws[-1], bs[-1] = Ws[-1] * s, bs[-1] * s
    return [W.float() for W in Ws], [b.float() for b in bs]


def _pitched(view, rows):
    """The whole [rows, ld] extent of an engine buffer whose view is ``view`` (micro-batch 0).  The padding columns of
    the last row lie beyond the storage ``from_blob`` gives the view, so ``as_strided`` cannot reach them; the buffer
    is mapped again through the CUDA array interface."""
    ld = view.stride(0)

    class _Buf:
        __cuda_array_interface__ = {"shape": (rows, ld), "typestr": "<f4", "data": (view.data_ptr(), False),
                                    "version": 3, "strides": None}

    return torch.as_tensor(_Buf(), device=view.device)


def _poison(eng, model, sizes, rows, training, gated=False):
    """NaN into every padding column the kernels must not read: act / dz of l >= 1 in [cols, ld), the gate of every
    activated layer in [cols, ld) when ``gated``, and the weight arena in [in + 1, ld)."""
    for l in range(1, len(sizes)):
        bufs = [eng.act(0, l)] + ([eng.dz(0, l)] if training else [])
        if gated and l < len(sizes) - 1:
            bufs.append(eng.gate(0, l))
        for v in bufs:
            _pitched(v, rows)[:, sizes[l]:] = float("nan")
    for i, (o, k) in enumerate(model.arena.blocks):
        model.arena.block(i)[:, k + 1:] = float("nan")


def _gather(fn, n_mu):
    return torch.cat([fn(mu).double().cpu() for mu in range(n_mu)])


KINDS = ["relu", "gelu", "silu", "tanh"]
DROP_P, DROP_SEED = 0.3, 0xC0FF_EE00_1234_5678


def _run(sizes, mb_rows, n_mu, precision, expect_chain, inference=False, env=(), monkeypatch=None, activation="relu",
         dropout=0.0, loss="mse"):
    """One step at the given shape; returns {check: max err / bound} after asserting the path and non-vacuity.  With a
    smooth ``activation`` or ``dropout`` > 0, every hidden layer has features with far biases, the gate padding is
    poisoned, and the layers are checked per element by ``check_layers``."""
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    for k in env:
        monkeypatch.setenv(k, "1")
    plain = activation == "relu" and dropout == 0.0
    gated = activation != "relu" and not inference
    loss_kind = loss
    L, C, rows = len(sizes) - 1, sizes[-1], mb_rows * n_mu
    gen = torch.Generator().manual_seed(hash((tuple(sizes), mb_rows, n_mu)) & 0xFFFFFFFF)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen, activation, far=not plain)

    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=LR, precision=precision, loss=loss_kind,
                 activation=activation, dropout=dropout, dropout_seed=DROP_SEED)
    model = tr.model
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
    if inference:
        sched = InferenceSchedule(n_mu, 1, 0)
        eng = tr.worker.engine_for(sched)
    else:
        eng = tr.engine
    assert eng.uses_chain() == expect_chain
    if "SSB_NO_COALESCE" in env:
        assert not eng.coalesced()
    _poison(eng, model, sizes, rows, not inference, gated)
    W0 = [model.arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
    W0_flat = model.arena.weights.detach().clone()
    xh, th = x.pin_memory(), t.pin_memory()
    if inference:
        tr.worker.step_from(sched, xh, th)
        eng.synchronize()
        loss = None
    else:
        loss = float(tr.step(xh, th))
    torch.cuda.synchronize()

    act = [x.double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
    probs = _gather(eng.probs, n_mu)
    rtol = RTOL[precision]
    res = {}
    # non-vacuity: a dead network passes any oracle
    for l in range(1, L):
        frac = float((act[l] > 0).double().mean())
        assert 0.05 <= frac <= 0.95, f"layer {l}: {frac:.3f} of the activations are positive"
    if not plain:
        # the tails of f and f' are reached inside the kernel: every activated layer has |z| > 4 and |z| > 9
        for l in range(1, L):
            z = act[l - 1] @ W0[l - 1][:, :-1].T + W0[l - 1][:, -1]
            assert bool((z.abs() > 4).any()) and bool((z.abs() > 9).any()), f"layer {l}: no pre-activation in the tails"
    if plain:
        # forward, every layer from the kernel's own input (act[L] holds the logits: no ReLU)
        for l in range(1, L + 1):
            W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
            ref, bound = fwd_oracle(act[l - 1], W, b, l < L, rtol)
            res[f"fwd{l}"] = excess(act[l], ref, bound)
    elif inference:
        # inference applies f and neither drops nor stores gates
        for l in range(1, L + 1):
            W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
            if l < L:
                (ref, bound), _, _ = act_fwd_oracle(activation, act[l - 1], W, b, None, 1.0, rtol)
            else:
                ref, bound = fwd_oracle(act[l - 1], W, b, False, rtol)
            res[f"fwd{l}"] = excess(act[l], ref, bound)
    # loss head, per micro-batch (MSE: the softmax shift is the micro-batch's global max)
    if loss_kind == "mse":
        head = head_oracle
    else:
        from test_gpu_cross_entropy import ce_head_oracle as head
    dz = None
    if not inference:
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"dz[{l}] is all zero"
    loss_ref = loss_bound = 0.0
    for mu in range(n_mu):
        r = slice(mu * mb_rows, (mu + 1) * mb_rows)
        (p, bp), (g, bg), (lv, bl) = head(act[L][r], t[r], rows, HEAD_RTOL)
        res["probs"] = max(res.get("probs", 0.0), excess(probs[r], p, bp))
        if not inference:
            res["dzL"] = max(res.get("dzL", 0.0), excess(dz[L][r], g, bg))
        loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
    if not inference:
        res["loss"] = abs(loss - loss_ref) / loss_bound if math.isfinite(loss) else math.inf
    if not inference and plain:
        # dgrad chain (layer 1's dgrad is skipped on the first stage)
        for l in range(L, 1, -1):
            ref, bound = dgrad_oracle(dz[l], W0[l - 1][:, :-1], act[l - 1], rtol)
            res[f"dgrad{l}"] = excess(dz[l - 1], ref, bound)
        # SGD update over all micro-batches (grouped wgrad + SGD epilogue)
        for i, (_, k) in enumerate(model.arena.blocks):
            W1 = model.arena.block(i)[:, : k + 1].double().cpu()
            ref, bound = update_oracle(dz[i + 1], act[i], W0[i], LR, rtol)
            res[f"upd{i + 1}"] = excess(W1 - W0[i], ref, bound)
    elif not inference:
        res.update(check_layers(eng, model, W0_flat, x, n_mu, mb_rows, precision, LR,
                                lambda mu: mu * mb_rows + torch.arange(mb_rows)))
    if gated:
        for l in range(1, L):
            pad = _pitched(eng.gate(0, l), rows)[:, sizes[l]:]
            assert bool(pad.isnan().all()), f"layer {l}: a kernel wrote into the gate's padding"
    worst = max(res, key=res.get)
    if not plain:
        note_worst(("chain" if expect_chain else "layer-wise", activation, dropout > 0, precision), res,
                   f"sizes={sizes} mb_rows={mb_rows} env={list(env)} inference={inference}")
    print(f"\n[chain] sizes={sizes} mb_rows={mb_rows} n_mu={n_mu} {precision} chain={expect_chain} env={list(env)} "
          f"inference={inference} {activation} p={dropout} {loss_kind}: max err/bound {res[worst]:.3g} ({worst}); "
          + " ".join(f"{k}={v:.2g}" for k, v in res.items()))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mb_rows", MB_GRID)
def test_chain_micro_batch_sizes(mb_rows, precision):
    _run(BASE, mb_rows, _n_mu(mb_rows), precision, expect_chain=True)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mb_rows", [24, 128])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_chain_widths_depths_classes(shape, mb_rows, precision):
    _run(SHAPES[shape], mb_rows, _n_mu(mb_rows), precision, expect_chain=True)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mb_rows", [24, 128])
@pytest.mark.parametrize("shape", list(FALLBACKS))
def test_layerwise_fallback_shapes(shape, mb_rows, precision):
    _run(FALLBACKS[shape], mb_rows, _n_mu(mb_rows), precision, expect_chain=False)


LAUNCH_FORMS = {"coalesced": (), "per-micro-batch": ("SSB_NO_COALESCE",), "layer-wise": ("SSB_NO_CHAIN",),
                # per-micro-batch weight gradients accumulating in the gradient arena, then a separate SGD pass
                "layer-wise-per-micro-batch": ("SSB_NO_COALESCE", "SSB_NO_CHAIN")}


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(LAUNCH_FORMS))
@pytest.mark.parametrize("mb_rows", [24, 40, 100])                      # NTW 2 / 4 / 8, all with mb_rows % 16 != 0
@pytest.mark.parametrize("sizes", [BASE, SHAPES["straddle-c17"]], ids=["base", "straddle-c17"])
def test_launch_forms(sizes, mb_rows, form, monkeypatch):
    env = LAUNCH_FORMS[form]
    _run(sizes, mb_rows, 2, "fp32", expect_chain="SSB_NO_CHAIN" not in env, env=env, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,mb_rows", [(BASE, 40), (SHAPES["straddle-c17"], 100)])
def test_chain_inference(sizes, mb_rows):
    _run(sizes, mb_rows, 2, "fp32", expect_chain=True, inference=True)


# ---------------------------------------------------------------- the same grid with every activation and dropout
ACT_VARIANTS = [("relu", DROP_P)] + [(k, p) for k in KINDS[1:] for p in (0.0, DROP_P)]


def _act_grid():
    """(sizes, mb_rows, n_mu, precision, launch form, inference, loss) of every case run for each ACT_VARIANTS pair: the
    micro-batch sizes in both precisions, the shapes with a hidden layer (cross-entropy in tf32), the launch forms and
    inference."""
    cases = [(BASE, mb, _n_mu(mb), pr, "coalesced", False, "mse") for mb in MB_GRID for pr in ("fp32", "tf32")]
    cases += [(SHAPES[s], mb, _n_mu(mb), pr, "coalesced", False, "cross_entropy" if pr == "tf32" else "mse")
              for s in SHAPES if len(SHAPES[s]) > 2 for mb in (24, 128) for pr in ("fp32", "tf32")]
    cases += [(BASE, mb, 2, "fp32", form, False, "mse") for form in LAUNCH_FORMS for mb in (24, 40, 100)]
    cases += [(BASE, 40, 2, "fp32", "coalesced", True, "mse"), (SHAPES["straddle-c17"], 100, 2, "fp32", "coalesced", True, "mse")]
    return cases


ACT_GRID = _act_grid()


def _act_case_id(c):
    sizes, mb, _, pr, form, inference, loss = c
    name = next((k for k, v in SHAPES.items() if v == sizes), "base")
    return f"{name}-mb{mb}-{pr}-{form}{'-inference' if inference else ''}{'-ce' if loss != 'mse' else ''}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACT_GRID, ids=[_act_case_id(c) for c in ACT_GRID])
@pytest.mark.parametrize("activation,dropout", ACT_VARIANTS, ids=[f"{k}-{'drop' if p else 'nodrop'}" for k, p in ACT_VARIANTS])
def test_activation_dropout_grid(activation, dropout, case, monkeypatch):
    sizes, mb_rows, n_mu, precision, form, inference, loss = case
    env = LAUNCH_FORMS[form]
    _run(sizes, mb_rows, n_mu, precision, expect_chain="SSB_NO_CHAIN" not in env, inference=inference, env=env,
         monkeypatch=monkeypatch, activation=activation, dropout=dropout, loss=loss)


# ================================================================================================== CPU side
def _chain_geometry(mb_rows):
    """Mirror of the kernel's shape decisions (mlp_chain.cu: chain_warp_cols, chain_launch, the per-warp half split):
    (n_pad, NTW, (n8 tiles of half 0, of half 1))."""
    n_pad = (mb_rows + 15) // 16 * 16
    cols = 16 * ((n_pad // 16 + 1) // 2)
    ntw = 2 if cols <= 16 else 4 if cols <= 32 else 8
    chunks = n_pad // 16
    nts = tuple((16 * ((chunks * (h + 1)) // 2) - 16 * ((chunks * h) // 2)) // 8 for h in (0, 1))
    return n_pad, ntw, nts


def _grid_cases():
    cases = [(BASE, mb) for mb in MB_GRID]
    cases += [(s, mb) for s in SHAPES.values() for mb in (24, 128)]
    cases += [(s, mb) for s in (BASE, SHAPES["straddle-c17"]) for mb in (24, 40, 100)]
    return cases


def test_grid_reaches_every_shape_branch_of_the_chain_kernel():
    from shallowspeed_b200 import _C

    ntws, nts, kps_seen, stage_seen, uneven, ragged, classes, depths = set(), set(), set(), set(), False, False, set(), set()
    for sizes, mb in _grid_cases():
        layers = list(zip(sizes[:-1], sizes[1:]))
        for split in (False, True):
            assert _C.chain_eligible(layers, mb, sizes[-1], True, split), (sizes, mb)
            ok, kps, stages, _smem = _C.chain_budget(mb, split)
            assert ok
            kps_seen.add(kps)
            stage_seen.add(stages)
        _n_pad, ntw, (nt0, nt1) = _chain_geometry(mb)
        assert max(nt0, nt1) <= ntw                       # a warp's block fits its accumulator
        ntws.add(ntw)
        nts |= {nt0, nt1}
        uneven |= nt0 != nt1
        ragged |= mb % 16 != 0
        classes.add(sizes[-1])
        depths.add(len(sizes) - 1)
    assert ntws == {2, 4, 8}
    assert nts == {0, 2, 4, 6, 8}
    assert kps_seen == {4, 2, 1} and {2, 3} <= stage_seen
    assert uneven and ragged
    assert {16, 17, 32} <= classes and min(classes) <= 16      # fast loss head, its edge, the slow one, the maximum
    assert {1, 16} <= depths
    for sizes in FALLBACKS.values():
        layers = list(zip(sizes[:-1], sizes[1:]))
        for mb in (24, 128):
            for split in (False, True):
                assert not _C.chain_eligible(layers, mb, sizes[-1], True, split), sizes


def _selftest_data(seed=0, rows=32, k=128, n=97):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, k, generator=g)
    W = torch.randn(n, k, generator=g) / math.sqrt(k)
    b = torch.randn(n, generator=g) * 0.1
    return x, W, b


def test_checker_rejects_injected_faults():
    """Every fault is applied to an exact fp64 result; the helpers must reject each one and accept the result itself,
    as well as a plain fp32 evaluation (fp32 bounds) and a single-pass TF32 one (tf32 bounds)."""
    x, W, b = _selftest_data()
    rtol = RTOL["fp32"]
    ref, bound = fwd_oracle(x, W, b, False, rtol)
    exact = ref.clone()
    assert excess(exact, ref, bound) <= 1.0
    assert excess(x @ W.T + b, ref, bound) <= 1.0                             # fp32 on the CPU: within the bound
    # one 32-wide k-block dropped
    keep = torch.ones(x.shape[1], dtype=torch.float64)
    keep[32:64] = 0.0
    assert excess((x.double() * keep) @ W.double().T + b.double(), ref, bound) > 1.0
    # the bias missing on one feature
    nob = exact.clone()
    nob[:, 5] -= b[5].double()
    assert excess(nob, ref, bound) > 1.0
    # the micro-batch rows shifted by one (row0 off by one)
    assert excess(torch.roll(exact, -1, dims=0), ref, bound) > 1.0
    # a 3xTF32 result replaced by its single-pass TF32 evaluation: rejected by the fp32 bound, accepted by tf32's
    single = tf32_trunc(x).double() @ tf32_trunc(W).double().T + b.double()
    assert excess(single, ref, bound) > 1.0
    assert excess(single, *fwd_oracle(x, W, b, False, RTOL["tf32"])) <= 1.0

    # one ReLU mask element flipped in the dgrad (the mask comes from the stored activation)
    g = torch.Generator().manual_seed(1)
    dz = torch.randn(32, 97, generator=g) * 1e-3
    act_prev = torch.randn(32, 128, generator=g).clamp_min(0.0)
    dref, dbound = dgrad_oracle(dz, W, act_prev, rtol)
    assert excess(dref, dref, dbound) <= 1.0
    i, j = (act_prev > 0).nonzero()[0].tolist()
    flipped = dref.clone()
    flipped[i, j] = 0.0
    assert excess(flipped, dref, dbound) > 1.0
    i, j = (act_prev == 0).nonzero()[0].tolist()
    flipped = dref.clone()
    flipped[i, j] = float(dz[i].double() @ W[:, j].double())
    assert excess(flipped, dref, dbound) > 1.0

    # probabilities computed with a per-row max shift instead of the micro-batch's global max
    from shallowspeed_b200.ops.functional import SOFTMAX_EPS

    z = torch.randn(32, 10, generator=g, dtype=torch.float64)
    z = z * (LOGIT_SPREAD / float(z.max() - z.min()))
    t = torch.nn.functional.one_hot(torch.randint(0, 10, (32,), generator=g), 10).double()
    (p, bp), (dzl, bdz), (loss, bl) = head_oracle(z, t, 64, HEAD_RTOL)
    assert excess(p, p, bp) <= 1.0 and excess(dzl, dzl, bdz) <= 1.0
    e = torch.exp(z.float() - z.float().max())                              # the contract, in fp32: accepted
    p32 = e / (e.sum(1, keepdim=True) + SOFTMAX_EPS)
    assert excess(p32, p, bp) <= 1.0
    er = torch.exp(z - z.max(1, keepdim=True).values)
    assert excess(er / (er.sum(1, keepdim=True) + SOFTMAX_EPS), p, bp) > 1.0

    # the update: a dropped k-block of the row sum (rows of one micro-batch missing) is rejected, exact accepted
    a_prev = torch.randn(64, 128, generator=g).clamp_min(0.0)
    dzu = torch.randn(64, 97, generator=g) * 1e-3
    W0 = torch.cat([W, b[:, None]], dim=1)
    d, bd = update_oracle(dzu, a_prev, W0, LR, rtol)
    assert excess(d, d, bd) <= 1.0
    d_half, _ = update_oracle(dzu[:32], a_prev[:32], W0, LR, rtol)
    assert excess(d_half, d, bd) > 1.0


def test_activation_grid_reaches_every_form_for_every_variant():
    """Every (activation, dropout) pair of the grid reaches NTW 2 / 4 / 8, ragged micro-batches, the k-split cluster and
    the one-CTA chain, per-micro-batch launches, the layer-wise fallback, inference and both losses."""
    from shallowspeed_b200 import _C

    assert {k for k, _ in ACT_VARIANTS} == set(KINDS)
    assert {(k, p > 0) for k, p in ACT_VARIANTS} == {(k, d) for k in KINDS for d in (False, True)} - {("relu", False)}
    seen = {"ntw": set(), "ragged": False, "ksplit": False, "one-cta": False, "forms": set(), "losses": set(),
            "inference": False, "precisions": set()}
    for sizes, mb, _n, pr, form, inference, loss in ACT_GRID:
        layers = list(zip(sizes[:-1], sizes[1:]))
        seen["forms"].add(form)
        seen["losses"].add(loss)
        seen["inference"] |= inference
        seen["precisions"].add(pr)
        if "SSB_NO_CHAIN" in LAUNCH_FORMS[form]:
            continue
        assert _C.chain_eligible(layers, mb, sizes[-1], True, pr == "fp32"), (sizes, mb)
        seen["ntw"].add(_chain_geometry(mb)[1])
        seen["ragged"] |= mb % 16 != 0
        c = _C.chain_cluster_size(layers, True, True, True, True, False, False)
        assert _C.chain_cluster_budget(mb, c, pr == "fp32")[0] if c > 1 else True
        seen["one-cta"] |= c == 1
        seen["ksplit"] |= c > 1 and -(-sizes[0] // 32) > 4              # test_gpu_chain_ksplit: > 4 k-blocks
    assert seen["ntw"] == {2, 4, 8} and seen["ragged"] and seen["ksplit"] and seen["one-cta"]
    assert seen["forms"] == set(LAUNCH_FORMS) and seen["losses"] == {"mse", "cross_entropy"} and seen["inference"]
    assert seen["precisions"] == {"fp32", "tf32"}


def _device_formulas_fp32(kind, z):
    """ptx.cuh: act_fwd evaluated op by op in fp32 on the CPU (torch's erf / exp / tanh instead of the CUDA Math API)."""
    z = z.float()
    if kind == "gelu":
        c = 0.5 * (1.0 + torch.erf(z * 0.70710678118654752))
        return z * c, c + z * (torch.exp(-0.5 * z * z) * 0.39894228040143268)
    if kind == "silu":
        s = 1.0 / (1.0 + torch.exp(-z))
        return z * s, s * (1.0 + z * (1.0 - s))
    t = torch.tanh(z)
    return t, 1.0 - t * t


def test_activation_oracles_reject_injected_faults():
    """The activated-layer oracles accept the exact result and an fp32 evaluation of the device formulas, and reject:
    the tanh-approximate GELU, a GELU gate without its z phi(z) term, a gate without keep * s, a dgrad element without
    the dropout scale, one mask element drawn for the wrong sample or step, a gate shifted by one row, an update without
    its bias column.  All against the fp32 bounds; the tf32 bounds reject the same faults except where noted."""
    from shallowspeed_b200.ops import functional as F

    g = torch.Generator().manual_seed(11)
    rows, k, n = 32, 64, 48
    x = torch.randn(rows, k, generator=g)
    W = torch.randn(n, k, generator=g) * math.sqrt(2.0 / k)
    b = torch.randn(n, generator=g) * 0.1
    b[:4] = torch.tensor(FAR_BIASES)
    s = F.dropout_scale(DROP_P)
    samples = 3 + torch.arange(rows) * 2 + 1                      # row_base 3, dp 2, rank 1
    keep = F.dropout_mask(DROP_P, DROP_SEED, 5, 7, samples, n)
    kf = keep.double()
    for precision in ("fp32", "tf32"):
        rtol = RTOL[precision]
        strict = precision == "fp32"
        for kind in KINDS[1:]:
            (ra, ba), (rg, bg), z = act_fwd_oracle(kind, x, W, b, keep, s, rtol)
            assert excess(ra, ra, ba) <= 1.0 and excess(rg, rg, bg) <= 1.0
            # the device formulas in fp32 from an fp32 z: accepted
            a32, g32 = _device_formulas_fp32(kind, (x @ W.T + b))
            keep32 = keep.float()
            assert excess(a32 * s * keep32, ra, ba) <= 1.0 and excess(g32 * s * keep32, rg, bg) <= 1.0
            # gate without keep * s: rejected in both precisions
            assert excess(g32.double(), rg, bg) > 1.0
            # one mask element from the wrong sample (row_base off by one) or the wrong step
            for wrong in (F.dropout_mask(DROP_P, DROP_SEED, 5, 7, samples + 2, n),
                          F.dropout_mask(DROP_P, DROP_SEED, 5, 8, samples, n)):
                i, j = ((wrong != keep) & (a32.abs() > 0.1)).nonzero()[0].tolist()
                bad = a32 * s * keep32
                bad[i, j] = (a32[i, j] * s) if wrong[i, j] else 0.0
                assert excess(bad, ra, ba) > 1.0, (kind, precision)
            # a gate shifted by one row
            assert excess(torch.roll(g32 * s * keep32, 1, dims=0), rg, bg) > 1.0
        # GELU: the tanh approximation, and the gate without z phi(z)
        (ra, ba), (rg, bg), z = act_fwd_oracle("gelu", x, W, b, None, 1.0, rtol)
        z32 = (x @ W.T + b)
        approx = torch.nn.functional.gelu(z32.double(), approximate="tanh")
        if strict:                                                     # tf32's bound is wider than its 5e-4 difference
            assert excess(approx, ra, ba) > 1.0
        Phi = 0.5 * torch.special.erfc(-z / _SQRT2)
        assert excess(Phi, rg, bg) > 1.0

    rtol = RTOL["fp32"]
    # dgrad through ReLU + dropout: the scale missing on one kept element
    dz = torch.randn(rows, n, generator=g) * 1e-2
    W2 = torch.randn(n, k, generator=g) / math.sqrt(n)
    act_prev = torch.where(torch.rand(rows, k, generator=g) < 0.7, torch.rand(rows, k, generator=g), torch.zeros(()))
    ref, bound = act_dgrad_oracle(dz, W2, "relu", act_prev, None, s, rtol)
    got = ((dz @ W2) * (act_prev > 0) * s).double()
    assert excess(got, ref, bound) <= 1.0
    i, j = (act_prev > 0).nonzero()[0].tolist()
    got[i, j] /= s
    assert excess(got, ref, bound) > 1.0
    # dgrad through a gate: the gate shifted by one row
    gam = torch.rand(rows, k, generator=g) * s * (act_prev > 0)
    ref, bound = act_dgrad_oracle(dz, W2, "gelu", None, gam, s, rtol)
    assert excess((dz @ W2) * gam, ref, bound) <= 1.0
    assert excess((dz.double() @ W2.double()) * torch.roll(gam, 1, dims=0).double(), ref, bound) > 1.0

    # the update without its bias column (1024 rows: the bias bound carries its per-row roundings)
    dzu = torch.randn(1024, n, generator=g) * 1e-3
    au = torch.randn(1024, k, generator=g).clamp_min(0.0)
    W0 = torch.cat([W, b[:, None]], 1)
    for precision in ("fp32", "tf32"):
        d, bd = rows_update_oracle(dzu, au, W0, LR, RTOL[precision])
        assert excess(d, d, bd) <= 1.0
        nob = d.clone()
        nob[:, -1] = 0.0
        assert excess(nob, d, bd) > 1.0
