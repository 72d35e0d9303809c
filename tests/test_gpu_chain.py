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


# ================================================================================================== GPU side
def _init_weights(sizes, x, n_mu, gen):
    """He-scaled weights and non-zero biases (a zero bias would hide a kernel that drops it), with the last layer scaled
    so that the logits of the widest micro-batch span LOGIT_SPREAD."""
    Ws, bs = [], []
    for i, o in zip(sizes[:-1], sizes[1:]):
        Ws.append(torch.randn(o, i, generator=gen, dtype=torch.float64) * math.sqrt(2.0 / i))
        bs.append(torch.randn(o, generator=gen, dtype=torch.float64) * 0.1)
    a = x.double()
    for l, (W, b) in enumerate(zip(Ws, bs)):
        a = a @ W.T + b
        if l < len(Ws) - 1:
            a = a.clamp_min(0.0)
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


def _poison(eng, model, sizes, rows, training):
    """NaN into every padding column the kernels must not read: act / dz of l >= 1 in [cols, ld) and the weight arena
    in [in + 1, ld)."""
    for l in range(1, len(sizes)):
        bufs = [eng.act(0, l)] + ([eng.dz(0, l)] if training else [])
        for v in bufs:
            _pitched(v, rows)[:, sizes[l]:] = float("nan")
    for i, (o, k) in enumerate(model.arena.blocks):
        model.arena.block(i)[:, k + 1:] = float("nan")


def _gather(fn, n_mu):
    return torch.cat([fn(mu).double().cpu() for mu in range(n_mu)])


def _run(sizes, mb_rows, n_mu, precision, expect_chain, inference=False, env=(), monkeypatch=None):
    """One step at the given shape; returns {check: max err / bound} after asserting the path and non-vacuity."""
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    for k in env:
        monkeypatch.setenv(k, "1")
    L, C, rows = len(sizes) - 1, sizes[-1], mb_rows * n_mu
    gen = torch.Generator().manual_seed(hash((tuple(sizes), mb_rows, n_mu)) & 0xFFFFFFFF)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen)

    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=LR, precision=precision)
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
    _poison(eng, model, sizes, rows, not inference)
    W0 = [model.arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
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
    # forward, every layer from the kernel's own input (act[L] holds the logits: no ReLU)
    for l in range(1, L + 1):
        W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
        ref, bound = fwd_oracle(act[l - 1], W, b, l < L, rtol)
        res[f"fwd{l}"] = excess(act[l], ref, bound)
    # loss head, per micro-batch (the softmax shift is the micro-batch's global max)
    dz = None
    if not inference:
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"dz[{l}] is all zero"
    loss_ref = loss_bound = 0.0
    for mu in range(n_mu):
        r = slice(mu * mb_rows, (mu + 1) * mb_rows)
        (p, bp), (g, bg), (lv, bl) = head_oracle(act[L][r], t[r], rows, HEAD_RTOL)
        res["probs"] = max(res.get("probs", 0.0), excess(probs[r], p, bp))
        if not inference:
            res["dzL"] = max(res.get("dzL", 0.0), excess(dz[L][r], g, bg))
        loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
    if not inference:
        res["loss"] = abs(loss - loss_ref) / loss_bound if math.isfinite(loss) else math.inf
        # dgrad chain (layer 1's dgrad is skipped on the first stage)
        for l in range(L, 1, -1):
            ref, bound = dgrad_oracle(dz[l], W0[l - 1][:, :-1], act[l - 1], rtol)
            res[f"dgrad{l}"] = excess(dz[l - 1], ref, bound)
        # SGD update over all micro-batches (grouped wgrad + SGD epilogue)
        for i, (_, k) in enumerate(model.arena.blocks):
            W1 = model.arena.block(i)[:, : k + 1].double().cpu()
            ref, bound = update_oracle(dz[i + 1], act[i], W0[i], LR, rtol)
            res[f"upd{i + 1}"] = excess(W1 - W0[i], ref, bound)
    worst = max(res, key=res.get)
    print(f"\n[chain] sizes={sizes} mb_rows={mb_rows} n_mu={n_mu} {precision} chain={expect_chain} env={list(env)} "
          f"inference={inference}: max err/bound {res[worst]:.3g} ({worst}); "
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
