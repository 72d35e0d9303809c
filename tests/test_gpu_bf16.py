"""``precision="bf16"`` per element against fp64: the stand-alone GEMMs, the chain kernel in each launch form, the grouped
weight gradient and its update, and the engine-level properties.

Every reference is computed from the operands rounded to bf16 (``Tensor.bfloat16()``: round to nearest even, as
``cvt.rn.bf16x2.f32`` in ptx.cuh: warp_mma_kblock).  Two bf16 values multiply exactly in fp32, so the only error left is
the accumulation, and the bound is test_gpu_chain's 3xTF32 class:

    |got - ref| <= RTOL_BF16 * (|a'| @ |b'|) + ATOL,   RTOL_BF16 = 2^-16         (a', b': the rounded operands)

plus test_gpu_gemm's extra fp32 rounding per k-block and split partial for K > 4096 (``rtol_bf16``).  Everything else is
fp32 and keeps its own bound: the bias (added unrounded in the epilogue), the loss head, the activations, and the bias
gradient, an fp32 column sum of the UNROUNDED dZ.  A tf32 or 3xTF32 result is off from these references by the bf16
rounding of its operands (up to 2^-9 of each), far outside the bound; ``test_tf32_fails_the_bf16_oracle`` checks that.

Worst err / bound, measured on an H100 80GB HBM3 (700 W power limit), the ``[bf16] worst`` table this file prints (-s):
the products 0.006 (stand-alone FWD / DGRAD / WGRAD, split-K included), 0.011 (chain forward), 0.015 (chain dgrad),
0.0074 (layer-wise engine); the update 0.49 and the fused SGD 0.37, which is the fp32 rounding of the stored weight (2^-24
of it against 2^-23 in the bound), as in fp32.  Hopper's BF16 accumulation sits far inside the 3xTF32 class, so the bound
needs no term of its own.  The same data in tf32 or fp32 reach 116 to 354 (``test_tf32_fails_the_bf16_oracle``).
"""
import math

import pytest
import torch

from test_gpu_chain import (ATOL, BASE, DROP_P, DROP_SEED, FP32_ULP, HEAD_RTOL, LR, MB_GRID, SHAPES,
                            _init_weights, _n_mu, _poison, act_dgrad_oracle, act_fwd_oracle, dgrad_oracle, excess,
                            fwd_oracle, head_oracle)
from test_gpu_gemm import GRID, NAN, SENTINEL, _gen, _ld, _mask_values, _out, _pitched

pytestmark = pytest.mark.gpu

RTOL_BF16 = 2.0**-16
U = 2.0**-24
WORST = {}                    # kernel -> (worst err / bound of the session, where)


def rtol_bf16(k, splits=1):
    """RTOL_BF16, plus one fp32 rounding per k-block sum and per split partial for K > 4096 (as test_gpu_gemm.rtol_for)."""
    return RTOL_BF16 + ((math.ceil(k / 32) + splits) * U if k > 4096 else 0.0)


def bf(t):
    """The operand the tensor core multiplies: fp32 rounded to bf16 (nearest even), as fp64."""
    return t.float().cpu().bfloat16().double()


def grad_oracle_bf16(dz, x, rtol):
    """test_gpu_gemm.grad_oracle on the bf16-rounded operands: ``[bf(dz).T @ bf(x) | colsum(dz)]`` in fp64, the bias
    column summed from the UNROUNDED dz in fp32 (one rounding per row).  Called with rtol 0.0 for a magnitude only."""
    dz, x = dz.double(), x.double()
    dzr, xr = bf(dz), bf(x)
    g = torch.cat([dzr.T @ xr, dz.sum(0)[:, None]], dim=1)
    mag = torch.cat([dzr.abs().T @ xr.abs(), dz.abs().sum(0)[:, None]], dim=1)
    bound = rtol * mag + ATOL
    bound[:, -1] += dz.shape[0] * U * mag[:, -1]
    return g, bound


def _note(kernel, res, what):
    v = max(res.values()) if res else 0.0
    if v > WORST.get(kernel, (-1.0, ""))[0]:
        WORST[kernel] = (v, what)
    print(f"\n[bf16] {kernel} {what}: max err/bound {v:.3g} (" + " ".join(f"{k}={x:.2g}" for k, x in res.items()) + ")")
    bad = {k: x for k, x in res.items() if not x <= 1.0}
    assert not bad, (kernel, what, bad)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    print()
    for kernel, (v, what) in sorted(WORST.items()):
        print(f"[bf16] worst err/bound {kernel:>14}: {v:.3g} at {what}")


def _K():
    from shallowspeed_b200.ops import cuda as K

    return K


# ================================================================================================== stand-alone GEMMs
@pytest.mark.parametrize("rows,m,k", GRID)
def test_fwd_dgrad_per_element(rows, m, k):
    """FWD (bias, ReLU) and DGRAD (mask) at test_gpu_gemm's tile edges, plain and with the planner's split-K where it
    splits, each split-K launch three times bit-identical."""
    from shallowspeed_b200 import _C

    K = _K()
    gen = _gen("bf16-fwd", rows, m, k)
    _, x = _pitched(rows, k, gen)
    wbuf, _ = _pitched(m, k + 1, gen, scale=1.0 / math.sqrt(k))
    wbuf[:, k] = torch.randn(m, generator=gen).cuda() * 0.5
    W, b = wbuf[:, :k], wbuf[:, k]
    _, dz = _pitched(rows, k, gen)
    _, Wd = _pitched(k, m, gen, scale=1.0 / math.sqrt(k))
    mbuf = torch.full((rows, _ld(m, 8)), NAN)
    mbuf[:, :m] = _mask_values(rows, m, gen)
    mask = mbuf.cuda()[:, :m]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    planner = _C.splitk_plan(m, rows, k, sms, 0)[0]
    res = {}
    for ks in (0, -1) if planner >= 2 else (0,):
        splits = planner if ks == -1 else 1
        for relu in (False, True):
            ybuf, y = _out(rows, m)
            K.linear_fwd(x, W, b, relu=relu, out=y, precision="bf16", k_splits=ks)
            torch.cuda.synchronize()
            ref, bound = fwd_oracle(bf(x), bf(W), b.cpu(), relu, rtol_bf16(k, splits))
            res[f"fwd-relu{int(relu)}-ks{ks}"] = excess(y, ref, bound)
            assert bool((ybuf[:, m:] == SENTINEL).all()), "FWD wrote into the output's padding"
        outs = []
        for _ in range(3 if ks else 1):
            dxbuf, dx = _out(rows, m)
            K.linear_dgrad(dz, Wd, mask=mask, out=dx, precision="bf16", k_splits=ks)
            torch.cuda.synchronize()
            outs.append(dx.cpu().contiguous().view(torch.int32))
            assert bool((dxbuf[:, m:] == SENTINEL).all()), "DGRAD wrote into the output's padding"
        ref, bound = dgrad_oracle(bf(dz), bf(Wd), mask.cpu(), rtol_bf16(k, splits))
        res[f"dgrad-ks{ks}"] = excess(outs[0].view(torch.float32), ref, bound)
        assert all(torch.equal(outs[0], o) for o in outs), f"k_splits={ks} is not deterministic"
    _note("fwd/dgrad", res, f"rows={rows} m={m} k={k} planner={planner}")


def _update_oracle(dz, a, W0, lr):
    """SGD step ``-lr * [bf(dz).T @ bf(a) | colsum(dz)]`` and its bound: the products of the rounded operands within
    RTOL_BF16, the bias column the fp32 column sum of the UNROUNDED dZ (one rounding per row), and one fp32 ulp of the
    weights for the stored result.  W0: the [out, in + 1] block before the step."""
    dz, a, W0 = dz.double().cpu(), a.double().cpu(), W0.double().cpu()
    dzr, ar = bf(dz), bf(a)
    d = -lr * torch.cat([dzr.T @ ar, dz.sum(0)[:, None]], dim=1)
    mag = abs(lr) * torch.cat([dzr.abs().T @ ar.abs(), dz.abs().sum(0)[:, None]], dim=1)
    bound = rtol_bf16(dz.shape[0]) * mag + FP32_ULP * (W0.abs() + d.abs()) + ATOL
    bound[:, -1] += dz.shape[0] * U * mag[:, -1]
    return d, bound


@pytest.mark.parametrize("rows,n_in,out", [(1, 5, 300), (32, 127, 126), (33, 65, 129), (128, 777, 200),
                                           (512, 64, 33), (2, 4, 1000), (100, 4096, 64)])
def test_wgrad_and_fused_sgd_per_element(rows, n_in, out):
    """WGRAD into G with the bias column, and the same product fused into the SGD update of the arena block."""
    K = _K()
    gen = _gen("bf16-wgrad", rows, n_in, out)
    _, dz = _pitched(rows, out, gen)
    _, x = _pitched(rows, n_in, gen)
    ld = _ld(n_in + 1)
    gbuf = torch.full((out, ld), SENTINEL, device="cuda")
    K.linear_wgrad(dz, x, gbuf[:, :n_in], grad_b=gbuf[:, n_in], precision="bf16")
    wbuf = torch.full((out, ld), NAN)
    wbuf[:, : n_in + 1] = torch.randn(out, n_in + 1, generator=gen)
    wbuf = wbuf.cuda()
    w0 = wbuf.cpu()
    g2 = torch.empty_like(wbuf)
    K.linear_wgrad(dz, x, g2[:, :n_in], grad_b=g2[:, n_in], weight=wbuf[:, :n_in], lr=0.25, fuse_sgd=True,
                   precision="bf16")
    torch.cuda.synchronize()
    res = {}
    d, bound = _update_oracle(dz, x, torch.zeros(out, n_in + 1), -1.0)   # lr = -1: the gradient itself
    res["G"] = excess(gbuf[:, :n_in], d[:, :n_in], bound[:, :n_in])
    res["db"] = excess(gbuf[:, n_in], d[:, n_in], bound[:, n_in])
    d, bound = _update_oracle(dz, x, w0[:, : n_in + 1], 0.25)
    res["sgd"] = excess(wbuf.cpu()[:, : n_in + 1] - w0[:, : n_in + 1].double(), d, bound)
    _note("wgrad/sgd", res, f"rows={rows} in={n_in} out={out}")


# ================================================================================================== the engine
def _step(sizes, mb_rows, n_mu, precision="bf16", activation="relu", dropout=0.0, loss="mse", inference=False,
          env=(), monkeypatch=None, seed=0):
    """One Trainer step (or an inference pass) at the given shape; returns (engine, model, x, t, W0 blocks, W0 arena,
    loss)."""
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    for k in env:
        monkeypatch.setenv(k, "1")
    rows = mb_rows * n_mu
    gen = torch.Generator().manual_seed(hash((tuple(sizes), mb_rows, n_mu, seed)) & 0xFFFFFFFF)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen, activation, far=activation != "relu" or dropout > 0)
    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=LR, precision=precision, loss=loss,
                 activation=activation, dropout=dropout, dropout_seed=DROP_SEED)
    model = tr.model
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
    sched = InferenceSchedule(n_mu, 1, 0) if inference else None
    eng = tr.worker.engine_for(sched) if inference else tr.engine
    _poison(eng, model, sizes, rows, not inference, activation != "relu" and not inference)
    W0 = [model.arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
    xh, th = x.pin_memory(), t.pin_memory()
    if inference:
        tr.worker.step_from(sched, xh, th)
        eng.synchronize()
        lv = None
    else:
        lv = float(tr.step(xh, th))
    torch.cuda.synchronize()
    return tr, eng, x, t, W0, lv


def check_bf16(tr, eng, x, t, W0, loss_value, mb_rows, n_mu, inference=False):
    """Every layer of the step per micro-batch and per element against the bf16 oracle, each from the engine's own
    buffers: forward products (through act_fwd_oracle for the activated layers, with the dropout masks), the loss head
    (fp32, HEAD_RTOL), the dgrads (the masks and gates as stored), and the update of every layer.  Returns
    {check: max err / bound}."""
    from shallowspeed_b200.ops import functional as F

    model = tr.model
    kind, p = model.activation, (0.0 if inference else model.dropout)
    s = F.dropout_scale(p) if p > 0 else 1.0
    L, rows = len(model.linears), mb_rows * n_mu
    res = {}

    def put(k, v):
        res[k] = max(res.get(k, 0.0), v)

    if model.loss == "mse":
        head = head_oracle
    else:
        from test_gpu_cross_entropy import ce_head_oracle as head
    upd_dz, upd_a = [[] for _ in range(L)], [[] for _ in range(L)]
    loss_ref = loss_bound = 0.0
    for mu in range(n_mu):
        r = slice(mu * mb_rows, (mu + 1) * mb_rows)
        samples = mu * mb_rows + torch.arange(mb_rows)
        acts = [x[r].double()] + [eng.act(mu, l).double().cpu() for l in range(1, L + 1)]
        dzs = [None] + ([eng.dz(mu, l).double().cpu() for l in range(1, L + 1)] if not inference else [None] * L)
        gates = [None] * (L + 1)
        for l, lin in enumerate(model.linears, start=1):
            W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
            if lin.activation is not None:
                keep = F.dropout_mask(p, model.dropout_seed, lin.dropout[2], 0, samples, lin.out_dims) if p > 0 else None
                (ra, ba), gam, _ = act_fwd_oracle(kind, bf(acts[l - 1]), bf(W), b, keep, s, RTOL_BF16)
                put(f"act{l}", excess(acts[l], ra, ba))
                if kind != "relu" and not inference:
                    gates[l] = eng.gate(mu, l).cpu()
                    put(f"gate{l}", excess(gates[l], *gam))
            else:
                ref, bound = fwd_oracle(bf(acts[l - 1]), bf(W), b, False, RTOL_BF16)
                put(f"fwd{l}", excess(acts[l], ref, bound))
            if not inference and l >= 2:
                prev = model.linears[l - 2]
                if prev.activation is None:
                    ref, bound = dgrad_oracle(bf(dzs[l]), bf(W), torch.ones_like(acts[l - 1]), RTOL_BF16)
                else:
                    ref, bound = act_dgrad_oracle(bf(dzs[l]), bf(W), kind, acts[l - 1], gates[l - 1], s, RTOL_BF16)
                put(f"dgrad{l}", excess(dzs[l - 1], ref, bound))
            upd_dz[l - 1].append(dzs[l])
            upd_a[l - 1].append(acts[l - 1])
        (pr, bp), (g, bg), (lv, bl) = head(acts[L], t[r], rows, HEAD_RTOL)
        put("probs", excess(eng.probs(mu).cpu(), pr, bp))
        if not inference:
            put("dzL", excess(dzs[L], g, bg))
        loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
    if not inference:
        res["loss"] = abs(loss_value - loss_ref) / loss_bound if math.isfinite(loss_value) else math.inf
        for l in range(1, L + 1):
            W1 = model.arena.block(l - 1)[:, : model.linears[l - 1].in_dims + 1].double().cpu()
            ref, bound = _update_oracle(torch.cat(upd_dz[l - 1]), torch.cat(upd_a[l - 1]), W0[l - 1], LR)
            put(f"upd{l}", excess(W1 - W0[l - 1], ref, bound))
    return res


def _chain_case(sizes, mb_rows, n_mu, what, **kw):
    tr, eng, x, t, W0, lv = _step(sizes, mb_rows, n_mu, **kw)
    assert eng.uses_chain()
    res = check_bf16(tr, eng, x, t, W0, lv, mb_rows, n_mu, inference=kw.get("inference", False))
    _note("chain" if not kw.get("inference") else "chain-infer", res, what)
    return eng


@pytest.mark.parametrize("mb_rows", MB_GRID)
def test_chain_micro_batch_sizes(mb_rows):
    """The reference-like BASE model: the cluster form with the k-split layer 1 (784 inputs)."""
    eng = _chain_case(BASE, mb_rows, _n_mu(mb_rows), f"BASE mb={mb_rows}")
    assert (eng.chain_cluster(), eng.chain_ksplit()) == (4, 2)


# one CTA per micro-batch (narrow), a cluster without k-split (128 inputs), the widest heads and the deepest chain
FORMS = {"one-cta": ([33, 32, 31, 17], (1, 1)), "one-cta-k784": ([784, 32, 24, 10], (1, 1)),
         "cluster": ([128, 128, 97, 33, 10], (4, 1)), "c32-k4096": (SHAPES["c32-k4096"], None),
         "depth16": (SHAPES["depth16"], None), "tiny": (SHAPES["tiny"], None)}


@pytest.mark.parametrize("mb_rows", [24, 128])
@pytest.mark.parametrize("form", list(FORMS))
def test_chain_launch_forms_and_shapes(form, mb_rows):
    sizes, cp = FORMS[form]
    eng = _chain_case(sizes, mb_rows, _n_mu(mb_rows), f"{form} mb={mb_rows}")
    if cp is not None:
        assert (eng.chain_cluster(), eng.chain_ksplit()) == cp


@pytest.mark.parametrize("mb_rows", [24, 40, 100])
def test_chain_per_micro_batch_launches(mb_rows, monkeypatch):
    _chain_case(BASE, mb_rows, 2, f"per-micro-batch mb={mb_rows}", env=("SSB_NO_COALESCE",), monkeypatch=monkeypatch)


@pytest.mark.parametrize("variant", ["cross_entropy", "gelu+drop", "silu", "tanh+drop", "relu+drop"])
@pytest.mark.parametrize("sizes", [BASE, [33, 32, 31, 17]], ids=["ksplit", "one-cta"])
def test_chain_heads_activations_dropout(sizes, variant):
    kw = {"loss": "cross_entropy"} if variant == "cross_entropy" else {}
    kind = variant.split("+")[0]
    if variant != "cross_entropy":
        kw.update(activation=kind, dropout=DROP_P if variant.endswith("+drop") else 0.0)
    _chain_case(sizes, 40, 2, f"{variant} sizes={sizes}", **kw)


@pytest.mark.parametrize("sizes,mb_rows", [(BASE, 40), ([33, 32, 31, 17], 100), ([128, 128, 97, 33, 10], 24)])
def test_chain_inference(sizes, mb_rows):
    _chain_case(sizes, mb_rows, 2, f"inference sizes={sizes} mb={mb_rows}", inference=True)


@pytest.mark.parametrize("sizes", [[784, 129, 10], [100] + [40] * 16 + [10]], ids=["too-wide", "depth17"])
def test_layerwise_fallback(sizes):
    tr, eng, x, t, W0, lv = _step(sizes, 32, 2)
    assert not eng.uses_chain()
    _note("layer-wise", check_bf16(tr, eng, x, t, W0, lv, 32, 2), f"sizes={sizes}")


def test_tf32_fails_the_bf16_oracle():
    """Non-vacuity: the same data run in tf32 and in fp32 (3xTF32) fail the bf16 oracle in every GEMM kind."""
    for precision in ("tf32", "fp32"):
        tr, eng, x, t, W0, lv = _step(BASE, 40, 2, precision=precision)
        res = check_bf16(tr, eng, x, t, W0, lv, 40, 2)
        worst = {k: max(v for c, v in res.items() if c.startswith(k)) for k in ("fwd", "act", "dgrad", "upd")}
        print(f"\n[bf16] {precision} against the bf16 oracle: " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
        assert all(v > 1.0 for v in worst.values()), (precision, worst)
    K = _K()
    gen = _gen("bf16-nonvacuous")
    _, a = _pitched(64, 300, gen)
    _, W = _pitched(100, 300, gen, scale=300 ** -0.5)
    bias = torch.zeros(100)
    for precision in ("tf32", "fp32"):
        _, y = _out(64, 100)
        K.linear_fwd(a, W, None, out=y, precision=precision)
        torch.cuda.synchronize()
        assert excess(y, *fwd_oracle(bf(a), bf(W), bias, False, RTOL_BF16)) > 1.0, precision


# ================================================================================================== engine properties
def test_two_runs_are_bit_identical():
    outs = []
    for _ in range(2):
        tr, eng, x, t, W0, lv = _step(BASE, 32, 4)
        outs.append((lv, tr.model.arena.weights.detach().cpu().view(torch.int32).clone()))
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("sizes", [BASE, [784, 97, 65, 31, 1, 32], [4096, 128, 33, 64, 127, 10]],
                         ids=lambda s: "-".join(map(str, s)))
def test_plan_matches_fp32(sizes):
    """bf16 changes the products only: the same launches, chain form and kernel count as the fp32 plan."""
    from shallowspeed_b200.parallel.engine import Trainer

    got = []
    for precision in ("fp32", "bf16"):
        tr = Trainer(sizes, global_batch_size=128, n_mubatches=4, lr=0.01, precision=precision)
        eng = tr.engine
        got.append((tr.worker.kernels_per_step(tr.schedule), eng.uses_chain(), eng.chain_cluster(), eng.chain_ksplit(),
                    eng.plan_text(0)))
    assert got[0] == got[1]


@pytest.mark.parametrize("opt", ["sgd", "momentum_wd"])
@pytest.mark.parametrize("rows", [8, 100, 512])
@pytest.mark.parametrize("sizes", [[4096, 128, 33, 64, 127, 10], [784, 97, 65, 31, 1, 32]],
                         ids=lambda s: "-".join(map(str, s)))
def test_grouped_wgrad_equals_the_per_layer_kernel(sizes, rows, opt):
    """The grouped launch on its narrow tiles equals the stand-alone per-layer kernel bit for bit in bf16 (the k-block
    sums are the same instructions on the same operands), as test_gpu_wgrad_group_tiles checks in tf32 and fp32."""
    import test_gpu_wgrad_group_tiles as G

    monkey = pytest.MonkeyPatch()
    try:
        monkey.setattr(G, "STEPS", 2)
        G.test_grouped_narrow_tiles_equal_the_stand_alone_per_layer_kernel(sizes, rows, "bf16", opt)
    finally:
        monkey.undo()


def test_unknown_precision_names_raise():
    from shallowspeed_b200.parallel.engine import Trainer

    with pytest.raises(ValueError):
        Trainer([784, 32, 10], global_batch_size=32, n_mubatches=1, precision="bf-16")
    K = _K()
    _, x = _pitched(4, 8, _gen("names"))
    _, W = _pitched(8, 8, _gen("names-w"))
    with pytest.raises(ValueError):
        K.linear_fwd(x, W, None, precision="fp16")


def test_loss_curve_tracks_fp32():
    """The reference model trained from the same initial weights on the same data: the bf16 loss stays within 1e-4 of
    the fp32 loss at every one of 300 steps.  Measured on an H100 80GB HBM3 (700 W power limit): at most 1.25e-5 (tf32:
    2.4e-5), a margin of 8 (BASELINE.md §16)."""
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    sizes, gbs, steps = [784, 128, 127, 126, 125, 124, 123, 10], 128, 300
    x, y = synthetic_mnist(n=steps * gbs)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    curves = {}
    for precision in ("fp32", "bf16"):
        tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=4, lr=0.006, precision=precision)
        curves[precision] = [float(tr.step(xh[i * gbs:(i + 1) * gbs], yh[i * gbs:(i + 1) * gbs])) for i in range(steps)]
    gap = max(abs(a - b) for a, b in zip(curves["bf16"], curves["fp32"]))
    print(f"\n[bf16] loss curve: max |bf16 - fp32| over {steps} steps {gap:.3g}; final {curves['bf16'][-1]:.6f} "
          f"vs {curves['fp32'][-1]:.6f}")
    assert gap <= 1e-4 and curves["bf16"][-1] < curves["bf16"][0]
