"""Residual connections on one GPU, against fp64, from the engine's own buffers after a Trainer step:

* per layer, micro-batch and element: a residual layer's act[l] = act[l-1] + f(z) * keep * s (test_gpu_chain:
  act_fwd_oracle for the branch, plus one rounding of the add), the gate gate[l] (ReLU included: residual plans gate
  every activation), every dgrad dz[l-1] = (dz[l] W_l + g_l) * gate[l-1] and the update.  g_l = dL/da_l is read from the
  engine's g[l] on the layer-wise path (where dz[l] = g[l] * gate[l] must hold bitwise) and rebuilt in fp64 from the
  kernel's own dz on the chain path, which keeps it in registers.  Paths: the cluster chain at C = 4 and 2, the one-CTA
  chain (C = 1, micro-batches of 32 and 128 rows), per-micro-batch chain launches, the layer-wise GEMMs (coalesced and
  per micro-batch) and split-K on wide layers; widths on and off multiples of 8; relu / gelu / silu / tanh, dropout 0 and
  0.3, fp32 / tf32 / bf16, MSE and cross-entropy;
* inference plans add the skip and keep no gates;
* a pipeline stage with its neighbours replayed from memory, a residual layer on each side of both boundaries, folded,
  unfolded and layer-wise: the received gradient is kept (g[L]), dz[L] = g[L] * gate[L], and the gradient sent upstream
  is W_1^T dz_1 + g_1;
* several engine steps against the Python VM;
* a residual plan launches as many kernels and graph nodes as the same model's gated plan and differs from its plan text
  only by its res= (and, for ReLU, act=) tags; residual=False is the default model bit for bit;
* the residual grid (RES_GRID): every chain micro-batch size, NTW 2 / 4 / 8, uneven and empty warp halves, clusters of
  1 to 4 CTAs (a residual layer whose last CTAs own no feature), the k-split layer 1 feeding a residual layer, a residual
  layer 1 on stage 0 (its skip is the staging buffer), depth 16, 16 / 17 / 32 classes and the four launch forms, for
  every (activation, dropout, precision) pair, with the loss head checked from the kernel's logits; a residual layer 1
  over three steps in both staging sets; the split-K residual GEMMs over two steps.

Bounds: the products as test_gpu_chain (bf16: the operands rounded by test_gpu_bf16.bf, RTOL_BF16), the skip and g_l
unrounded fp32 in every precision, plus one rounding of the add.  Every residual layer of the grid has nil features
(nil_features), where the branch is exactly zero and the skip or g_l is checked to one rounding: the bound of a product
is far wider than a skip rounded like an operand, the bound of a nil feature is not.  The CPU tests check that the grid
reaches every branch it names and that the checker rejects a set of residual faults in an emulated step.
"""
import math
import re
import zlib

import pytest
import torch

from test_gpu_chain import (ATOL, DROP_P, DROP_SEED, FAR_BIASES, HEAD_RTOL, LAUNCH_FORMS, LOGIT_SPREAD, MB_GRID, RTOL, U,
                            _chain_geometry, _gather, _n_mu, _pitched, _poison, act_fwd_oracle, excess, fwd_oracle,
                            head_oracle, rows_update_oracle)

KINDS = ["relu", "gelu", "silu", "tanh"]
P, SEED = 0.3, 0x5EED_0F_0DD_5EED
UPD_TOL = 2e-2                              # whole trajectories against the Python VM


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _batch(rows, in_dim, classes, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(rows, in_dim, generator=g)
    y = torch.zeros(rows, classes)
    y[torch.arange(rows), torch.randint(0, classes, (rows,), generator=g)] = 1.0
    return x.pin_memory(), y.pin_memory()


def operand_model(precision):
    """(operand, rtol) of the products: bf16 multiplies the operands rounded to bf16 (test_gpu_bf16.bf), exactly, and
    is bounded by RTOL_BF16 = 2^-16 of sum |a'||b'|; fp32 and tf32 take the operands as they are, with RTOL.  The skip
    and the skip gradient g_l never go through an operand: they stay unrounded fp32 in every precision."""
    if precision == "bf16":
        from test_gpu_bf16 import RTOL_BF16, bf

        return bf, RTOL_BF16
    return (lambda t: t.double()), RTOL[precision]


def nil_features(W, b):
    """(output features whose row of W and bias are zero, input features whose column of W is zero) of one layer: the
    branch f(z) of a nil output is f(0) = 0 exactly, and a nil input adds nothing to the dgrad."""
    rows = (W == 0).all(1) & (b == 0)
    cols = (W == 0).all(0)
    return rows.nonzero().flatten(), cols.nonzero().flatten()


def check_residual_layers(eng, model, W0, x, n_mu, mb, precision, lr, step=0, g_in=None, samples_of=None,
                          training=True):
    """Every layer of the step that just ran against fp64 from the engine's own buffers; returns {check: err / bound}.
    ``g_in``: the gradient a non-last stage received ([n_mu, mb, out]), else None.  ``samples_of(mu)``: the global
    sample index of every row of micro-batch mu, whose dropout masks the rows draw (default: mu * mb + n, one replica).
    ``training=False``: an inference pass (no dropout, gates, dgrads or update).

    At the nil features of a residual layer (nil_features) the skip terms stand alone and are checked to one rounding:
    ``skip{l}``, act[l] = act[l - 1] at a nil output; ``gskip{l}``, the dgrad of layer l at a nil input is g_l alone,
    then gated by layer l - 1 (or stored as ITS g).  g_l is the engine's stored g[l] (layer-wise), the received gradient,
    or, on the chain path, which keeps it in registers, dz[l] / gate[l] where dz[l] is a normal fp32 number (one rounding
    away from the kernel's g_l)."""
    from shallowspeed_b200.ops import functional as F

    op, rtol = operand_model(precision)
    kind, p = model.activation, (model.dropout if training else 0.0)
    s = F.dropout_scale(p) if p > 0 else 1.0
    L = len(model.linears)
    res = {}
    blocks = []
    for lin in model.linears:
        blk = W0[model.arena.offsets[lin.block_index]:][: lin.out_dims * model.arena.lds[lin.block_index]]
        blocks.append(blk.view(lin.out_dims, -1)[:, : lin.in_dims + 1].double().cpu())
    nils = [nil_features(blk[:, :-1], blk[:, -1]) if lin.residual else None for lin, blk in zip(model.linears, blocks)]
    upd_dz, upd_a = [[] for _ in range(L)], [[] for _ in range(L)]

    def put(k, v):
        res[k] = max(res.get(k, 0.0), v)

    for mu in range(n_mu):
        samples = samples_of(mu) if samples_of is not None else mu * mb + torch.arange(mb)
        acts = [x[mu * mb:(mu + 1) * mb].double()] + [eng.act(mu, l).double().cpu() for l in range(1, L + 1)]
        dzs = [eng.dz(mu, l).cpu() for l in range(L + 1)] if training else None
        gates = [None] * (L + 1)
        gs = [None] * (L + 1)
        for l, lin in enumerate(model.linears, start=1):
            W, b = blocks[l - 1][:, :-1], blocks[l - 1][:, -1]
            if lin.activation is None:
                ref, bound = fwd_oracle(op(acts[l - 1]), op(W), b, False, rtol)
                put(f"fwd{l}", excess(acts[l], ref, bound))
                continue
            keep = F.dropout_mask(p, model.dropout_seed, lin.dropout[2], step, samples, lin.out_dims) if p > 0 else None
            (ra, ba), gam, z = act_fwd_oracle(kind, op(acts[l - 1]), op(W), b, keep, s, rtol)
            if training:
                gates[l] = eng.gate(mu, l).cpu()
                if kind == "relu":
                    # the kernel's gate is 1[z > 0] * keep * s of ITS z: exact where z is farther from 0 than its error
                    e = fwd_oracle(op(acts[l - 1]), op(W), b, False, rtol)[1]
                    want = ((z > 0).double() * s * (1.0 if keep is None else keep.double()))
                    sure = z.abs() > e
                    assert torch.equal(gates[l].double()[sure], want[sure]), (mu, l)
                    assert bool(((gates[l] == 0) | (gates[l] == s)).all()), (mu, l)
                else:
                    put(f"gate{l}", excess(gates[l], *gam))
                if keep is not None:
                    assert bool((gates[l][~keep].view(torch.int32) == 0).all()), (mu, l)
            if lin.residual:
                skip = acts[l - 1]                          # unrounded fp32, in every precision
                ra = skip + ra
                ba = ba * (1.0 + U) + U * ra.abs() + ATOL   # the add's one rounding
                if training and not eng.uses_chain():
                    gs[l] = eng.g(mu, l).double().cpu()
                J = nils[l - 1][0]
                if len(J):
                    # f(0) = 0: act[l] is the skip itself, up to the add's rounding
                    put(f"skip{l}", excess(acts[l][:, J], skip[:, J], U * skip[:, J].abs() + ATOL))
            put(f"act{l}", excess(acts[l], ra, ba))
        if not training:
            continue
        for l in range(1, L + 1):
            upd_a[l - 1].append(acts[l - 1])
            upd_dz[l - 1].append(dzs[l].double())
        if g_in is not None and model.linears[-1].residual:
            # the received gradient is kept as g[L], gated out of place into dz[L]: one fp32 multiply
            cols = model.linears[-1].out_dims
            assert torch.equal(eng.g(mu, L)[:, :cols].cpu(), g_in[mu][:, :cols])
            assert torch.equal(dzs[L][:, :cols], g_in[mu][:, :cols] * gates[L][:, :cols])
        # g_l = dL/da_l of a residual layer: what the layer-wise dgrad stored (g[l]), or, on the chain path, which keeps
        # it in registers, rebuilt in fp64 from the kernel's own dz with the bound it accumulates
        g_val, g_bnd = None, None
        if g_in is not None and model.linears[-1].residual:
            g_val, g_bnd = g_in[mu].double(), torch.zeros_like(g_in[mu].double())
        for l in range(L, 0, -1):
            lin = model.linears[l - 1]
            if l == 1 and model.stage_idx == 0:
                continue                                   # the first stage runs no dgrad of layer 1
            W = blocks[l - 1][:, :-1]
            d = dzs[l].double()
            pre = op(d) @ op(W)
            mag = op(d).abs() @ op(W).abs()
            skip = g_val if lin.residual else torch.zeros_like(pre)
            skip_b = g_bnd if lin.residual else torch.zeros_like(pre)
            pre_ref = pre + skip[:, : pre.shape[1]]
            pre_b = rtol * mag + skip_b[:, : pre.shape[1]] + U * (pre.abs() + skip[:, : pre.shape[1]].abs()) + ATOL
            prev = model.linears[l - 2] if l >= 2 else None
            J = nils[l - 1][1] if lin.residual else []
            if len(J):
                # a nil input: the dgrad is g_l alone.  The kernel's own g_l: stored (exact) or dz[l] / gate[l]
                if gs[l] is not None or (g_in is not None and l == L):
                    gk, rel, ok = (gs[l] if gs[l] is not None else g_in[mu].double()), 0.0, None
                else:
                    gl = gates[l].double()
                    ok = (gl != 0) & (d.abs() >= 2.0**-126)       # a normal fp32 dz[l]: one relative rounding of g_l
                    gk, rel = torch.where(ok, d / torch.where(ok, gl, 1.0), 0.0), U
                gk = gk[:, J]
                ok = torch.ones_like(gk, dtype=torch.bool) if ok is None else ok[:, J]
                if prev is not None and prev.residual and gs[l - 1] is not None:
                    got, ref = gs[l - 1][:, J], gk
                elif prev is not None and prev.activation is not None:
                    got, ref = dzs[l - 1][:, J].double(), gk * gates[l - 1][:, J].double()
                else:
                    got, ref = dzs[l - 1][:, J].double(), gk
                bound = (rel + U) * (1.0 + 2.0 * U) * ref.abs() + ATOL
                put(f"gskip{l}", excess(got[ok], ref[ok], bound[ok]))
            if prev is not None and prev.residual and gs[l - 1] is not None:
                put(f"g{l - 1}", excess(gs[l - 1], pre_ref, pre_b))
                # dz[l - 1] is the stored g[l - 1] times the stored gate, one fp32 multiply
                cols = prev.out_dims
                assert torch.equal(dzs[l - 1][:, :cols], gs[l - 1][:, :cols].float() * gates[l - 1][:, :cols]), (mu, l)
                g_val, g_bnd = gs[l - 1], torch.zeros_like(pre_ref)
                continue
            if prev is not None and prev.activation is not None:
                m = gates[l - 1].double()
                put(f"dgrad{l}", excess(dzs[l - 1], pre_ref * m, pre_b * m.abs() + U * (pre_ref * m).abs() + ATOL))
            else:
                put(f"dgrad{l}", excess(dzs[l - 1], pre_ref, pre_b))
            if prev is not None and prev.residual:
                g_val, g_bnd = pre_ref, pre_b
    W1 = model.arena.weights.detach().double().cpu()
    for l, lin in enumerate(model.linears, start=1):
        if g_in is not None or not training:
            break                                          # a replayed stage: the update is checked by its own tests
        o, ld = lin.out_dims, model.arena.lds[lin.block_index]
        off = model.arena.offsets[lin.block_index]
        d = (W1[off:off + o * ld] - W0[off:off + o * ld].double().cpu()).view(o, ld)[:, : lin.in_dims + 1]
        if precision == "bf16":
            from test_gpu_bf16 import _update_oracle

            ref, bound = _update_oracle(torch.cat(upd_dz[l - 1]), torch.cat(upd_a[l - 1]), blocks[l - 1], lr)
        else:
            ref, bound = rows_update_oracle(torch.cat(upd_dz[l - 1]), torch.cat(upd_a[l - 1]), blocks[l - 1], lr, rtol)
        put(f"upd{l}", excess(d, ref, bound))
    worst = max(res, key=res.get)
    print(f"\n[residual] {kind} p={p} {precision} n_mu={n_mu} mb={mb}: max err/bound {res[worst]:.3g} ({worst}); "
          + " ".join(f"{k}={v:.2g}" for k, v in res.items()))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


NO_COALESCE = {"SSB_NO_COALESCE": "1"}
NO_CHAIN = {"SSB_NO_CHAIN": "1"}
CASES = {
    # name: (sizes, global batch, micro-batches, precision, loss, env, path)
    "cluster4-127": ([784, 127, 127, 127, 10], 128, 4, "fp32", "mse", {}, "cluster4"),
    "cluster4-128-bf16": ([784, 128, 128, 128, 128, 10], 128, 4, "bf16", "mse", {}, "cluster4"),
    "cluster2-64-tf32-ce": ([784, 64, 64, 64, 10], 128, 4, "tf32", "cross_entropy", {}, "cluster2"),
    "one-cta-24": ([784, 24, 24, 24, 10], 128, 4, "fp32", "mse", {}, "one-cta"),
    "one-cta-32-mb128-tf32": ([784, 32, 32, 32, 32, 10], 256, 2, "tf32", "cross_entropy", {}, "one-cta"),
    "per-mubatch-127": ([784, 127, 127, 127, 10], 128, 4, "fp32", "cross_entropy", NO_COALESCE, "per-mubatch"),
    "layerwise-127": ([784, 127, 127, 127, 10], 128, 4, "fp32", "mse", NO_CHAIN, "layerwise"),
    "layerwise-24-tf32-ce": ([784, 24, 24, 24, 10], 128, 4, "tf32", "cross_entropy", NO_CHAIN, "layerwise"),
    "layerwise-per-mubatch-bf16": ([784, 64, 64, 64, 10], 128, 4, "bf16", "mse", {**NO_CHAIN, **NO_COALESCE},
                                   "layerwise-per-mubatch"),
    "splitk-2048": ([784, 2048, 2048, 10], 64, 2, "fp32", "mse", {}, "splitk"),
}


def _check_path(eng, path, text):
    lines = text.splitlines()
    if path.startswith("cluster") or path == "one-cta":
        assert eng.uses_chain() and eng.coalesced()
        assert eng.chain_cluster() == {"cluster4": 4, "cluster2": 2, "one-cta": 1}[path], eng.chain_cluster()
        assert any("mlp_chain" in ln and "res=1" in ln for ln in lines), text
        return
    if path == "per-mubatch":
        assert eng.uses_chain() and not eng.coalesced() and all(f"mu={mu}" in text for mu in range(4)), text
        return
    assert not eng.uses_chain()
    assert any("gemm" in ln and "res=1" in ln for ln in lines), text
    if path == "layerwise":
        assert eng.coalesced()
    elif path == "layerwise-per-mubatch":
        assert not eng.coalesced() and all(f"mu={mu}" in text for mu in range(4)), text
    elif path == "splitk":
        assert sum(1 for ln in lines if "splits=" in ln and "res=1" in ln) >= 2, text


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, P], ids=["nodrop", "drop"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_every_layer_matches_fp64(case, kind, p, monkeypatch):
    from shallowspeed_b200.parallel.engine import Trainer

    sizes, gbs, n_mu, precision, loss, env, path = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    lr = 0.05
    tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=lr, precision=precision, loss=loss, dropout=p,
                 dropout_seed=SEED, activation=kind, residual=True, device="cuda:0")
    eng, model = tr.engine, tr.model
    _check_path(eng, path, eng.plan_text(0))
    W0 = model.arena.weights.detach().clone()
    x, y = _batch(gbs, sizes[0], sizes[-1], seed=3)
    tr.step(x, y)
    tr.synchronize()
    check_residual_layers(eng, model, W0, x, n_mu, gbs // n_mu, precision, lr)


@pytest.mark.gpu
def test_the_checker_is_not_vacuous(monkeypatch):
    """A plain (non-residual) run of the same weights fails the residual checks: its act lacks the skip."""
    from shallowspeed_b200.parallel.engine import Trainer

    sizes = [784, 64, 64, 10]
    tr = Trainer(sizes, lr=0.05, activation="gelu", device="cuda:0")
    x, y = _batch(128, 784, 10)
    W0 = tr.model.arena.weights.detach().clone()
    tr.step(x, y)
    tr.synchronize()
    ref = Trainer(sizes, lr=0.05, activation="gelu", residual=True, device="cuda:0")

    class _Eng:                                           # the plain engine's buffers under the residual model's eyes
        def __getattr__(self, name):
            return getattr(tr.engine, name)

        def g(self, mu, l):
            return torch.zeros_like(tr.engine.act(mu, l))

    with pytest.raises(AssertionError):
        check_residual_layers(_Eng(), ref.model, W0, x, 4, 32, "fp32", 0.05)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relu", "gelu"])
def test_inference_adds_the_skip_without_gates(kind):
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.ops import functional as F
    from shallowspeed_b200.parallel.engine import NativeWorker, Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    sizes = [784, 96, 96, 96, 10]
    tr = Trainer(sizes, lr=0.05, device="cuda:0", activation=kind, residual=True, dropout=0.5, dropout_seed=2)
    x, y = _batch(128, 784, 10)
    tr.step(x, y)
    tr.synchronize()
    ds = Dataset(None, 128, 128, device="cuda")
    ds.local_batch_size = 128
    ds.from_arrays(x.numpy(), y.numpy())
    vw = NativeWorker(None, None, tr.model, ds, None)
    tr.model.eval()
    vw.execute(InferenceSchedule(1, 1, 0), 0)
    eng = vw.engine_for(InferenceSchedule(1, 1, 0))
    for l in (1, 2):
        with pytest.raises(RuntimeError):
            eng.gate(0, l)
        with pytest.raises(RuntimeError):
            eng.g(0, l)
    assert "res=1" in eng.plan_text(0)
    probs = vw.output_buffers[0].double().cpu()
    a = x.double()
    for lin in tr.model.linears:
        z = a @ lin._params["W"].data.double().cpu().T + lin._params["b"].data.double().cpu()
        if lin.activation is None:
            a = z
        else:
            br = F.activation_ref(kind, z)[0]
            a = a + br if lin.residual else br
    assert _frob(probs, F.softmax_ref(a)) < 1e-4


# ---------------------------------------------------------------- pipeline stages, neighbours replayed from memory
RES_SIZES = [784, 48, 48, 48, 48, 48, 48, 10]


PP_CASES = {"folded": {}, "unfolded": {"SSB_PP_FOLD": "0"}, "layerwise": NO_CHAIN}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relu", "gelu"])
@pytest.mark.parametrize("p", [0.0, P], ids=["nodrop", "drop"])
@pytest.mark.parametrize("case", sorted(PP_CASES))
def test_pipeline_stage_keeps_the_received_gradient_as_its_skip(case, kind, p, monkeypatch):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E
    from shallowspeed_b200.pipe import PipeDreamSchedule
    from test_gpu_dp_replay import _StandInComm
    from test_gpu_pp_replay import _Ctx, _nan_pad, check_tiles, own_flags

    from shallowspeed_b200 import _C as C

    for k, v in PP_CASES[case].items():
        monkeypatch.setenv(k, v)
    pp, st, mb, n_mu, lr = 4, 1, 32, 4, 0.05
    rows = mb * n_mu
    model = MLP(RES_SIZES, st, pp, rows, dropout=p, dropout_seed=SEED, activation=kind, residual=True).to("cuda")
    assert [lin.residual for lin in model.linears] == [True, True]      # both sides of both boundaries
    opt = SGD(model.parameters(), lr, arena=model.arena)
    ctxs = {}

    def make_pp_context(comm, eng, n_mu, mb_rows, is_first, is_last):
        ld_in, ld_out = eng.boundary_lds()
        me = C.PpContext(int(n_mu), int(mb_rows), int(ld_in), int(ld_out), False, False)
        prev = C.PpContext(int(n_mu), int(mb_rows), int(ld_in), int(ld_in), True, False)
        nxt = C.PpContext(int(n_mu), int(mb_rows), int(ld_out), int(ld_out), False, False)
        me.open_local(prev, nxt)
        ctxs.update(me=me, prev=prev, next=nxt)
        torch.cuda.synchronize()
        return me

    monkeypatch.setattr(E, "make_nccl_comm", lambda comm: None)
    monkeypatch.setattr(E, "make_pp_context", make_pp_context)

    class _Shape:
        mubatch_size = mb

    w = E.NativeWorker(None, _StandInComm(pp, st), model, _Shape(), opt, pp_transport="peer")
    sched = PipeDreamSchedule(n_mu, pp, st)
    eng = w.engine_for(sched)
    text = eng.plan_text(0)
    assert eng.uses_chain() == (case != "layerwise")
    assert ("pp_push" in text) == (case != "folded"), text
    if case == "layerwise":
        assert any("relu_mask" in ln and "res=1" in ln and f"act={kind}" in ln for ln in text.splitlines()), text
    ld_in, ld_out = eng.boundary_lds()
    me = _Ctx(ctxs["me"], n_mu, mb, ld_in, ld_out)
    nb = {side: _Ctx(ctxs[side], n_mu, mb, ld_in if side == "prev" else ld_out, ld_in if side == "prev" else ld_out)
          for side in ("prev", "next")}
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(rows, 48, generator=gen)
    dz_in = torch.randn(rows, 48, generator=gen) * 1e-2
    e = int(me.epoch[0].item()) + 1
    me.act_in.copy_(_nan_pad(x, ld_in).view(n_mu, mb, ld_in).cuda())
    me.dz_in.copy_(_nan_pad(dz_in, ld_out).view(n_mu, mb, ld_out).cuda())
    me.flags.copy_(own_flags(me.layout, me.flags.numel(), n_mu, e).cuda())
    for ctx in nb.values():
        ctx.act_in.fill_(float("nan"))
        ctx.dz_in.fill_(float("nan"))
    torch.cuda.synchronize()
    W0 = model.arena.weights.detach().clone()
    model.dropout_step = 3
    w.step_from(sched, None, None)
    eng.synchronize()
    torch.cuda.synchronize()
    L = len(model.linears)
    act_L = torch.stack([eng.act(mu, L).cpu() for mu in range(n_mu)])
    dz_0 = torch.stack([eng.dz(mu, 0).cpu() for mu in range(n_mu)])
    check_tiles(nb["next"].act_in.cpu(), act_L, 48, "act pushed to stage 2")
    check_tiles(nb["prev"].dz_in.cpu(), dz_0, 48, "dz pushed to stage 0")
    # the receive slot still holds the received gradient after the step (it was read, not gated in place)
    assert torch.equal(me.dz_in.cpu()[..., :48], dz_in.view(n_mu, mb, 48))
    check_residual_layers(eng, model, W0, x, n_mu, mb, "fp32", lr, step=3, g_in=dz_in.view(n_mu, mb, 48))
    # what went upstream is W_1^T dz_1 + g_1: the skip gradient of the stage's residual first layer
    W1 = W0[model.arena.offsets[0]:][: 48 * model.arena.lds[0]].view(48, -1)[:, :48].double().cpu()
    W2 = W0[model.arena.offsets[1]:][: 48 * model.arena.lds[1]].view(48, -1)[:, :48].double().cpu()
    for mu in range(n_mu):
        dz1, dz2 = eng.dz(mu, 1).double().cpu(), eng.dz(mu, 2).double().cpu()
        g2 = dz_in.view(n_mu, mb, 48)[mu].double()
        g1 = dz2 @ W2 + g2                               # rebuilt from the kernel's own dz (the chain keeps it in registers)
        b1 = RTOL["fp32"] * (dz2.abs() @ W2.abs()) + U * (g1.abs() + g2.abs()) + ATOL
        ref = dz1 @ W1 + g1
        bound = RTOL["fp32"] * (dz1.abs() @ W1.abs()) + b1 + U * (ref.abs() + g1.abs()) + ATOL
        assert excess(dz_0[mu][:, :48], ref, bound) <= 1.0
    assert not torch.equal(W0, model.arena.weights.detach())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_engine_steps_match_the_python_vm(kind):
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule, Worker

    steps, n_mu = 4, 4
    x, y = synthetic_mnist(n=128 * steps)
    runs = {}
    for dev in ("cpu", "cuda"):
        model = MLP(RES_SIZES, 0, 1, 128, dropout=P, dropout_seed=SEED, activation=kind, residual=True).to(dev)
        opt = SGD(model.parameters(), 0.05, arena=model.arena)
        ds = Dataset(None, 128, 128 // n_mu, device=dev)
        ds.local_batch_size = 128
        ds.from_arrays(x, y)
        w = Worker(None, None, model, ds, opt) if dev == "cpu" else NativeWorker(None, None, model, ds, opt)
        runs[dev] = (model, w)
    init = MLP(RES_SIZES, 0, 1, 128)
    for b in range(steps):
        for dev in ("cpu", "cuda"):
            model, w = runs[dev]
            model.dropout_step = b
            w.execute(GPipeSchedule(n_mu, 1, 0), b)
        runs["cuda"][1].sync_to_model()
        for p0, pc, pg in zip(init.parameters(), runs["cpu"][0].parameters(), runs["cuda"][0].parameters()):
            assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL, b


def _strip(text):
    return re.sub(r" (act|res)=\w+", "", text)


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{}, NO_CHAIN, NO_COALESCE], ids=["chain", "layerwise", "per-mubatch"])
@pytest.mark.parametrize("p", [0.0, P], ids=["nodrop", "drop"])
def test_residual_plans_launch_what_gated_plans_launch(env, p, monkeypatch):
    """The same model without skips and gated (a smooth activation), on the same path: the same kernels, graph nodes and
    plan text but for the tags."""
    from shallowspeed_b200.parallel.engine import Trainer

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sizes = [784, 64, 64, 64, 10]
    gated = Trainer(sizes, lr=0.05, device="cuda:0", dropout=p, dropout_seed=1, activation="gelu").engine
    for kind in KINDS:
        eng = Trainer(sizes, lr=0.05, device="cuda:0", dropout=p, dropout_seed=1, activation=kind, residual=True).engine
        assert eng.uses_chain() == gated.uses_chain() and eng.chain_cluster() == gated.chain_cluster()
        assert eng.kernels_per_step() == gated.kernels_per_step()
        assert eng.graph_nodes() == gated.graph_nodes()
        assert "res=1" in eng.plan_text(0)
        assert _strip(eng.plan_text(0)) == _strip(gated.plan_text(0))


@pytest.mark.gpu
def test_residual_false_is_the_default_bit_for_bit():
    from shallowspeed_b200.parallel.engine import Trainer

    sizes = [784, 64, 64, 64, 10]
    batches = [_batch(128, 784, 10, seed=i) for i in range(3)]
    runs = []
    for kw in ({}, {"residual": False}):
        tr = Trainer(sizes, lr=0.05, device="cuda:0", **kw)
        losses = [tr.step(x, y) for x, y in batches]
        tr.synchronize()
        runs.append((tr, losses))
    (a, la), (b, lb) = runs
    assert la == lb and torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert a.engine.plan_text(0) == b.engine.plan_text(0) and "res=" not in a.engine.plan_text(0)
    assert a.engine.uses_chain()
    with pytest.raises(RuntimeError):
        a.engine.g(0, 2)
    other = Trainer(sizes, lr=0.05, device="cuda:0", residual=True)
    for x, y in batches:
        other.step(x, y)
    other.synchronize()
    assert not torch.equal(a.model.arena.weights, other.model.arena.weights)


@pytest.mark.gpu
def test_train_cli_trains_a_deep_residual_model(tmp_path):
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "train.py", "--synthetic", "--no-eval", "--hidden", "256", "--n-layers", "7",
                        "--residual", "--activation", "gelu", "--steps", "20"], cwd=root, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])


# ================================================================================================== the residual grid
# Every chain micro-batch size, cluster shape and launch form with residual layers, checked per element by
# check_residual_layers (bf16 through the bf() operand model) and the test_gpu_chain head oracles.  Every residual layer
# has nil features (nil_features: output feature NIL_ROW(o) with a zero row and bias, input feature NIL_COL with a zero
# column), where the skip and g_l stand alone; features 0..3 of every hidden layer carry FAR_BIASES for the tails.
RES_SHAPES = {
    "res-base": [784, 128, 128, 97, 97, 33, 33, 10],     # k-split layer 1 feeding a residual layer; C = 4; 33 = 32 + 1 + 0 + 0
    "res-first": [64, 64, 64, 64, 10],                  # residual layer 1 on stage 0: its skip is the staging buffer; C = 2
    "res-c3": [96, 96, 65, 65, 17],                     # C = 3, the last CTA of the 65-wide layers one feature wide; slow head
    "res-tiny": [7, 7, 7, 3],                           # C = 1; fan-in below one k-block
    "res-depth16": [40] * 16 + [10],                    # kChainMaxLayers: 15 residual layers
    "res-one-cta-32": [784, 32, 32, 32, 32],            # C = 1; 32 classes
    "res-full": [128, 128, 128, 128, 16],               # C = 4; 16 classes, the fast head's edge
}
NIL_COL = 4


def NIL_ROW(o):
    return o - 2


RES_VARIANTS = [(k, p) for k in KINDS for p in (0.0, DROP_P)]
RES_PRECISIONS = ["fp32", "tf32", "bf16"]
RES_LR = 1.0                  # test_gpu_chain.LR: the update stands well above the fp32 rounding of the weights


def _res_grid():
    """(shape, mb_rows, n_mu, precision, form, inference, loss, kind, p).  The cross is too large to run whole; it is cut
    so that every (variant, precision) pair reaches every launch form, NTW 2 / 4 / 8 on the chain and every cluster size
    (test_residual_grid_reaches_every_branch asserts it):
    * per pair: the four launch forms on res-base / res-first (coalesced at mb 24, per micro-batch at 40, the layer-wise
      forms at 100 and 24), res-c3 at mb 128 (C = 3, NTW 8), res-tiny or res-one-cta-32 (C = 1);
    * res-base at every MB_GRID size in each precision, the variants in turn;
    * the other shapes at mb 24, 40 and 128, precisions and variants in turn;
    * inference at two shapes."""
    forms = list(LAUNCH_FORMS)
    cases = []
    i = 0
    for v, (kind, p) in enumerate(RES_VARIANTS):
        for q, pr in enumerate(RES_PRECISIONS):
            loss = ("mse", "cross_entropy")[i % 2]
            pair = ("res-base", "res-first") if i % 2 == 0 else ("res-first", "res-base")
            cases.append((pair[0], 24, 2, pr, forms[0], False, loss, kind, p))
            cases.append((pair[1], 40, 2, pr, forms[1], False, loss, kind, p))
            cases.append((pair[0], 100, 2, pr, forms[2], False, loss, kind, p))
            cases.append((pair[1], 24, 2, pr, forms[3], False, loss, kind, p))
            cases.append(("res-c3", 128, 1, pr, "coalesced", False, loss, kind, p))
            cases.append((("res-tiny", "res-one-cta-32")[i % 2], (24, 40, 128)[i % 3], _n_mu((24, 40, 128)[i % 3]), pr,
                          "coalesced", False, loss, kind, p))
            i += 1
    for q, pr in enumerate(RES_PRECISIONS):
        for j, mb in enumerate(MB_GRID):
            kind, p = RES_VARIANTS[(j + 3 * q) % len(RES_VARIANTS)]
            cases.append(("res-base", mb, _n_mu(mb), pr, "coalesced", False, ("mse", "cross_entropy")[j % 2], kind, p))
    j = 0
    for shape in RES_SHAPES:
        if shape == "res-base":
            continue
        for mb in (24, 40, 128):
            kind, p = RES_VARIANTS[(5 * j + 1) % len(RES_VARIANTS)]
            cases.append((shape, mb, _n_mu(mb), RES_PRECISIONS[j % 3], "coalesced", False, ("mse", "cross_entropy")[j % 2],
                          kind, p))
            j += 1
    cases.append(("res-base", 40, 2, "fp32", "coalesced", True, "mse", "gelu", 0.0))
    cases.append(("res-c3", 100, 2, "bf16", "coalesced", True, "mse", "relu", 0.0))
    return cases


RES_GRID = _res_grid()


def _res_case_id(c):
    shape, mb, _n, pr, form, inference, loss, kind, p = c
    return (f"{shape}-mb{mb}-{pr}-{form}-{kind}{'-drop' if p else ''}{'-inference' if inference else ''}"
            f"{'-ce' if loss != 'mse' else ''}")


def _chain_cluster(sizes):
    from shallowspeed_b200 import _C

    return _C.chain_cluster_size(list(zip(sizes[:-1], sizes[1:])), True, True, True, True, False, False)


def _init_res_weights(sizes, residual, x, n_mu, gen, activation):
    """_init_weights for a residual model: He-scaled weights, non-zero biases, FAR_BIASES on features 0..3 of every
    hidden layer, the nil features of every residual layer, and the last layer scaled so that the logits of the widest
    micro-batch span LOGIT_SPREAD through the residual forward."""
    from shallowspeed_b200.ops import functional as F

    L = len(sizes) - 1
    Ws, bs = [], []
    for l, (i, o) in enumerate(zip(sizes[:-1], sizes[1:]), start=1):
        W = torch.randn(o, i, generator=gen, dtype=torch.float64) * math.sqrt(2.0 / i)
        b = torch.randn(o, generator=gen, dtype=torch.float64) * 0.1
        if l < L:
            n = min(len(FAR_BIASES), o)
            b[:n] = torch.tensor(FAR_BIASES[:n], dtype=torch.float64)
        if residual[l - 1]:
            W[NIL_ROW(o)] = 0.0
            b[NIL_ROW(o)] = 0.0
            W[:, NIL_COL] = 0.0
        Ws.append(W)
        bs.append(b)
    a = x.double()
    for l, (W, b) in enumerate(zip(Ws, bs), start=1):
        z = a @ W.T + b
        if l < L:
            br = F.activation_ref(activation, z)[0]
            a = a + br if residual[l - 1] else br
        else:
            a = z
    spread = max(float(z.max() - z.min()) for z in a.chunk(n_mu))
    s = LOGIT_SPREAD / spread
    Ws[-1], bs[-1] = Ws[-1] * s, bs[-1] * s
    return [W.float() for W in Ws], [b.float() for b in bs]


WORST = {}                    # (kernel, precision) -> (worst err / bound, its check and case)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    if WORST:
        print()
    for (kernel, precision), (v, what) in sorted(WORST.items()):
        print(f"[residual] worst err/bound {kernel:>10} {precision}: {v:.3g} ({what})")


def _note_worst(kernel, precision, res, what):
    for k, v in res.items():
        if v > WORST.get((kernel, precision), (-1.0, ""))[0]:
            WORST[(kernel, precision)] = (v, f"{k} at {what}")


def _branch_nonvacuous(model, blocks, acts, kind, p):
    """Non-vacuity on the branch f(z) of every activated layer (a = x + f(z) of a residual layer need not change sign):
    5 - 95 % of z positive outside the nil features, and, for a smooth kind or dropout, |z| > 4 in every layer and
    |z| > 9 in one (a micro-batch of one row need not reach the far tail behind a skip)."""
    far = False
    for l, lin in enumerate(model.linears, start=1):
        if lin.activation is None:
            continue
        W, b = blocks[l - 1][:, :-1], blocks[l - 1][:, -1]
        z = acts[l - 1] @ W.T + b
        live = torch.ones(z.shape[1], dtype=torch.bool)
        if lin.residual:
            live[nil_features(W, b)[0]] = False
        frac = float((z[:, live] > 0).double().mean())
        assert 0.05 <= frac <= 0.95, f"layer {l}: {frac:.3f} of the branch's z are positive"
        if kind != "relu" or p > 0:
            assert bool((z.abs() > 4).any()), f"layer {l}: no z in the tails"
            far |= bool((z.abs() > 9).any())
    assert far or (kind == "relu" and p == 0), "no z beyond 9"


def res_run(shape, mb, n_mu, precision, form, inference, loss, kind, p, monkeypatch, steps=1):
    """``steps`` Trainer steps (or one inference pass) of a residual model at the given shape, on new inputs each step,
    each checked per element against the weights snapshot taken just before it; returns the last {check: err / bound}."""
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    sizes = RES_SHAPES[shape]
    env = LAUNCH_FORMS[form]
    for k in env:
        monkeypatch.setenv(k, "1")
    L, C, rows = len(sizes) - 1, sizes[-1], mb * n_mu
    gen = torch.Generator().manual_seed(zlib.crc32(repr((shape, mb, n_mu, precision, form, kind, p, loss)).encode()))
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(steps)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float() for _ in range(steps)]
    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=RES_LR, precision=precision, loss=loss,
                 activation=kind, dropout=p, dropout_seed=DROP_SEED, residual=True, device="cuda:0")
    model = tr.model
    residual = [lin.residual for lin in model.linears]
    assert any(residual)
    Ws, bs = _init_res_weights(sizes, residual, xs[0], n_mu, gen, kind)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
    if inference:
        sched = InferenceSchedule(n_mu, 1, 0)
        eng = tr.worker.engine_for(sched)
    else:
        eng = tr.engine
    chain = "SSB_NO_CHAIN" not in env
    assert eng.uses_chain() == chain
    assert eng.coalesced() == ("SSB_NO_COALESCE" not in env)
    text = eng.plan_text(0)
    if chain:
        assert eng.chain_cluster() == _chain_cluster(sizes), (eng.chain_cluster(), sizes)
        assert any("mlp_chain" in ln and "res=1" in ln for ln in text.splitlines()), text
    else:
        assert any("gemm" in ln and "res=1" in ln for ln in text.splitlines()), text
    _poison(eng, model, sizes, rows, not inference, gated=not inference)
    if loss == "mse":
        head = head_oracle
    else:
        from test_gpu_cross_entropy import ce_head_oracle as head
    res = {}
    for step in range(steps):
        if step > 0:
            # the update moved the nil columns (their inputs are live); zero them again, and the nil rows with them
            for i, lin in enumerate(model.linears):
                if lin.residual:
                    model.arena.weight_view(i)[:, NIL_COL] = 0.0
                    model.arena.weight_view(i)[NIL_ROW(lin.out_dims)] = 0.0
                    model.arena.bias_view(i)[:, NIL_ROW(lin.out_dims)] = 0.0
            torch.cuda.synchronize()
        W0 = model.arena.weights.detach().clone()
        x, t = xs[step], ts[step]
        if inference:
            tr.worker.step_from(sched, x.pin_memory(), t.pin_memory())
            eng.synchronize()
            lv = None
        else:
            lv = float(tr.step(x.pin_memory(), t.pin_memory()))
            assert model.dropout_step == step
        torch.cuda.synchronize()
        blocks = [W0[model.arena.offsets[i]:][: o * model.arena.lds[i]].view(o, -1)[:, : k + 1].double().cpu()
                  for i, (o, k) in enumerate(model.arena.blocks)]
        acts = [x.double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
        _branch_nonvacuous(model, blocks, acts, kind, 0.0 if inference else p)
        res = dict(check_residual_layers(eng, model, W0, x, n_mu, mb, precision, RES_LR, step=step,
                                         training=not inference))
        if not inference:
            for l in range(1, L + 1):
                assert float(_gather(lambda mu: eng.dz(mu, l), n_mu).abs().max()) > 0.0, f"dz[{l}] is all zero"
            assert any(k.startswith("skip") for k in res) and any(k.startswith("gskip") for k in res), res
        # the loss head from the kernel's logits, per micro-batch
        probs = _gather(eng.probs, n_mu)
        loss_ref = loss_bound = 0.0
        for mu in range(n_mu):
            r = slice(mu * mb, (mu + 1) * mb)
            (pp, bp), (g, bg), (lr_, bl) = head(acts[L][r], t[r], rows, HEAD_RTOL)
            res["probs"] = max(res.get("probs", 0.0), excess(probs[r], pp, bp))
            if not inference:
                res["dzL"] = max(res.get("dzL", 0.0), excess(eng.dz(mu, L).cpu(), g, bg))
            loss_ref, loss_bound = loss_ref + lr_, loss_bound + bl
        if not inference:
            res["loss"] = abs(lv - loss_ref) / loss_bound if math.isfinite(lv) else math.inf
            for l in range(1, L):
                pad = _pitched(eng.gate(0, l), rows)[:, sizes[l]:]
                assert bool(pad.isnan().all()), f"layer {l}: a kernel wrote into the gate's padding"
        what = f"{shape} mb={mb} {form} {kind} p={p} {loss}{' inference' if inference else ''} step={step}"
        _note_worst("chain" if chain else "layer-wise", precision, res, what)
        bad = {k: v for k, v in res.items() if not v <= 1.0}
        assert not bad, (what, bad)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", RES_GRID, ids=[_res_case_id(c) for c in RES_GRID])
def test_residual_grid_per_element(case, monkeypatch):
    res_run(*case, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("form", ["coalesced", "per-micro-batch", "layer-wise"])
def test_residual_first_layer_over_both_staging_sets(form, precision, monkeypatch):
    """res-first (layer 1 residual on stage 0: its skip is the staging buffer of the step's input set) over three steps on
    new inputs, ReLU with dropout: each step per element against its own input and weights, at its own dropout step.  A
    skip read from the other staging set (the previous step's input) fails act1 and skip1."""
    res_run("res-first", 40, 2, precision, form, False, "mse", "relu", DROP_P, monkeypatch, steps=3)


@pytest.mark.gpu
def test_splitk_residual_layers_over_two_steps(monkeypatch):
    """The wide residual layer's split-K FWD and DGRAD (tc_gemm_res_kernel with k_splits > 1) over two steps on new
    inputs, each step per element against its own weights: an output tile whose counter was not re-armed would keep the
    first step's value."""
    from shallowspeed_b200.parallel.engine import Trainer

    sizes, gbs, n_mu = [784, 2048, 2048, 10], 64, 2
    tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=0.05, activation="gelu", dropout=P,
                 dropout_seed=SEED, residual=True, device="cuda:0")
    eng, model = tr.engine, tr.model
    text = eng.plan_text(0)
    assert sum(1 for ln in text.splitlines() if "splits=" in ln and "res=1" in ln) >= 2, text
    for step in range(2):
        W0 = model.arena.weights.detach().clone()
        x, y = _batch(gbs, sizes[0], sizes[-1], seed=10 + step)
        tr.step(x, y)
        tr.synchronize()
        res = check_residual_layers(eng, model, W0, x, n_mu, gbs // n_mu, "fp32", 0.05, step=step)
        _note_worst("layer-wise", "fp32", res, f"splitk {sizes} step={step}")


# ================================================================================================== CPU side
def _residual_flags(sizes):
    """Which Linears of a one-stage model are residual: the hidden ones of equal width (models.mlp.residual_layers)."""
    L = len(sizes) - 1
    return [l < L and i == o for l, (i, o) in enumerate(zip(sizes[:-1], sizes[1:]), start=1)]


def test_residual_grid_reaches_every_branch():
    """The grid reaches NTW 2 / 4 / 8, every n-tile split, uneven halves and ragged rows; clusters of 1 to 4 CTAs and a
    residual layer with featureless CTAs; a k-split layer 1 and a residual layer 1 on stage 0; residual layers next to
    plain ones on both sides; depth 16 and 16, 17 and 32 classes; and every launch form, NTW and cluster size for every
    (variant, precision) pair."""
    from shallowspeed_b200 import _C
    from shallowspeed_b200.models.mlp import MLP
    from shallowspeed_b200.ops.functional import precision_code

    for shape, sizes in RES_SHAPES.items():
        assert [lin.residual for lin in MLP(sizes, 0, 1, 32, residual=True).linears] == _residual_flags(sizes), shape
    seen = {"ntw": set(), "nts": set(), "uneven": False, "ragged": False, "C": set(), "featureless": False,
            "one-wide": False, "ksplit": False, "res-first": False, "after-plain": False, "before-plain": False,
            "depths": set(), "classes": set(), "inference": set(), "losses": set()}
    pairs = {(k, p > 0, pr): {"forms": set(), "ntw": set(), "C": set()} for k, p in RES_VARIANTS for pr in RES_PRECISIONS}
    for shape, mb, n_mu, pr, form, inference, loss, kind, p in RES_GRID:
        sizes = RES_SHAPES[shape]
        layers = list(zip(sizes[:-1], sizes[1:]))
        res = _residual_flags(sizes)
        seen["depths"].add(len(layers))
        seen["classes"].add(sizes[-1])
        seen["losses"].add(loss)
        pair = pairs[(kind, p > 0, pr)]
        pair["forms"].add(form)
        if inference:
            seen["inference"].add(shape)
            continue
        for l in range(1, len(res)):
            seen["after-plain"] |= res[l] and not res[l - 1]
            seen["before-plain"] |= res[l - 1] and not res[l] and l < len(res) - 1
        if "SSB_NO_CHAIN" in LAUNCH_FORMS[form]:
            continue
        assert _C.chain_eligible(layers, mb, sizes[-1], True, precision_code(pr)), (shape, mb)
        C = _chain_cluster(sizes)
        assert (_C.chain_cluster_budget(mb, C, precision_code(pr)) if C > 1 else _C.chain_budget(mb, precision_code(pr)))[0]
        _n_pad, ntw, (nt0, nt1) = _chain_geometry(mb)
        seen["ntw"].add(ntw)
        seen["nts"] |= {nt0, nt1}
        seen["uneven"] |= nt0 != nt1
        seen["ragged"] |= mb % 16 != 0
        seen["C"].add(C)
        for (i, o), r in zip(layers, res):
            if r and C > 1:
                seen["featureless"] |= 32 * (C - 1) >= o            # the last CTA's 32-feature slice is empty
                seen["one-wide"] |= o % 32 == 1
        seen["ksplit"] |= C > 1 and -(-sizes[0] // 32) > 4
        seen["res-first"] |= res[0]
        pair["ntw"].add(ntw)
        pair["C"].add(C)
    assert seen["ntw"] == {2, 4, 8} and seen["nts"] == {0, 2, 4, 6, 8} and seen["uneven"] and seen["ragged"]
    assert seen["C"] == {1, 2, 3, 4} and seen["featureless"] and seen["one-wide"]
    assert seen["ksplit"] and seen["res-first"] and seen["after-plain"] and seen["before-plain"]
    assert 16 in seen["depths"] and {16, 17, 32} <= seen["classes"]
    assert len(seen["inference"]) == 2 and seen["losses"] == {"mse", "cross_entropy"}
    for key, pair in pairs.items():
        assert pair["forms"] == set(LAUNCH_FORMS), key
        assert pair["ntw"] == {2, 4, 8}, (key, pair["ntw"])
        assert pair["C"] == {1, 2, 3, 4}, (key, pair["C"])
    # every residual layer of every shape has both kinds of nil feature, apart from FAR_BIASES' features 0..3
    for sizes in RES_SHAPES.values():
        for (i, o), r in zip(zip(sizes[:-1], sizes[1:]), _residual_flags(sizes)):
            if r:
                assert len({0, 1, 2, 3, NIL_COL, NIL_ROW(o)} & set(range(o))) == min(o, 6), sizes


EMU_SIZES = [12, 12, 12, 12, 5]          # res-first in small: residual layers 1, 2 and 3 on stage 0
EMU_FAULTS = {
    # fault: the precisions whose checks must reject it
    "skip-missing": ("fp32",),
    "skip-row": ("fp32",),                 # the skip of row n + 1 (row0 off by one)
    "skip-prev-step": ("fp32",),           # layer 1's skip from the previous step's input (the other staging set)
    "skip-rounded": ("tf32", "bf16"),      # the skip truncated to tf32 / rounded to bf16, as an operand would be
    "g-dropped": ("fp32",),
    "g-after-gate": ("fp32",),
    "g-rounded": ("fp32", "tf32", "bf16"),
    "gpre-after-mask": ("fp32",),          # layer-wise: g[l - 1] stored after the gate
    "tf32-products": ("bf16",),            # the products of a bf16 plan in tf32: outside the bf16 operand model
}


def _emulated_residual_step(precision, chain, fault=None, kind="gelu", p=DROP_P, step=1):
    """One training step of a residual model (EMU_SIZES, stage 0, two micro-batches of 6 rows) emulated on the CPU: the
    products in fp64 from the precision's operands (bf16: rounded), every stored value rounded to fp32 where the kernels
    round it, g_l kept in fp32 as in the chain kernel's registers (``chain``) or stored to g[l] (layer-wise).  ``fault``
    injects one of EMU_FAULTS.  Returns (engine stand-in, model, W0, x, n_mu, mb)."""
    from shallowspeed_b200.models.mlp import MLP
    from shallowspeed_b200.ops import functional as F
    from test_gpu_bf16 import bf
    from test_gpu_chain import act_ref, tf32_trunc

    n_mu, mb, lr = 2, 6, RES_LR
    rows, L = n_mu * mb, len(EMU_SIZES) - 1
    model = MLP(EMU_SIZES, 0, 1, rows, dropout=p, dropout_seed=DROP_SEED, activation=kind, residual=True)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(rows, EMU_SIZES[0], generator=gen)
    x_prev = torch.randn(rows, EMU_SIZES[0], generator=gen)
    Ws, bs = _init_res_weights(EMU_SIZES, [lin.residual for lin in model.linears], x, n_mu, gen, kind)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
    W0 = model.arena.weights.detach().clone()
    if fault == "tf32-products":
        op = lambda t: tf32_trunc(t).double()
    else:
        op = operand_model(precision)[0]
    rnd = bf if precision == "bf16" else (lambda t: tf32_trunc(t).double())   # an operand's rounding of the precision
    s = F.dropout_scale(p) if p > 0 else 1.0
    samples = torch.arange(rows)
    acts, gates = [x], [None]
    for l, lin in enumerate(model.linears, start=1):
        W, b = Ws[l - 1].double(), bs[l - 1].double()
        z = op(acts[-1]) @ op(W).T + b
        if lin.activation is None:
            acts.append(z.float())
            gates.append(None)
            continue
        keep = F.dropout_mask(p, DROP_SEED, lin.dropout[2], step, samples, lin.out_dims) if p > 0 else \
            torch.ones_like(z, dtype=torch.bool)
        f, f1 = (z.clamp_min(0.0), (z > 0).double()) if kind == "relu" else act_ref(kind, z)[:2]
        br = torch.where(keep, f * s, 0.0).float()
        gates.append(torch.where(keep, f1 * s, 0.0).float())
        if not lin.residual:
            acts.append(br)
            continue
        sk = acts[-1].double()
        if fault == "skip-missing":
            sk = torch.zeros_like(sk)
        elif fault == "skip-row":
            sk = torch.cat([torch.roll(c, -1, dims=0) for c in sk.chunk(n_mu)])
        elif fault == "skip-prev-step" and l == 1:
            sk = x_prev.double()
        elif fault == "skip-rounded":
            sk = rnd(sk)
        acts.append((sk + br.double()).float())
    dz = [torch.full((rows, EMU_SIZES[0]), float("nan"))] + [None] * L
    dz[L] = torch.randn(rows, EMU_SIZES[-1], generator=gen) * 1e-2
    gstore = [None] * (L + 1)
    g = None                                       # g_l of the layer below, fp32
    for l in range(L, 1, -1):
        lin, prev = model.linears[l - 1], model.linears[l - 2]
        prod = op(dz[l].double()) @ op(Ws[l - 1].double())
        gl = g.double() if lin.residual else torch.zeros_like(prod)
        if lin.residual and fault == "g-rounded":
            gl = rnd(gl)
        pre = (prod if (fault == "g-dropped" and lin.residual) else prod + gl).float()
        if fault == "g-after-gate" and lin.residual:
            dz[l - 1] = (prod.float().double() * gates[l - 1].double() + gl).float()
        else:
            dz[l - 1] = (pre.double() * gates[l - 1].double()).float()
        if prev.residual:
            gstore[l - 1] = dz[l - 1] if fault == "gpre-after-mask" else pre
        g = pre if prev.residual else None
    for i in range(L):
        dzi, ai = dz[i + 1].double(), acts[i].double()
        d = torch.cat([op(dzi).T @ op(ai), dzi.sum(0)[:, None]], 1)
        blk = model.arena.block(i)
        blk[:, : EMU_SIZES[i] + 1] = (blk[:, : EMU_SIZES[i] + 1].double() - lr * d).float()

    class Eng:
        def act(self, mu, l):
            return acts[l][mu * mb:(mu + 1) * mb]

        def dz(self, mu, l):
            return dz[l][mu * mb:(mu + 1) * mb]

        def gate(self, mu, l):
            return gates[l][mu * mb:(mu + 1) * mb]

        def g(self, mu, l):
            if chain:
                raise RuntimeError("the chain kernel keeps g in registers")
            return gstore[l][mu * mb:(mu + 1) * mb]

        def uses_chain(self):
            return chain

    return Eng(), model, W0, x, n_mu, mb


def test_residual_checker_rejects_injected_faults():
    """check_residual_layers accepts the emulated step in every precision, on the chain path (g_l in registers) and the
    layer-wise one (g[l] stored), and rejects each fault of EMU_FAULTS under the precisions listed with it: the skip
    missing, from the neighbouring row, from the previous step's input, or rounded like an operand; g_l dropped, added
    after the gate, or rounded; g[l - 1] stored after the mask; and tf32 products under the bf16 operand model."""
    for precision in RES_PRECISIONS:
        for chain in (True, False):
            for kind, p in (("gelu", DROP_P), ("relu", 0.0)):
                eng, model, W0, x, n_mu, mb = _emulated_residual_step(precision, chain, kind=kind, p=p)
                res = check_residual_layers(eng, model, W0, x, n_mu, mb, precision, RES_LR, step=1)
                assert {"skip1", "skip2", "skip3", "gskip2", "gskip3"} <= set(res), res
    for fault, precisions in EMU_FAULTS.items():
        for precision in precisions:
            for chain in ((False,) if fault == "gpre-after-mask" else (True, False)):
                eng, model, W0, x, n_mu, mb = _emulated_residual_step(precision, chain, fault)
                with pytest.raises(AssertionError):
                    check_residual_layers(eng, model, W0, x, n_mu, mb, precision, RES_LR, step=1)
