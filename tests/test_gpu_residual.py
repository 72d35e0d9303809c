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
  only by its res= (and, for ReLU, act=) tags; residual=False is the default model bit for bit.
"""
import re

import pytest
import torch

from test_gpu_chain import ATOL, RTOL, U, act_fwd_oracle, excess, fwd_oracle, rows_update_oracle

pytestmark = pytest.mark.gpu

KINDS = ["relu", "gelu", "silu", "tanh"]
P, SEED = 0.3, 0x5EED_0F_0DD_5EED
RT = {**RTOL, "bf16": 2.0**-7}             # bf16: one rounding of each 8-bit-mantissa operand of every product
UPD_TOL = 2e-2                              # whole trajectories against the Python VM


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _batch(rows, in_dim, classes, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(rows, in_dim, generator=g)
    y = torch.zeros(rows, classes)
    y[torch.arange(rows), torch.randint(0, classes, (rows,), generator=g)] = 1.0
    return x.pin_memory(), y.pin_memory()


def check_residual_layers(eng, model, W0, x, n_mu, mb, precision, lr, step=0, g_in=None, samples_of=None):
    """Every layer of the step that just ran against fp64 from the engine's own buffers; returns {check: err / bound}.
    ``g_in``: the gradient a non-last stage received ([n_mu, mb, out]), else None.  ``samples_of(mu)``: the global
    sample index of every row of micro-batch mu, whose dropout masks the rows draw (default: mu * mb + n, one replica)."""
    from shallowspeed_b200.ops import functional as F

    kind, p, rtol = model.activation, model.dropout, RT[precision]
    s = F.dropout_scale(p) if p > 0 else 1.0
    L = len(model.linears)
    res = {}
    blocks = []
    for lin in model.linears:
        blk = W0[model.arena.offsets[lin.block_index]:][: lin.out_dims * model.arena.lds[lin.block_index]]
        blocks.append(blk.view(lin.out_dims, -1)[:, : lin.in_dims + 1].double().cpu())
    upd_dz, upd_a = [[] for _ in range(L)], [[] for _ in range(L)]

    def put(k, v):
        res[k] = max(res.get(k, 0.0), v)

    for mu in range(n_mu):
        samples = samples_of(mu) if samples_of is not None else mu * mb + torch.arange(mb)
        acts = [x[mu * mb:(mu + 1) * mb].double()] + [eng.act(mu, l).double().cpu() for l in range(1, L + 1)]
        dzs = [eng.dz(mu, l).cpu() for l in range(L + 1)]
        gates = [None] * (L + 1)
        gs = [None] * (L + 1)
        for l, lin in enumerate(model.linears, start=1):
            W, b = blocks[l - 1][:, :-1], blocks[l - 1][:, -1]
            if lin.activation is None:
                ref, bound = fwd_oracle(acts[l - 1], W, b, False, rtol)
                put(f"fwd{l}", excess(acts[l], ref, bound))
                continue
            keep = F.dropout_mask(p, model.dropout_seed, lin.dropout[2], step, samples, lin.out_dims) if p > 0 else None
            (ra, ba), gam, z = act_fwd_oracle(kind, acts[l - 1], W, b, keep, s, rtol)
            gates[l] = eng.gate(mu, l).cpu()
            if kind == "relu":
                # the kernel's gate is 1[z > 0] * keep * s of ITS z: exact where z is farther from 0 than its error
                e = fwd_oracle(acts[l - 1], W, b, False, rtol)[1]
                want = ((z > 0).double() * s * (1.0 if keep is None else keep.double()))
                sure = z.abs() > e
                assert torch.equal(gates[l].double()[sure], want[sure]), (mu, l)
                assert bool(((gates[l] == 0) | (gates[l] == s)).all()), (mu, l)
            else:
                put(f"gate{l}", excess(gates[l], *gam))
            if keep is not None:
                assert bool((gates[l][~keep].view(torch.int32) == 0).all()), (mu, l)
            if lin.residual:
                ra = acts[l - 1] + ra
                ba = ba + U * (acts[l - 1].abs() + ra.abs())        # the add's rounding
                if not eng.uses_chain():
                    gs[l] = eng.g(mu, l).double().cpu()
            put(f"act{l}", excess(acts[l], ra, ba))
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
            pre = d @ W
            mag = d.abs() @ W.abs()
            skip = g_val if lin.residual else torch.zeros_like(pre)
            skip_b = g_bnd if lin.residual else torch.zeros_like(pre)
            pre_ref = pre + skip[:, : pre.shape[1]]
            pre_b = rtol * mag + skip_b[:, : pre.shape[1]] + U * (pre.abs() + skip[:, : pre.shape[1]].abs()) + ATOL
            prev = model.linears[l - 2] if l >= 2 else None
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
        if g_in is not None:
            break                                          # a replayed stage: the update is checked by its own tests
        o, ld = lin.out_dims, model.arena.lds[lin.block_index]
        off = model.arena.offsets[lin.block_index]
        d = (W1[off:off + o * ld] - W0[off:off + o * ld].double().cpu()).view(o, ld)[:, : lin.in_dims + 1]
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


def test_train_cli_trains_a_deep_residual_model(tmp_path):
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "train.py", "--synthetic", "--no-eval", "--hidden", "256", "--n-layers", "7",
                        "--residual", "--activation", "gelu", "--steps", "20"], cwd=root, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
