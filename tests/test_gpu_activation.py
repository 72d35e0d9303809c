"""GELU, SiLU and tanh hidden layers on one GPU, against fp64 (ops.functional.activation_ref, dropout_mask):

* per layer, micro-batch and element, from the engine's own buffers after one Trainer step (test_gpu_chain:
  check_layers): act[l] matches f(z) * keep * s, the gate gate[l] matches f'(z) * keep * s, every dgrad matches
  (dz[l] @ W) * gamma, and the update matches act and dz.  The
  cluster chain (k-split layer 1), the one-CTA chain, per-micro-batch launches, the layer-wise GEMMs, split-K on wide
  layers; fp32 and tf32, MSE and cross-entropy, with and without dropout;
* a pipeline stage with its neighbours replayed from memory: folded and unfolded boundaries and the layer-wise plan,
  the last forward layer's gate applied to the received gradient;
* several engine steps against the Python VM on the CPU;
* the stand-alone act_fwd kernel across the fp32 range within the device formulas' rounding bound, gate_mul_ on
  pitched buffers bitwise;
* inference plans apply f and keep no gates; gated plans launch as many kernels and graph nodes as ReLU's and differ
  from its plan text only by their act= tags; activation="relu" is the default model bit for bit.
"""
import re

import pytest
import torch

from test_gpu_chain import check_layers, worst_table  # noqa: F401  (the table of worst err / bound)

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
KINDS = ["gelu", "silu", "tanh"]
P, SEED = 0.3, 0xDEAD_BEEF_1234_5678
UPD_TOL = 2e-2                              # whole trajectories against the Python VM


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _batch(rows, in_dim, classes, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(rows, in_dim, generator=g)
    y = torch.zeros(rows, classes)
    y[torch.arange(rows), torch.randint(0, classes, (rows,), generator=g)] = 1.0
    return x.pin_memory(), y.pin_memory()


NO_COALESCE = {"SSB_NO_COALESCE": "1"}
CASES = {
    # name: (sizes, global batch, micro-batches, precision, loss, env, path)
    "chain-ksplit-fp32": (SIZES, 128, 4, "fp32", "mse", {}, "cluster"),
    "chain-ksplit-tf32-ce": (SIZES, 128, 4, "tf32", "cross_entropy", {}, "cluster"),
    "chain-one-cta": ([784, 32, 24, 10], 128, 4, "fp32", "mse", {}, "one-cta"),
    "chain-per-mubatch": (SIZES, 128, 4, "fp32", "mse", NO_COALESCE, "per-mubatch"),
    "layerwise-129-33-ce": ([784, 129, 129, 33], 1024, 4, "fp32", "cross_entropy", {"SSB_NO_CHAIN": "1"}, "layerwise"),
    "layerwise-per-mubatch-tf32": (SIZES, 128, 4, "tf32", "mse", {"SSB_NO_CHAIN": "1", **NO_COALESCE}, "per-mubatch"),
    "splitk-wide": ([784, 4096, 4096, 10], 64, 2, "fp32", "mse", {"SSB_SPLITK": "1"}, "splitk"),
}


def _check_path(eng, path, text, kind):
    if path in ("cluster", "one-cta"):
        assert eng.uses_chain() and eng.coalesced()
        assert (eng.chain_cluster() == 1) == (path == "one-cta"), eng.chain_cluster()
        if path == "cluster":
            assert eng.chain_ksplit() == 2
    elif path == "per-mubatch":
        assert not eng.coalesced()
        assert all(f"mu={mu}" in text for mu in range(4)), text
    elif path == "layerwise":
        assert not eng.uses_chain()
        lines = text.splitlines()
        assert any("gemm" in ln and f"act={kind}" in ln for ln in lines), text
    elif path == "splitk":
        assert not eng.uses_chain()
        assert sum(1 for ln in text.splitlines() if "splits=" in ln and f"act={kind}" in ln) >= 2, text


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
                 dropout_seed=SEED, activation=kind, device="cuda:0")
    eng, model = tr.engine, tr.model
    _check_path(eng, path, eng.plan_text(0), kind)
    W0 = model.arena.weights.detach().clone()
    x, y = _batch(gbs, sizes[0], sizes[-1], seed=3)
    tr.step(x, y)
    tr.synchronize()
    mb = gbs // n_mu
    check_layers(eng, model, W0, x, n_mu, mb, precision, lr, lambda mu: mu * mb + torch.arange(mb))


# ---------------------------------------------------------------- pipeline stages, neighbours replayed from memory
PP_CASES = {"folded": {}, "unfolded": {"SSB_PP_FOLD": "0"}, "layerwise": {"SSB_NO_CHAIN": "1"}}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", sorted(PP_CASES))
def test_pipeline_stage_applies_its_gates_at_the_boundary(case, kind, monkeypatch):
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
    model = MLP(SIZES, st, pp, rows, dropout=P, dropout_seed=SEED, activation=kind).to("cuda")
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
        assert any("relu_mask" in ln and f"act={kind}" in ln for ln in text.splitlines()), text
    ld_in, ld_out = eng.boundary_lds()
    me = _Ctx(ctxs["me"], n_mu, mb, ld_in, ld_out)
    nb = {side: _Ctx(ctxs[side], n_mu, mb, ld_in if side == "prev" else ld_out, ld_in if side == "prev" else ld_out)
          for side in ("prev", "next")}
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(rows, 127, generator=gen)                     # what stage 0 sends: a smooth activation, any sign
    dz_in = torch.randn(rows, 125, generator=gen) * 1e-2
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
    gate_L = torch.stack([eng.gate(mu, L).cpu() for mu in range(n_mu)])
    dz_L = torch.stack([eng.dz(mu, L).cpu() for mu in range(n_mu)])
    dz_0 = torch.stack([eng.dz(mu, 0).cpu() for mu in range(n_mu)])
    check_tiles(nb["next"].act_in.cpu(), act_L, 125, "act pushed to stage 2")
    check_tiles(nb["prev"].dz_in.cpu(), dz_0, 127, "dz pushed to stage 0")
    # the received gradient times this stage's last gate (which holds keep * s): one fp32 multiply
    assert torch.equal(dz_L[..., :125], dz_in.view(n_mu, mb, 125) * gate_L[..., :125])
    check_layers(eng, model, W0, x, n_mu, mb, "fp32", lr, lambda mu: mu * mb + torch.arange(mb), step=3,
                 check_update=False)
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
        model = MLP(SIZES, 0, 1, 128, dropout=P, dropout_seed=SEED, activation=kind).to(dev)
        opt = SGD(model.parameters(), 0.05, arena=model.arena)
        ds = Dataset(None, 128, 128 // n_mu, device=dev)
        ds.local_batch_size = 128
        ds.from_arrays(x, y)
        w = Worker(None, None, model, ds, opt) if dev == "cpu" else NativeWorker(None, None, model, ds, opt)
        runs[dev] = (model, w)
    init = MLP(SIZES, 0, 1, 128)
    for b in range(steps):
        for dev in ("cpu", "cuda"):
            model, w = runs[dev]
            model.dropout_step = b
            w.execute(GPipeSchedule(n_mu, 1, 0), b)
        runs["cuda"][1].sync_to_model()
        for p0, pc, pg in zip(init.parameters(), runs["cpu"][0].parameters(), runs["cuda"][0].parameters()):
            assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL, b


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("env", [{}, {"SSB_NO_CHAIN": "1"}], ids=["chain", "layerwise"])
def test_inference_applies_f_without_gates(kind, env, monkeypatch):
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.ops import functional as F
    from shallowspeed_b200.parallel.engine import NativeWorker, Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    tr = Trainer(SIZES, lr=0.05, device="cuda:0", activation=kind, dropout=0.5, dropout_seed=2)
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
    with pytest.raises(RuntimeError):
        eng.gate(0, 1)
    probs = vw.output_buffers[0].double().cpu()
    a = x.double()
    for lin in tr.model.linears:
        a = a @ lin._params["W"].data.double().cpu().T + lin._params["b"].data.double().cpu()
        if lin.activation is not None:
            a = F.activation_ref(kind, a)[0]
    assert _frob(probs, F.softmax_ref(a)) < 1e-4


def _strip(text):
    return re.sub(r" act=\w+", "", text)


@pytest.mark.parametrize("env", [{}, {"SSB_NO_CHAIN": "1"}, NO_COALESCE], ids=["chain", "layerwise", "per-mubatch"])
@pytest.mark.parametrize("p", [0.0, P], ids=["nodrop", "drop"])
def test_gated_plans_launch_what_relu_launches(env, p, monkeypatch):
    from shallowspeed_b200.parallel.engine import Trainer

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    relu = Trainer(SIZES, lr=0.05, device="cuda:0", dropout=p, dropout_seed=1).engine
    for kind in KINDS:
        eng = Trainer(SIZES, lr=0.05, device="cuda:0", dropout=p, dropout_seed=1, activation=kind).engine
        assert eng.kernels_per_step() == relu.kernels_per_step()
        assert eng.graph_nodes() == relu.graph_nodes()
        assert f"act={kind}" in eng.plan_text(0)
        assert _strip(eng.plan_text(0)) == relu.plan_text(0)


def test_explicit_relu_is_the_default_bit_for_bit():
    from shallowspeed_b200.parallel.engine import Trainer

    batches = [_batch(128, 784, 10, seed=i) for i in range(3)]
    runs = []
    for kw in ({}, {"activation": "relu"}):
        tr = Trainer(SIZES, lr=0.05, device="cuda:0", **kw)
        losses = [tr.step(x, y) for x, y in batches]
        tr.synchronize()
        runs.append((tr, losses))
    (a, la), (b, lb) = runs
    assert la == lb and torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert a.engine.plan_text(0) == b.engine.plan_text(0) and "act=" not in a.engine.plan_text(0)
    with pytest.raises(RuntimeError):
        a.engine.gate(0, 1)
    other = Trainer(SIZES, lr=0.05, device="cuda:0", activation="gelu")
    for x, y in batches:
        other.step(x, y)
    other.synchronize()
    assert not torch.equal(a.model.arena.weights, other.model.arena.weights)


def _sweep():
    """fp32 inputs of the stand-alone act_fwd check: every 2^10-th bit pattern with |z| in [2^-20, 2^8], +-0, subnormals,
    +-FLT_MAX, and 64 consecutive patterns on either side of SiLU's expf overflow (88.72), of GELU's z * z overflow
    (sqrt(FLT_MAX) = 1.84e19) and of tanh's saturation (9), all with both signs."""
    f32 = lambda v: torch.tensor([v], dtype=torch.float32).view(torch.int32).item()
    pats = [torch.arange(f32(2.0**-20), f32(2.0**8) + 1, 1024, dtype=torch.int64)]
    pats.append(torch.tensor([0, 1, 2, 3, 0x3FFFFF, 0x7FFFFF, 0x800000, f32(3.4028234663852886e38)], dtype=torch.int64))
    for edge in (88.72283935546875, 1.8446742974197924e19, 9.0):
        pats.append(f32(edge) + torch.arange(-64, 65, dtype=torch.int64))
    bits = torch.cat(pats).to(torch.int32)
    z = bits.view(torch.float32)
    return torch.cat([z, -z])


ACT_WORST = {}


@pytest.mark.parametrize("kind", KINDS)
def test_module_path_kernels_match_the_oracle(kind):
    """The stand-alone activation kernel (ptx.cuh: act_fwd) per element against fp64 across the fp32 range, within the
    device formulas' rounding bound (test_gpu_chain: act_rounding_bound); every finite input gives finite outputs."""
    from test_gpu_chain import ATOL, act_ref, act_rounding_bound

    from shallowspeed_b200.ops import cuda as K

    z = _sweep()
    a, g = K.act_fwd(kind, z.cuda())
    a, g = a.cpu(), g.cpu()
    assert bool(torch.isfinite(a).all()) and bool(torch.isfinite(g).all()), kind
    f, f1, _ = act_ref(kind, z)
    Ba, Bg = act_rounding_bound(kind, z, 0.0)
    ra = ((a.double() - f).abs() / (Ba + ATOL))
    rg = ((g.double() - f1).abs() / (Bg + ATOL))
    worst = {"a": (float(ra.max()), float(z[ra.argmax()])), "g": (float(rg.max()), float(z[rg.argmax()]))}
    print(f"\n[act_fwd] {kind}: {z.numel()} inputs, worst err/bound a {worst['a'][0]:.3g} at z={worst['a'][1]:.6g}, "
          f"g {worst['g'][0]:.3g} at z={worst['g'][1]:.6g}")
    assert worst["a"][0] <= 1.0 and worst["g"][0] <= 1.0, worst


def test_gate_mul_on_pitched_buffers():
    """g *= gamma bitwise in fp32 on buffers of different row pitches, NaN in both paddings, which keep their bits."""
    from shallowspeed_b200 import _C

    gen = torch.Generator().manual_seed(4)
    rows, cols = 37, 45
    gbuf = torch.full((rows, 48), float("nan"))
    gbuf[:, :cols] = torch.randn(rows, cols, generator=gen)
    hbuf = torch.full((rows, 56), float("nan"))
    hbuf[:, :cols] = torch.randn(rows, cols, generator=gen)
    want = gbuf[:, :cols] * hbuf[:, :cols]
    gd, hd = gbuf.cuda(), hbuf.cuda()
    _C.gate_mul_(gd[:, :cols], hd[:, :cols])
    torch.cuda.synchronize()
    got = gd.cpu()
    bits = lambda t: t.contiguous().view(torch.int32)
    assert torch.equal(bits(got[:, :cols]), bits(want))
    assert torch.equal(bits(got[:, cols:]), bits(gbuf[:, cols:])) and torch.equal(bits(hd.cpu()), bits(hbuf))
