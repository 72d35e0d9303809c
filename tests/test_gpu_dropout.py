"""Dropout on one GPU.  The masks come from ops.functional.dropout_mask (the torch Philox), the numbers from fp64:

* per layer and per element, from the kernels' own buffers after one Trainer step (test_gpu_chain: check_layers): where
  the mask drops, act[l] is +0 bitwise; where it keeps, act[l] matches relu(z) * s; every dgrad matches
  (dz @ W) * (a > 0) * s; the update matches act and dz.  The
  chain kernel (cluster and one-CTA launches, MSE and cross-entropy, fp32 and tf32), the layer-wise GEMMs (a 129-wide
  layer, 33 classes, 256-row micro-batches) and a wide model whose forward runs split-K;
* several engine steps against the Python VM on the CPU;
* p = 0 is bit-identical to a model without dropout, and dropout adds no kernel and no graph node;
* inference plans do not drop.
"""
import pytest
import torch

from test_gpu_chain import check_layers, worst_table  # noqa: F401  (the table of worst err / bound)

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
P, SEED = 0.3, 0xDEAD_BEEF_1234_5678
UPD_TOL = 2e-2                              # whole trajectories against the Python VM (as tests/test_gpu_lr_schedule.py)


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
    "chain-mb32-fp32": (SIZES, 128, 4, "fp32", "mse", {}, "cluster"),
    "chain-mb32-tf32-ce": (SIZES, 128, 4, "tf32", "cross_entropy", {}, "cluster"),
    "chain-mb8-fp32": (SIZES, 32, 4, "fp32", "mse", {}, "cluster"),
    "chain-mb64-fp32-ce": (SIZES, 128, 2, "fp32", "cross_entropy", {}, "cluster"),
    "chain-one-cta": ([784, 32, 24, 10], 128, 4, "fp32", "mse", {}, "one-cta"),
    # one launch per micro-batch (mu_base = mu): the rows of micro-batch mu are samples mu * mb + n
    "chain-per-mubatch": (SIZES, 128, 4, "fp32", "mse", NO_COALESCE, "per-mubatch"),
    "layerwise-129-33": ([784, 129, 129, 33], 1024, 4, "fp32", "cross_entropy", {"SSB_NO_CHAIN": "1"}, "layerwise"),
    "layerwise-ref-tf32": (SIZES, 128, 4, "tf32", "mse", {"SSB_NO_CHAIN": "1"}, "layerwise"),
    # per-micro-batch GEMMs: row_base = mu * mb
    "layerwise-per-mubatch": (SIZES, 128, 4, "fp32", "mse", {"SSB_NO_CHAIN": "1", **NO_COALESCE}, "per-mubatch"),
    # forward and dgrad of the 4096-wide layers run split-K
    "splitk-wide": ([784, 4096, 4096, 10], 64, 2, "fp32", "mse", {"SSB_SPLITK": "1"}, "splitk"),
}


def _check_path(eng, path, text):
    if path in ("cluster", "one-cta"):
        assert eng.uses_chain() and eng.coalesced()
        assert (eng.chain_cluster() == 1) == (path == "one-cta"), eng.chain_cluster()
    elif path == "per-mubatch":
        assert not eng.coalesced()
        assert all(f"mu={mu}" in text for mu in range(4)), text
    elif path == "layerwise":
        assert not eng.uses_chain() and "drop=fwd" in text and "drop=dgrad" in text, text
    elif path == "splitk":
        assert not eng.uses_chain()
        lines = text.splitlines()
        assert any("splits=" in ln and "drop=fwd" in ln for ln in lines), text
        assert any("splits=" in ln and "drop=dgrad" in ln for ln in lines), text


@pytest.mark.parametrize("case", sorted(CASES))
def test_every_layer_matches_fp64(case, monkeypatch):
    from shallowspeed_b200.parallel.engine import Trainer

    sizes, gbs, n_mu, precision, loss, env, path = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    lr = 0.05
    tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=lr, precision=precision, loss=loss, dropout=P,
                 dropout_seed=SEED, device="cuda:0")
    eng, model = tr.engine, tr.model
    _check_path(eng, path, eng.plan_text(0))
    W0 = model.arena.weights.detach().clone()
    x, y = _batch(gbs, sizes[0], sizes[-1], seed=3)
    tr.step(x, y)                                       # step 0: Trainer sets model.dropout_step
    tr.synchronize()
    mb = gbs // n_mu
    check_layers(eng, model, W0, x, n_mu, mb, precision, lr, lambda mu: mu * mb + torch.arange(mb))


@pytest.mark.parametrize("rank", [0, 1])
def test_dp_replica_draws_the_masks_of_its_samples(rank, monkeypatch):
    """Replica ``rank`` of dp = 2 (a stand-in communicator; the update stays local, nothing is exchanged): row n of its
    DP-local batch is global sample n * 2 + rank, in both launch forms of the chain kernel."""
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E
    from shallowspeed_b200.pipe import GPipeSchedule
    from test_gpu_dp_replay import _StandInComm

    monkeypatch.setitem(E.DP_MODE, "nccl", 0)          # a replica that updates from its own gradient
    monkeypatch.setattr(E, "make_nccl_comm", lambda comm: None)
    if rank == 1:
        monkeypatch.setenv("SSB_NO_COALESCE", "1")
    dp, n_mu, mb, lr = 2, 4, 16, 0.05
    model = MLP(SIZES, 0, 1, mb * n_mu * dp, dropout=P, dropout_seed=SEED).to("cuda")
    opt = SGD(model.parameters(), lr, arena=model.arena)
    x, y = _batch(mb * n_mu, 784, 10, seed=rank)
    ds = Dataset(None, mb * n_mu * dp, mb, device="cuda")
    ds.local_batch_size = mb * n_mu
    ds.from_arrays(x.cuda(), y.cuda())
    w = E.NativeWorker(_StandInComm(dp, rank), None, model, ds, opt, comm_mode="nccl")
    sched = GPipeSchedule(n_mu, 1, 0)
    eng = w.engine_for(sched)
    assert eng.uses_chain() and eng.coalesced() == (rank == 0)
    W0 = model.arena.weights.detach().clone()
    model.dropout_step = 5
    w.execute(sched, 0)
    w.sync_to_model()
    check_layers(eng, model, W0, x, n_mu, mb, "fp32", lr, lambda mu: (mu * mb + torch.arange(mb)) * dp + rank, step=5)


# ---------------------------------------------------------------- pipeline stages, neighbours replayed from memory
PP_CASES = {
    # stage 1 of 4 (global layers 2 and 3): chain launches per micro-batch with the boundaries folded in
    "folded": {},
    # the chain without folding: the received gradient is staged by the backward-only launch, tiles are pushed
    "unfolded": {"SSB_PP_FOLD": "0"},
    # layer-wise GEMMs per micro-batch and the scaled relu_mask on the received gradient
    "layerwise": {"SSB_NO_CHAIN": "1"},
}


@pytest.mark.parametrize("case", sorted(PP_CASES))
def test_pipeline_stage_draws_the_masks_of_its_layers_and_rows(case, monkeypatch):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.ops import functional as F
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
    model = MLP(SIZES, st, pp, rows, dropout=P, dropout_seed=SEED).to("cuda")
    assert model.layer_base == 2
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
        assert "drop=scaled" in text and "drop=fwd" in text, text
    ld_in, ld_out = eng.boundary_lds()
    me = _Ctx(ctxs["me"], n_mu, mb, ld_in, ld_out)
    nb = {side: _Ctx(ctxs[side], n_mu, mb, ld_in if side == "prev" else ld_out, ld_in if side == "prev" else ld_out)
          for side in ("prev", "next")}
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(rows, 127, generator=gen).clamp_(min=0.0)     # what stage 0 sends: a dropped ReLU output
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
    dz_L = torch.stack([eng.dz(mu, L).cpu() for mu in range(n_mu)])
    dz_0 = torch.stack([eng.dz(mu, 0).cpu() for mu in range(n_mu)])
    # the outbound tiles are the dropped activations and the stage-input gradients, micro-batch for micro-batch
    check_tiles(nb["next"].act_in.cpu(), act_L, 125, "act pushed to stage 2")
    check_tiles(nb["prev"].dz_in.cpu(), dz_0, 127, "dz pushed to stage 0")
    # the received gradient: masked by the dropped act_L and scaled by s, one fp32 multiply
    s = torch.tensor(F.dropout_scale(P), dtype=torch.float32)
    want = torch.where(act_L[..., :125] > 0, dz_in.view(n_mu, mb, 125) * s, torch.zeros(()))
    assert torch.equal(dz_L[..., :125], want)
    # every layer, from the kernels' own buffers; dz[0] (layer 1's dgrad) is not masked by this stage
    check_layers(eng, model, W0, x, n_mu, mb, "fp32", lr, lambda mu: mu * mb + torch.arange(mb), step=3,
                 check_update=False)
    W1 = model.arena.weights.detach()
    assert not torch.equal(W0, W1)


@pytest.mark.parametrize("sched", ["naive", "gpipe"])
def test_engine_steps_match_the_python_vm(sched):
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS, Worker

    steps, n_mu = 4, 4
    x, y = synthetic_mnist(n=128 * steps)
    runs = {}
    for dev in ("cpu", "cuda"):
        model = MLP(SIZES, 0, 1, 128, dropout=P, dropout_seed=SEED).to(dev)
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
            w.execute(SCHEDULE_NAME_TO_CLS[sched](n_mu, 1, 0), b)
        runs["cuda"][1].sync_to_model()
        for p0, pc, pg in zip(init.parameters(), runs["cpu"][0].parameters(), runs["cuda"][0].parameters()):
            assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL, b


def test_p_zero_changes_nothing_and_dropout_adds_no_launch():
    from shallowspeed_b200.parallel.engine import Trainer

    batches = [_batch(128, 784, 10, seed=i) for i in range(3)]
    runs = {}
    for name, kw in (("plain", {}), ("zero", dict(dropout=0.0, dropout_seed=9)), ("drop", dict(dropout=0.2))):
        tr = Trainer(SIZES, lr=0.05, device="cuda:0", **kw)
        losses = [tr.step(x, y) for x, y in batches]
        tr.synchronize()
        runs[name] = (tr, losses)
    (a, la), (b, lb), (c, lc) = runs["plain"], runs["zero"], runs["drop"]
    assert la == lb and torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert not torch.equal(a.model.arena.weights, c.model.arena.weights)
    for t in (b, c):
        assert t.engine.kernels_per_step() == a.engine.kernels_per_step()
        assert t.engine.graph_nodes() == a.engine.graph_nodes()


def test_masks_follow_the_step():
    from shallowspeed_b200.parallel.engine import Trainer

    x, y = _batch(128, 784, 10)
    acts = []
    tr = Trainer(SIZES, lr=0.0, device="cuda:0", dropout=0.5, dropout_seed=1)
    for _ in range(2):
        tr.step(x, y)                                   # lr 0: same weights, only the step differs
        tr.synchronize()
        acts.append(tr.engine.act(0, 1).clone())
    assert not torch.equal(acts[0] > 0, acts[1] > 0)


def test_inference_does_not_drop():
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.ops import functional as F
    from shallowspeed_b200.parallel.engine import NativeWorker, Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    tr = Trainer(SIZES, lr=0.05, device="cuda:0", dropout=0.5, dropout_seed=2)
    x, y = _batch(128, 784, 10)
    tr.step(x, y)
    tr.synchronize()
    ds = Dataset(None, 128, 128, device="cuda")
    ds.local_batch_size = 128
    ds.from_arrays(x.numpy(), y.numpy())
    vw = NativeWorker(None, None, tr.model, ds, None)
    tr.model.eval()
    vw.execute(InferenceSchedule(1, 1, 0), 0)
    probs = vw.output_buffers[0].double().cpu()
    a = x.double()
    for lin in tr.model.linears:
        a = a @ lin._params["W"].data.double().cpu().T + lin._params["b"].data.double().cpu()
        if lin.activation is not None:
            a = a.clamp_min(0)
    assert _frob(probs, F.softmax_ref(a)) < 1e-4
