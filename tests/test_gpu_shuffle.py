"""Shuffled input staging on one GPU.  The permutation comes from ops.functional.shuffle_index (the torch oracle):

* the device helper (``_C.shuffle_index``) equals the oracle bit for bit;
* ``PipeEngine.stage_gather`` writes exactly the oracle's rows (``index_select``) into both staging sets, on first, last
  and middle pipeline stages, for DP ranks of dp = 2 and 4, through the float4 and the scalar copy, and leaves the
  NaN-poisoned pitch padding alone; it stages what ``stage_inputs`` stages from the pre-gathered batch;
* two shuffled epochs through ``NativeWorker.execute`` equal an engine fed the oracle's batches through
  ``stage_inputs`` bit for bit, and the Python VM within the tolerance of the other engine-vs-VM tests;
* shuffling changes no plan: graph nodes, kernels per step and ``plan_text()`` are those of an unshuffled worker.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
NS = [1, 2, 3, 5, 127, 128, 129, 59500, 65536, 65537]
SEEDS = [0, 0x9E37_79B9_7F4A_7C15, 2 ** 64 - 1]
EPOCHS = [0, 1, 2 ** 32 - 1]
SEED, GBS, N_ROWS = 0xC0FFEE_0000_0001, 128, 1000
UPD_TOL = 2e-2                              # as tests/test_gpu_dropout.py


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _C():
    from shallowspeed_b200 import _C as C

    return C


@pytest.mark.parametrize("n", NS)
def test_device_permutation_matches_the_oracle(n):
    from shallowspeed_b200.ops import functional as F

    q = torch.arange(n)
    for seed in SEEDS:
        for epoch in EPOCHS:
            got = _C().shuffle_index(n, seed, epoch, q.cuda()).cpu()
            assert torch.equal(got, F.shuffle_index(n, seed, epoch, q)), (n, seed, epoch)


def _data(in_dim, out_dim, n=N_ROWS, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, in_dim, generator=g), torch.randn(n, out_dim, generator=g)


def test_gather_rows_binding_scalar_and_vector_paths():
    """The kernel on its own: float4 rows (784 wide) and scalar rows (30 wide), padding untouched."""
    from shallowspeed_b200.ops import functional as F

    for in_dim, ld in ((784, 788), (30, 33)):
        x, y = _data(in_dim, 10)
        for dp, rank in ((1, 0), (4, 3)):
            rows = GBS // dp
            xd = torch.full((rows, ld), float("nan"), device="cuda")
            yd = torch.full((rows, 16), float("nan"), device="cuda")
            _C().gather_rows(x.cuda(), y.cuda(), SEED, 9, GBS, dp, rank, 5, xd[:, :in_dim], yd[:, :10])
            ids = F.shuffle_index(N_ROWS, SEED, 9, 5 * GBS + torch.arange(rows) * dp + rank)
            assert torch.equal(xd[:, :in_dim].cpu(), x[ids]) and torch.equal(yd[:, :10].cpu(), y[ids])
            assert bool(xd[:, in_dim:].isnan().all()) and bool(yd[:, 10:].isnan().all())
    with pytest.raises(RuntimeError):   # past the last full global batch
        _C().gather_rows(x.cuda(), None, SEED, 0, GBS, 1, 0, N_ROWS // GBS, torch.empty(GBS, 30, device="cuda"), None)


def _worker(sizes, dp, rank, pp, stage, monkeypatch, n_mu=4, **kw):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E
    from shallowspeed_b200.pipe import GPipeSchedule
    from test_gpu_dp_replay import _StandInComm

    monkeypatch.setattr(E, "make_nccl_comm", lambda comm: None)
    model = MLP(sizes, stage, pp, GBS).to("cuda")
    opt = SGD(model.parameters(), 0.05, arena=model.arena)

    class _Shape:
        mubatch_size = GBS // dp // n_mu

    w = E.NativeWorker(None, _StandInComm(pp, stage) if pp > 1 else None, model, _Shape(), opt, pp_transport="nccl", **kw)
    sched = GPipeSchedule(n_mu, pp, stage)
    return w, w.engine_for(sched), sched


def _poison(eng, set_):
    for t in eng.staging(set_):
        t.fill_(float("nan"))
    torch.cuda.synchronize()


def _check_set(eng, set_, x_all, y_all, ids, in_dim, write_x, write_y, x_before=None, y_before=None):
    xs, ys = (t.cpu() for t in eng.staging(set_))
    if write_x:
        assert torch.equal(xs[:, :in_dim], x_all[ids])
        assert bool(xs[:, in_dim:].isnan().all())
    else:
        assert bool(xs.isnan().all())
    if write_y:
        assert torch.equal(ys[:, :10], y_all[ids])
        assert bool(ys[:, 10:].isnan().all())
    else:
        assert bool(ys.isnan().all())


@pytest.mark.parametrize("dp,rank", [(1, 0), (2, 0), (2, 1), (4, 0), (4, 1)])
@pytest.mark.parametrize("in_dim", [784, 30])
def test_stage_gather_fills_both_sets(dp, rank, in_dim, monkeypatch):
    """A one-stage engine: set 0, one step, then set 1 - x also through act(mu, 0), which the plan reads."""
    from shallowspeed_b200.ops import functional as F

    sizes = [in_dim] + SIZES[1:] if in_dim == 784 else [in_dim, 64, 10]
    w, eng, sched = _worker(sizes, dp, rank, 1, 0, monkeypatch)
    x_all, y_all = _data(in_dim, 10)
    xd, yd = x_all.cuda(), y_all.cuda()
    rows = GBS // dp
    mb = rows // 4
    for set_, (epoch, batch) in enumerate(((3, 6), (4, 0))):
        assert eng.fill_set() == set_
        _poison(eng, set_)
        eng.stage_gather(xd, yd, SEED, epoch, GBS, dp, rank, batch)
        torch.cuda.synchronize()
        ids = F.shuffle_index(N_ROWS, SEED, epoch, batch * GBS + torch.arange(rows) * dp + rank)
        _check_set(eng, set_, x_all, y_all, ids, in_dim, True, True)
        if set_ == 1:    # the planner's act[.][0] points into set 1
            for mu in range(4):
                assert torch.equal(eng.act(mu, 0).cpu(), x_all[ids[mu * mb:(mu + 1) * mb]])
        else:
            eng.run()
            eng.synchronize()


@pytest.mark.parametrize("stage", [0, 1, 3])
def test_stage_gather_writes_only_the_inputs_a_stage_takes(stage, monkeypatch):
    """Stages of a four-stage pipeline: the first gathers x only, the last y only, a middle one launches nothing."""
    from shallowspeed_b200.ops import functional as F

    w, eng, sched = _worker(SIZES, 2, 1, 4, stage, monkeypatch, use_graph=False)
    x_all, y_all = _data(784, 10)
    _poison(eng, 0)
    eng.stage_gather(x_all.cuda(), y_all.cuda(), SEED, 1, GBS, 2, 1, 2)
    torch.cuda.synchronize()
    ids = F.shuffle_index(N_ROWS, SEED, 1, 2 * GBS + torch.arange(GBS // 2) * 2 + 1)
    _check_set(eng, 0, x_all, y_all, ids, 784, stage == 0, stage == 3)


def test_stage_gather_stages_what_stage_inputs_stages(monkeypatch):
    from shallowspeed_b200.ops import functional as F

    w, eng, sched = _worker(SIZES, 1, 0, 1, 0, monkeypatch)
    x_all, y_all = _data(784, 10)
    ids = F.shuffle_index(N_ROWS, SEED, 2, 3 * GBS + torch.arange(GBS))
    snaps = []
    for via_gather in (False, True):
        _poison(eng, 0)
        if via_gather:
            eng.stage_gather(x_all.cuda(), y_all.cuda(), SEED, 2, GBS, 1, 0, 3)
        else:
            eng.stage_inputs(x_all[ids].cuda(), y_all[ids].cuda())
        torch.cuda.synchronize()
        snaps.append([t.cpu() for t in eng.staging(0)])
    for a, b in zip(*snaps):
        assert torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


def test_stage_gather_rejects_bad_sources(monkeypatch):
    w, eng, sched = _worker(SIZES, 1, 0, 1, 0, monkeypatch)
    x_all, y_all = _data(784, 10)
    for args in ((x_all, None), (x_all.cuda()[:, :700], None), (x_all.cuda().double(), None),
                 (x_all.cuda(), y_all.cuda()[:999]), (x_all.cuda().t().contiguous().t(), None)):
        with pytest.raises(RuntimeError):
            eng.stage_gather(*args, SEED, 0, GBS, 1, 0, 0)
    with pytest.raises(RuntimeError):   # batch 7 of 1000 rows does not exist
        eng.stage_gather(x_all.cuda(), y_all.cuda(), SEED, 0, GBS, 1, 0, N_ROWS // GBS)


# ---------------------------------------------------------------- training
def _dataset(dev, shuffle=True, n_mu=4):
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist

    x, y = synthetic_mnist(n=N_ROWS)
    ds = Dataset(None, GBS, GBS // n_mu, device=dev, shuffle_seed=SEED if shuffle else None)
    if shuffle:
        return ds.from_arrays(x, y, DP_rank=0, DP_size=1)
    ds.local_batch_size = GBS
    full = N_ROWS - N_ROWS % GBS
    return ds.from_arrays(x[:full], y[:full])


@pytest.mark.parametrize("sched", ["naive", "gpipe"])
def test_two_shuffled_epochs_match_oracle_batches_and_the_python_vm(sched):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS, Worker

    n_mu = 4
    runs = {}
    for name in ("gather", "oracle", "vm"):
        dev = "cpu" if name == "vm" else "cuda"
        model = MLP(SIZES, 0, 1, GBS).to(dev)
        opt = SGD(model.parameters(), 0.05, arena=model.arena)
        ds = _dataset(dev)
        w = Worker(None, None, model, ds, opt) if name == "vm" else NativeWorker(None, None, model, ds, opt)
        runs[name] = (model, ds, w, [])
    s = SCHEDULE_NAME_TO_CLS[sched](n_mu, 1, 0)
    n = runs["gather"][1].get_num_batches()
    for epoch in range(2):
        for b in range(n):
            for name, (model, ds, w, losses) in runs.items():
                ds.set_epoch(epoch)
                if name == "oracle":
                    x, y = ds.load_batch(b)               # the torch oracle's gather, staged by stage_inputs
                    w.step_from(s, x, y)
                else:
                    w.execute(s, b)
                losses.append(w.batch_loss())
    assert runs["gather"][3] == runs["oracle"][3]
    for name in ("gather", "oracle"):
        runs[name][2].sync_to_model()
    assert torch.equal(runs["gather"][0].arena.weights, runs["oracle"][0].arena.weights)
    init = MLP(SIZES, 0, 1, GBS)
    for p0, pc, pg in zip(init.parameters(), runs["vm"][0].parameters(), runs["gather"][0].parameters()):
        assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL
    for a, b in zip(runs["gather"][3], runs["vm"][3]):
        assert abs(a - b) <= 1e-3 * abs(b), (a, b)


def test_shuffling_changes_no_plan_and_training_differs():
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule

    out = {}
    for shuffle in (False, True):
        model = MLP(SIZES, 0, 1, GBS).to("cuda")
        opt = SGD(model.parameters(), 0.05, arena=model.arena)
        w = NativeWorker(None, None, model, _dataset("cuda", shuffle), opt)
        s = GPipeSchedule(4, 1, 0)
        for b in range(3):
            w.execute(s, b)
        w.sync_to_model()
        eng = w.engine_for(s)
        out[shuffle] = (eng.graph_nodes(), eng.kernels_per_step(), eng.plan_text(0), eng.plan_text(1),
                        model.arena.weights.clone())
    assert out[False][:4] == out[True][:4]
    assert not torch.equal(out[False][4], out[True][4])


def test_shuffled_dataset_must_live_on_the_engine_device():
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule

    model = MLP(SIZES, 0, 1, GBS).to("cuda")
    w = NativeWorker(None, None, model, _dataset("cpu"), SGD(model.parameters(), 0.05, arena=model.arena))
    with pytest.raises(ValueError):
        w.execute(GPipeSchedule(4, 1, 0), 0)
