"""Learning-rate schedules on one GPU: every native update kernel reads ``lr`` from device memory, the engine keeps one
``lr`` slot per input-staging set and rewrites it only when the rate changes.

* kernel level: the fused wgrad epilogue (plain and stateful) and the flat SGD kernels against fp64, with ``lr`` a
  device tensor whose value is written after the inputs are prepared;
* a constant schedule on an engine built with another rate is bit-identical to an engine built with that constant;
* a rate that changes every step (including 0) against the Python VM on the CPU, and the ``lr == 0`` step bit for bit;
* ``Trainer.step_pipelined`` (no host sync between steps) against ``Trainer.step``, and ``run()`` without staging;
* the data-parallel kernels on one GPU with their peers replayed from memory (``test_gpu_dp_replay.py``), one rate
  per step.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]
MU, WD = 0.9, 1e-2
UPD_TOL = {"tf32": 6e-2, "fp32": 2e-2}       # as tests/test_gpu_momentum.py
RATES = [0.05, 0.0, 0.02, 0.08, 0.01, 0.03]


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _rule64(w, g, v, lr, mu, wd, nesterov):
    w, g, v = w.double(), g.double(), v.double()
    gp = g + wd * w
    v = mu * v + gp
    d = gp + mu * v if nesterov else v
    return w - lr * d, v


# ------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("stateful", [False, True])
def test_fused_wgrad_reads_lr_from_device(stateful):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(11)
    rows, k, n = 32, 127, 126
    ld = 128
    dz, x = torch.randn(rows, n, device="cuda"), torch.randn(rows, k, device="cuda")
    g = torch.cat([dz.double().T @ x.double(), dz.double().sum(0, keepdim=True).T], dim=1)
    lr_dev = torch.empty(1, device="cuda")
    for lr in (0.05, 0.0125):
        Wb = torch.zeros(n, ld, device="cuda")
        Wb[:, : k + 1] = torch.randn(n, k + 1, device="cuda")
        Vb = torch.zeros(n, ld, device="cuda")
        Vb[:, : k + 1] = torch.randn(n, k + 1, device="cuda") * 0.1
        W0, V0, Gb = Wb.clone(), Vb.clone(), torch.zeros(n, ld, device="cuda")
        lr_dev.fill_(lr)                                   # the value is written after the inputs are prepared
        rule = dict(velocity=Vb[:, :k], momentum=MU, weight_decay=WD, nesterov=True) if stateful else {}
        K.linear_wgrad(dz, x, Gb[:, :k], grad_b=Gb[:, k], weight=Wb[:, :k], lr=lr_dev, fuse_sgd=True, precision="fp32",
                       **rule)
        torch.cuda.synchronize()
        w_ref, v_ref = _rule64(W0[:, : k + 1], g, V0[:, : k + 1], lr, MU if stateful else 0.0, WD if stateful else 0.0,
                               stateful)
        dw = Wb[:, : k + 1].double() - W0[:, : k + 1].double()
        want = w_ref - W0[:, : k + 1].double()
        assert _frob(dw[:, :k], want[:, :k]) < 3e-3, lr
        assert _frob(dw[:, k], want[:, k]) < 1e-4, lr                       # bias column
        if stateful:
            assert _frob(Vb[:, : k + 1].double(), v_ref) < 1e-5


@pytest.mark.parametrize("n", [7, 100003])
@pytest.mark.parametrize("stateful", [False, True])
def test_flat_sgd_kernels_read_lr_from_device(n, stateful):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(n)
    lr_dev = torch.empty(1, device="cuda")
    for lr in (0.05, 0.0):
        w, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
        v = torch.randn(n, device="cuda")
        w0, v0 = w.clone(), v.clone()
        lr_dev.fill_(lr)
        if stateful:
            K.sgd_momentum_step_(w, g, v, lr_dev, MU, WD, True)
        else:
            K.sgd_step_(w, g, lr_dev)
        torch.cuda.synchronize()
        w_ref, v_ref = _rule64(w0, g, v0, lr, MU if stateful else 0.0, WD if stateful else 0.0, stateful)
        assert bool(((w.double() - w_ref).abs() <= 1e-6 * (1 + w_ref.abs())).all()), lr
        if lr == 0.0:
            assert torch.equal(w, w0)                                          # lr scales only the final step
        if stateful:
            assert bool(((v.double() - v_ref).abs() <= 1e-6 * (1 + v_ref.abs())).all())
            assert not torch.equal(v, v0)                                      # the momentum advances at any lr


def test_kernels_reject_a_bad_lr_tensor():
    from shallowspeed_b200.ops import cuda as K

    w, g = torch.randn(64, device="cuda"), torch.randn(64, device="cuda")
    for bad in (torch.ones(2, device="cuda"), torch.ones(1, device="cuda", dtype=torch.float64), torch.ones(1)):
        with pytest.raises(RuntimeError, match="lr"):
            K.sgd_step_(w, g, bad)


# ------------------------------------------------------------------ constant schedule == constant lr, bit for bit
def _batches(steps):
    from shallowspeed_b200.dataset import synthetic_mnist

    x, y = synthetic_mnist(n=128 * steps)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    return [(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(steps)]


def _train(sizes, batches, lr, pipelined=False, **kw):
    from shallowspeed_b200.parallel.engine import Trainer

    tr = Trainer(sizes, lr=lr, **kw)
    if pipelined:
        losses = [tr.step_pipelined(x, y) for x, y in batches][1:] + [tr.flush()]
    else:
        losses = [tr.step(x, y) for x, y in batches]
    tr.synchronize()
    torch.cuda.synchronize()
    return tr, losses


CONST = [(sizes, mom, prec, graph) for sizes in ("ref", "wide") for mom in (False, True) for prec in ("fp32", "tf32")
         for graph in (True, False)]


@pytest.mark.parametrize("sizes,mom,precision,graph", CONST)
def test_constant_schedule_is_bitwise_a_constant_lr(sizes, mom, precision, graph):
    sizes = {"ref": SIZES, "wide": WIDE}[sizes]
    batches = _batches(5)
    kw = dict(precision=precision, use_graph=graph)
    if mom:
        kw.update(momentum=MU, weight_decay=WD, nesterov=True)
    c = 0.03
    a, la = _train(sizes, batches, c, **kw)
    # built with another rate: the schedule's constant reaches every update through the slots alone
    b, lb = _train(sizes, batches, 0.5, lr_schedule=lambda i: c, **kw)
    assert b.optimizer.lr == c and b.lr == c and b.engine.lr() == pytest.approx(c)
    assert la == lb
    assert torch.equal(a.model.arena.weights, b.model.arena.weights)
    if mom:
        assert torch.equal(a.model.arena.momentum, b.model.arena.momentum)
    e, f = a.engine, b.engine
    assert e.kernels_per_step() == f.kernels_per_step() and e.graph_nodes() == f.graph_nodes()
    assert e.plan_text(0) == f.plan_text(0) and e.plan_text(1) == f.plan_text(1)
    assert f"lr={c:g}" in b.engine.describe()


# ------------------------------------------------------------------ a rate per step against the CPU oracle
def _oracle_pair(schedule_cls, steps, opt_kw, n_mu=4, precision="fp32"):
    """The native engine and the Python VM on the CPU, one step at a time under ``RATES``; yields after every step."""
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import Worker

    x, y = synthetic_mnist(n=128 * steps)
    runs = {}
    for dev in ("cpu", "cuda"):
        model = MLP(SIZES, 0, 1, 128).to(dev)
        opt = SGD(model.parameters(), 0.5, arena=model.arena, **opt_kw)     # the build-time rate is never used
        ds = Dataset(None, 128, 128 // n_mu, device=dev)
        ds.local_batch_size = 128
        ds.from_arrays(x, y)
        w = Worker(None, None, model, ds, opt) if dev == "cpu" else NativeWorker(None, None, model, ds, opt,
                                                                                precision=precision)
        runs[dev] = (model, opt, w)
    for b in range(steps):
        before = runs["cuda"][0].arena.weights.clone()
        for dev in ("cpu", "cuda"):
            model, opt, w = runs[dev]
            opt.lr = RATES[b]
            w.execute(schedule_cls(n_mu, 1, 0), b)
        runs["cuda"][2].sync_to_model()
        yield b, before, runs["cpu"][0], runs["cuda"][0]


@pytest.mark.parametrize("sched", ["naive", "gpipe"])
@pytest.mark.parametrize("stateful", [False, True])
def test_varying_rate_matches_the_cpu_oracle(sched, stateful):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS

    opt_kw = dict(momentum=MU, weight_decay=1e-3, nesterov=True) if stateful else {}
    init = MLP(SIZES, 0, 1, 128)
    for b, before, mc, mg in _oracle_pair(SCHEDULE_NAME_TO_CLS[sched], len(RATES), opt_kw):
        if RATES[b] == 0.0:
            assert torch.equal(mg.arena.weights, before), f"step {b}: lr == 0 changed the weights"
        for p0, pc, pg in zip(init.parameters(), mc.parameters(), mg.parameters()):
            assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL["fp32"], b
        if stateful:
            assert _frob(mg.arena.momentum.cpu(), mc.arena.momentum) < UPD_TOL["fp32"], b


# ------------------------------------------------------------------ pipelined steps keep their own rates
SCHEDULES = {
    "varying": lambda i: RATES[i % len(RATES)],
    "drop-at-3": lambda i: 0.05 if i < 3 else 0.01,        # a staging set that kept the old value fails here
}


@pytest.mark.parametrize("name", sorted(SCHEDULES))
@pytest.mark.parametrize("graph", [True, False])
def test_pipelined_steps_match_synchronous_steps(name, graph):
    batches = _batches(7)
    kw = dict(lr_schedule=SCHEDULES[name], use_graph=graph, momentum=MU, weight_decay=1e-3)
    a, la = _train(SIZES, batches, 0.5, **kw)
    b, lb = _train(SIZES, batches, 0.5, pipelined=True, **kw)
    assert la == lb
    assert torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert torch.equal(a.model.arena.momentum, b.model.arena.momentum)
    c, _ = _train(SIZES, batches, 0.05, use_graph=graph, momentum=MU, weight_decay=1e-3)
    assert not torch.equal(a.model.arena.weights, c.model.arena.weights)     # the schedule did change the run


def test_run_without_staging_writes_the_slot():
    """``run()`` without ``stage_inputs()`` re-runs the same staging set: it must write and order that set's slot."""
    batches = _batches(1)
    tr, _ = _train(SIZES, batches, 0.05)
    eng = tr.engine
    w0 = tr.model.arena.weights.clone()
    eng.set_lr(0.0)
    eng.run()
    eng.synchronize()
    assert torch.equal(tr.model.arena.weights, w0)
    eng.set_lr(0.05)
    eng.run()
    eng.synchronize()
    w1 = tr.model.arena.weights.clone()
    assert not torch.equal(w1, w0)
    eng.set_lr(0.0)
    eng.run()
    eng.run()
    eng.synchronize()
    assert torch.equal(tr.model.arena.weights, w1)


# ------------------------------------------------------------------ data-parallel kernels, peers replayed, a rate per step
DP_RATES = (0.125, 0.0, 0.375)       # the replica is built with 0.5 (test_gpu_dp_replay.LR)


def _replay_with_rates(case, sizes, dp, rank, protocol, monkeypatch, **kw):
    """``test_gpu_dp_replay._run`` with one rate per step: before each step the optimizer's rate (which the engine
    takes) and the rate of the harness's fp64 SGD oracle both become the step's rate, so every owned update, every
    phase-C line and every published tile is checked at the rate that step ran with."""
    import test_gpu_dp_replay as R

    from shallowspeed_b200.parallel.engine import NativeWorker

    rates = iter(DP_RATES)
    step_from = NativeWorker.step_from

    def step_at_rate(self, sched, x, y):
        lr = next(rates)
        monkeypatch.setattr(R, "LR", lr)
        self.optimizer.lr = lr
        return step_from(self, sched, x, y)

    monkeypatch.setattr(NativeWorker, "step_from", step_at_rate)
    R._run(case, sizes, dp, rank, protocol, monkeypatch=monkeypatch, steps=len(DP_RATES), **kw)
    assert next(rates, None) is None


@pytest.mark.parametrize("dp,rank,stateful", [(2, 1, False), (4, 2, True), (8, 5, False)])
def test_ll_replay_at_per_step_rates(dp, rank, stateful, monkeypatch):
    from test_gpu_dp_replay import REF

    _replay_with_rates(f"lr ll dp{dp} r{rank}", REF, dp, rank, "ll", monkeypatch, env={"SSB_DP_GATE": "1"},
                       mb_rows=128 // dp // 4, n_mu=4, stateful=stateful)


@pytest.mark.parametrize("shot,stateful", [("one-shot", False), ("two-shot", False), ("two-shot", True)])
def test_flag_replay_at_per_step_rates(shot, stateful, monkeypatch):
    from test_gpu_dp_replay import REF

    env = {"SSB_DP_LL": "0", "SSB_DP_ONE_SHOT" if shot == "one-shot" else "SSB_DP_TWO_SHOT": "1"}
    _replay_with_rates(f"lr flags {shot}", REF, 2, 1, shot, monkeypatch, env=env, stateful=stateful)


def test_flag_replay_wide_at_per_step_rates(monkeypatch):
    from test_gpu_dp_replay import WIDE as W

    _replay_with_rates("lr flags wide dp1", W, 1, 0, "one-shot+two-shot", monkeypatch)
