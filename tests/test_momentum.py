"""SGD momentum / Nesterov / weight decay on the CPU: the arena optimizer against torch.optim.SGD, input validation,
the CLI flags, layout equivalence of the Python VM and checkpoint round trips."""
import os
import subprocess
import sys
import threading

import pytest
import torch

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.layers import MLP
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.parallel.comm import ProcessGrid, ThreadFabric
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule, Worker
from shallowspeed_b200.utils import assert_sync, get_model_hash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
GBS, N_MU, LR = 128, 4, 0.05
_X, _Y = synthetic_mnist(n=GBS * 6)

COMBOS = [(mu, wd, nest) for mu in (0.0, 0.9) for wd in (0.0, 1e-2) for nest in (False, True) if not (nest and mu == 0.0)]


@pytest.mark.parametrize("mu,wd,nesterov", COMBOS)
def test_arena_sgd_matches_torch_sgd_bitwise(mu, wd, nesterov):
    model = MLP(SIZES, 0, 1, GBS)
    params = list(model.parameters())
    ref = [torch.nn.Parameter(p.data.clone()) for p in params]
    opt = SGD(params, LR, momentum=mu, weight_decay=wd, nesterov=nesterov, arena=model.arena)
    topt = torch.optim.SGD(ref, lr=LR, momentum=mu, weight_decay=wd, nesterov=nesterov)
    gen = torch.Generator().manual_seed(0)
    for _ in range(10):
        for p, r in zip(params, ref):
            g = torch.randn(p.data.shape, generator=gen)
            p.grad.copy_(g)
            r.grad = g.clone()
        opt.step()
        topt.step()
    for p, r in zip(params, ref):
        assert torch.equal(p.data, r.data)


def test_plain_sgd_is_todays_update_bitwise():
    model = MLP(SIZES, 0, 1, GBS)
    w0 = model.arena.weights.clone()
    g = torch.randn(model.arena.grads.shape, generator=torch.Generator().manual_seed(1))
    model.arena.grads.copy_(g)
    SGD(model.parameters(), LR, momentum=0.0, weight_decay=0.0, arena=model.arena).step()
    assert torch.equal(model.arena.weights, w0.add(g, alpha=-LR))
    assert model.arena.momentum is None                  # no state, no memory


def test_per_parameter_path_matches_arena_path():
    a, b = MLP(SIZES, 0, 1, GBS), MLP(SIZES, 0, 1, GBS)
    oa = SGD(a.parameters(), LR, momentum=0.9, weight_decay=1e-2, nesterov=True, arena=a.arena)
    ob = SGD(b.parameters(), LR, momentum=0.9, weight_decay=1e-2, nesterov=True)
    gen = torch.Generator().manual_seed(2)
    for _ in range(3):
        g = torch.randn(a.arena.grads.shape, generator=gen)
        a.arena.grads.copy_(g)
        b.arena.grads.copy_(g)
        oa.step()
        ob.step()
    for p, q in zip(a.parameters(), b.parameters()):
        assert float((p.data - q.data).abs().max()) < 1e-6


@pytest.mark.parametrize("kw", [dict(momentum=1.0), dict(momentum=-0.1), dict(weight_decay=-1e-4),
                                dict(nesterov=True), dict(momentum=0.0, nesterov=True)])
def test_bad_hyperparameters_raise(kw):
    model = MLP(SIZES, 0, 1, GBS)
    with pytest.raises(ValueError):
        SGD(model.parameters(), LR, arena=model.arena, **kw)


def test_momentum_buffer_follows_the_arena():
    model = MLP(SIZES, 0, 1, GBS)
    SGD(model.parameters(), LR, momentum=0.9, arena=model.arena)
    v = model.arena.momentum
    assert v is not None and v.numel() == model.arena.numel and v.dtype == torch.float32
    assert model.arena.momentum_block(0).shape == model.arena.block(0).shape
    w2 = torch.zeros_like(model.arena.weights)
    model.arena.rebind(w2, torch.zeros_like(model.arena.grads))
    assert model.arena.momentum is v                      # same device: the buffer stays where it is


def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_train_cli_momentum_flags(tmp_path):
    r = _run(["train.py", "--device", "cpu", "--engine", "python", "--steps", "2", "--no-eval", "--synthetic",
              "--momentum", "0.9", "--nesterov", "--weight-decay", "1e-4", "--save", str(tmp_path / "ck")])
    assert r.returncode == 0, r.stderr[-2000:]
    ck = torch.load(tmp_path / "ck" / "stage0of1.pt")
    assert ck["hparams"]["momentum"] == 0.9 and ck["hparams"]["nesterov"] is True
    assert ck["momentum"].shape == ck["weights"].shape and float(ck["momentum"].abs().sum()) > 0
    r = _run(["train.py", "--device", "cpu", "--steps", "1", "--no-eval", "--synthetic", "--nesterov"])
    assert r.returncode != 0 and "nesterov" in r.stderr


def test_train_cli_resume_with_momentum_is_bitwise(tmp_path):
    base = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic", "--momentum", "0.9",
            "--weight-decay", "1e-3"]
    for args in (["--steps", "4", "--save", str(tmp_path / "full")], ["--steps", "2", "--save", str(tmp_path / "part")],
                 ["--steps", "4", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(base + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 4
    assert torch.equal(a["weights"], b["weights"]) and torch.equal(a["momentum"], b["momentum"])
    r = _run(base[:-4] + ["--steps", "4", "--resume", str(tmp_path / "part"), "--momentum", "0.5", "--weight-decay", "1e-3"])
    assert r.returncode != 0 and "checkpoint was written with momentum" in (r.stderr + r.stdout)
    r = _run(base[:-4] + ["--steps", "4", "--resume", str(tmp_path / "part")])     # plain SGD on a momentum checkpoint
    assert r.returncode != 0 and "checkpoint was written with" in (r.stderr + r.stdout)


# ------------------------------------------------------------------ Python VM: layouts agree with momentum on
MOM = dict(momentum=0.9, weight_decay=1e-3, nesterov=True)


def run_layout(dp, pp, sched_cls, steps=4, opt_kw=MOM):
    dp_fabrics = [ThreadFabric(dp) for _ in range(pp)]
    pp_fabrics = [ThreadFabric(pp) for _ in range(dp)]
    results, errors = {}, []

    def rank_main(rank):
        try:
            torch.set_num_threads(1)
            grid = ProcessGrid(dp, pp, rank)
            dp_comm = dp_fabrics[grid.stage].comm(grid.replica)
            pp_comm = pp_fabrics[grid.replica].comm(grid.stage)
            model = MLP(SIZES, grid.stage, pp, GBS)
            opt = SGD(model.parameters(), LR, arena=model.arena, **opt_kw)
            ds = Dataset(None, GBS, GBS // dp // N_MU)
            ds.local_batch_size = GBS // dp
            ds.from_arrays(_X[grid.replica::dp], _Y[grid.replica::dp])
            worker = Worker(dp_comm, pp_comm, model, ds, opt)
            sched = sched_cls(N_MU, pp, grid.stage)
            for b in range(steps):
                worker.execute(sched, b)
            assert_sync(dp_comm, get_model_hash(model))
            results[rank] = [p.data.clone() for p in model.parameters()]
        except Exception as e:  # pragma: no cover
            errors.append((rank, e))
            for f in dp_fabrics + pp_fabrics:
                f.barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(dp * pp)]
    [t.start() for t in threads]
    [t.join(120) for t in threads]
    assert not errors, errors
    for rank in range(dp * pp):
        g = ProcessGrid(dp, pp, rank)
        for a, b in zip(results[rank], results[g.stage]):
            assert torch.equal(a, b), "DP replicas diverged"
    return [p for s in range(pp) for p in results[s]]


@pytest.fixture(scope="module")
def sequential():
    return run_layout(1, 1, NaiveParallelSchedule)


@pytest.mark.parametrize("dp,pp,cls", [(2, 1, NaiveParallelSchedule), (1, 2, GPipeSchedule), (1, 2, PipeDreamSchedule),
                                       (2, 2, GPipeSchedule)])
def test_vm_layouts_match_sequential_with_momentum(sequential, dp, pp, cls):
    got = run_layout(dp, pp, cls)
    for x, y in zip(got, sequential):
        assert float((x - y).abs().max()) < 2e-6


def test_vm_momentum_changes_the_trajectory(sequential):
    """The momentum runs above are not plain SGD in disguise."""
    plain = run_layout(1, 1, NaiveParallelSchedule, opt_kw={})
    assert max(float((x - y).abs().max()) for x, y in zip(plain, sequential)) > 1e-4


def test_checkpoint_roundtrip_in_process(tmp_path):
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    def fresh():
        model = MLP(SIZES, 0, 1, GBS)
        opt = SGD(model.parameters(), LR, arena=model.arena, **MOM)
        ds = Dataset(None, GBS, GBS // N_MU)
        ds.local_batch_size = GBS
        ds.from_arrays(_X, _Y)
        return model, Worker(None, None, model, ds, opt)

    hp = dict(lr=LR, **MOM)
    m1, w1 = fresh()
    for b in range(4):
        w1.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    m2, w2 = fresh()
    for b in range(2):
        w2.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    save_stage(m2, tmp_path, 0, 1, step=2, hparams=hp, momentum=m2.arena.momentum)
    m3, w3 = fresh()
    assert load_stage(m3, tmp_path, 0, 1, expect_hparams=hp) == 2
    for b in range(2, 4):
        w3.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    assert torch.equal(m1.arena.weights, m3.arena.weights) and torch.equal(m1.arena.momentum, m3.arena.momentum)
    with pytest.raises(ValueError, match="momentum"):
        load_stage(fresh()[0], tmp_path, 0, 1, expect_hparams=dict(hp, momentum=0.5))
