"""Residual connections: Linear / MLP forward and backward against torch autograd in fp64, which layers get a skip,
sequential == DP == PP == DP x PP in the Python VM, residual=False unchanged, and train.py (flag, resume, refusals)."""
import os
import subprocess
import sys
import threading

import pytest
import torch
import torch.nn.functional as TF

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.layers import MLP
from shallowspeed_b200.models.layers import Linear
from shallowspeed_b200.models.mlp import residual_layers
from shallowspeed_b200.ops import functional as F
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.parallel.comm import ProcessGrid, ThreadFabric
from shallowspeed_b200.parallel.worker import Worker
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule
from shallowspeed_b200.utils import assert_sync, get_model_hash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["relu", "gelu", "silu", "tanh"]
TORCH_F = {"relu": torch.relu, "gelu": lambda z: TF.gelu(z, approximate="none"), "silu": TF.silu, "tanh": torch.tanh}
REF_SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
RES_SIZES = [784, 48, 48, 48, 48, 48, 48, 10]        # 8 sizes: pp 1, 2, 4 and 8 all divide them
P, SEED = 0.3, 0x0BAD_5EED_1234_5678


# ------------------------------------------------------------------ modules against autograd
def _double(lin):
    lin.arena.weights = lin.arena.weights.double()
    lin.arena.grads = lin.arena.grads.double()
    lin._bind()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("p", [0.0, 0.4])
def test_linear_forward_and_backward_match_autograd(kind, p):
    lin = Linear(6, 6, activation=kind, residual=True)
    _double(lin)
    gen = torch.Generator().manual_seed(7)
    lin._params["b"].data.copy_(torch.randn(1, 6, dtype=torch.float64, generator=gen))
    x = torch.randn(4, 6, dtype=torch.float64, generator=gen) * 2
    g = torch.randn(4, 6, dtype=torch.float64, generator=gen)
    keep, s = torch.ones(4, 6, dtype=torch.bool), 1.0
    if p > 0:
        s = F.dropout_scale(p)
        lin.dropout = (p, 5, 3, s)
        lin.dropout_rows = (torch.arange(4), 2)
        keep = F.dropout_mask(p, 5, 3, 2, torch.arange(4), 6)
        assert 0 < int(keep.sum()) < keep.numel()
    W = lin._params["W"].data.clone().requires_grad_(True)
    b = lin._params["b"].data.clone().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    ref = xr + TORCH_F[kind](xr @ W.T + b) * keep * s
    ref_dx, ref_dw, ref_db = torch.autograd.grad((g * ref).sum(), (xr, W, b))
    lin.zero_grad()
    out = lin.forward(x)
    assert torch.allclose(out, ref.detach(), rtol=1e-13, atol=1e-13)
    dx = lin.backward(g)
    assert torch.allclose(dx, ref_dx, rtol=1e-12, atol=1e-13)
    assert torch.allclose(lin._params["W"].grad, ref_dw, rtol=1e-12, atol=1e-13)
    assert torch.allclose(lin._params["b"].grad, ref_db, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("p", [0.0, 0.3])
def test_mlp_forward_and_backward_match_autograd(kind, p):
    sizes = [5, 7, 7, 6, 6, 3]
    m = MLP(sizes, 0, 1, 4, activation=kind, residual=True, dropout=p, dropout_seed=11)
    assert [lin.residual for lin in m.linears] == [False, True, False, True, False]
    m.arena.weights, m.arena.grads = m.arena.weights.double(), m.arena.grads.double()
    for lin in m.linears:
        lin._bind()
    gen = torch.Generator().manual_seed(1)
    for lin in m.linears:
        lin._params["b"].data.copy_(torch.randn(1, lin.out_dims, dtype=torch.float64, generator=gen))
    x = torch.randn(4, 5, dtype=torch.float64, generator=gen)
    t = torch.softmax(torch.randn(4, 3, dtype=torch.float64, generator=gen), 1)
    params = [(lin._params["W"].data.clone().requires_grad_(True), lin._params["b"].data.clone().requires_grad_(True))
              for lin in m.linears]
    a = x
    for i, ((W, b), lin) in enumerate(zip(params, m.linears)):
        z = a @ W.T + b
        if lin.activation is None:
            a = z
            continue
        keep, s = torch.ones_like(z, dtype=torch.bool), 1.0
        if p > 0:
            keep, s = F.dropout_mask(p, 11, i, 0, torch.arange(4), z.shape[1]), F.dropout_scale(p)
        br = TORCH_F[kind](z) * keep * s
        a = a + br if lin.residual else br
    e = torch.exp(a - a.max().detach())                         # the reference head: a constant global max shift, + eps
    prob = e / (e.sum(dim=1, keepdim=True) + F.SOFTMAX_EPS)
    loss = ((t - prob) ** 2).sum() / 4
    grads = torch.autograd.grad(loss, [q for pair in params for q in pair])
    m.zero_grad()
    out = m.forward(x, 0)
    assert torch.allclose(out, prob.detach(), rtol=1e-12, atol=1e-13)
    m.backward(t, 0)
    for i, lin in enumerate(m.linears):
        assert torch.allclose(lin._params["W"].grad, grads[2 * i], rtol=1e-10, atol=1e-12), i
        assert torch.allclose(lin._params["b"].grad, grads[2 * i + 1], rtol=1e-10, atol=1e-12), i


# ------------------------------------------------------------------ which layers, and refusals
def test_residual_layers_follow_the_activation_rule():
    assert residual_layers(RES_SIZES) == [1, 2, 3, 4, 5]
    assert residual_layers([784, 128, 128, 10, 10]) == [1]          # the 10 -> 10 logits carry no activation
    assert residual_layers(REF_SIZES) == []
    for pp in (1, 2, 4, 8):
        got = [lin.residual for s in range(pp) for lin in MLP(RES_SIZES, s, pp, 64, residual=True).linears]
        assert got == [False, True, True, True, True, True, False]
        assert residual_layers(RES_SIZES, pp) == [1, 2, 3, 4, 5]


def test_refusals():
    for pp in (1, 2, 8):
        for s in range(pp):
            with pytest.raises(ValueError, match="no Linear"):
                MLP(REF_SIZES, s, pp, 128, residual=True)
    for bad in (1, 0, "yes", None):
        with pytest.raises(ValueError):
            MLP(RES_SIZES, 0, 1, 64, residual=bad)
        with pytest.raises(ValueError):
            Linear(4, 4, residual=bad)
    with pytest.raises(ValueError):
        Linear(4, 5, residual=True)
    with pytest.raises(ValueError):
        Linear(4, 4, activation=None, residual=True)
    from shallowspeed_b200.parallel.engine import Trainer

    with pytest.raises(ValueError):
        Trainer(REF_SIZES, residual=True, device="cpu")


def test_residual_false_is_the_current_model_bit_for_bit():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(16, 784, generator=gen)
    t = torch.softmax(torch.randn(16, 10, generator=gen), 1)
    for sizes in (REF_SIZES, RES_SIZES):
        for kind in ("relu", "gelu"):
            a = MLP(sizes, 0, 1, 16, activation=kind, dropout=0.2, dropout_seed=3)
            b = MLP(sizes, 0, 1, 16, activation=kind, dropout=0.2, dropout_seed=3, residual=False)
            assert not any(lin.residual for lin in b.linears)
            assert [repr(l) for l in a.layers] == [repr(l) for l in b.layers]
            assert torch.equal(a.forward(x, 0), b.forward(x, 0))
            assert torch.equal(a.backward(t, 0), b.backward(t, 0))
            assert torch.equal(a.arena.grads, b.arena.grads)


def test_residual_changes_the_model():
    x = torch.randn(8, 784, generator=torch.Generator().manual_seed(2))
    a = MLP(RES_SIZES, 0, 1, 8)
    b = MLP(RES_SIZES, 0, 1, 8, residual=True)
    assert torch.equal(a.arena.weights, b.arena.weights)
    assert not torch.equal(a.forward(x, 0), b.forward(x, 0))


# ------------------------------------------------------------------ sequential == DP == PP == DP x PP
GBS, N_MU, LR, STEPS = 64, 4, 0.05, 4
_X, _Y = synthetic_mnist(n=GBS * STEPS)


def run_layout(sizes, dp, pp, sched_cls, residual=True, activation="relu", dropout=0.0, steps=STEPS):
    """A copy of test_equivalence.run_layout that takes the model's sizes and settings: the parameters of replica 0 of
    every stage after ``steps`` steps (replicas must be bit-identical)."""
    dp_fabrics = [ThreadFabric(dp) for _ in range(pp)]
    pp_fabrics = [ThreadFabric(pp) for _ in range(dp)]
    results, errors = {}, []

    def rank_main(rank):
        try:
            torch.set_num_threads(1)
            grid = ProcessGrid(dp, pp, rank)
            dp_comm = dp_fabrics[grid.stage].comm(grid.replica)
            pp_comm = pp_fabrics[grid.replica].comm(grid.stage)
            model = MLP(sizes, grid.stage, pp, GBS, residual=residual, activation=activation, dropout=dropout,
                        dropout_seed=SEED)
            opt = SGD(model.parameters(), LR, arena=model.arena)
            ds = Dataset(None, GBS, GBS // dp // N_MU)
            ds.local_batch_size = GBS // dp
            ds = ds.from_arrays(_X[grid.replica::dp], _Y[grid.replica::dp])
            worker = Worker(dp_comm, pp_comm, model, ds, opt)
            sched = sched_cls(N_MU, pp, grid.stage)
            for b in range(steps):
                model.dropout_step = b
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


def _close(a, b, tol=2e-6):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert float((x - y).abs().max()) < tol, float((x - y).abs().max())


_SEQ = {}


@pytest.mark.parametrize("kind,dropout", [("relu", 0.0), ("gelu", P)])
@pytest.mark.parametrize("dp,pp,cls", [
    (2, 1, NaiveParallelSchedule), (1, 2, GPipeSchedule), (1, 4, PipeDreamSchedule), (2, 2, GPipeSchedule),
    (2, 4, GPipeSchedule), (4, 2, PipeDreamSchedule),
])
def test_layout_matches_sequential(kind, dropout, dp, pp, cls):
    key = (kind, dropout)
    if key not in _SEQ:
        _SEQ[key] = run_layout(RES_SIZES, 1, 1, NaiveParallelSchedule, activation=kind, dropout=dropout)
    _close(run_layout(RES_SIZES, dp, pp, cls, activation=kind, dropout=dropout), _SEQ[key])


def test_the_vm_trains_a_different_model_with_skips():
    a = run_layout(RES_SIZES, 1, 1, NaiveParallelSchedule, residual=False, steps=2)
    b = run_layout(RES_SIZES, 1, 1, NaiveParallelSchedule, residual=True, steps=2)
    assert any(not torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------ train.py
def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


CLI = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic", "--hidden", "32", "--n-layers", "4"]


def test_train_cli_resume_is_bitwise_and_refuses_a_mismatch(tmp_path):
    res = ["--residual", "--activation", "gelu"]
    for args in (["--steps", "5", "--save", str(tmp_path / "full")], ["--steps", "2", "--save", str(tmp_path / "part")],
                 ["--steps", "5", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(CLI + res + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 5 and a["hparams"]["residual"] is True
    assert torch.equal(a["weights"], b["weights"])
    r = _run(CLI + ["--activation", "gelu", "--steps", "5", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with residual" in (r.stderr + r.stdout)


def test_train_cli_checkpoint_without_the_key_counts_as_plain(tmp_path):
    r = _run(CLI + ["--steps", "2", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    path = tmp_path / "part" / "stage0of1.pt"
    ck = torch.load(path)
    assert ck["hparams"]["residual"] is False
    del ck["hparams"]["residual"]
    torch.save(ck, path)
    r = _run(CLI + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(CLI + ["--residual", "--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with residual" in (r.stderr + r.stdout)


def test_train_cli_refuses_residual_on_the_reference_sizes():
    r = _run(["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic", "--residual", "--steps", "1"])
    assert r.returncode != 0 and "ValueError" in r.stderr and "no Linear" in r.stderr


def test_train_cli_spawn_dp2_pp2_on_the_cpu():
    r = _run(["train.py", "--device", "cpu", "--spawn", "--dp", "2", "--pp", "2", "--no-eval", "--synthetic", "--hidden",
              "64", "--n-layers", "7", "--residual", "--activation", "gelu", "--steps", "3"])
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
