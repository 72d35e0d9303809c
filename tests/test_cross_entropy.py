"""Softmax cross-entropy on the CPU: the functional references against torch, one Python VM step against torch
autograd, layout equivalence of the VM, and the validation / CLI / checkpoint plumbing of the ``loss`` setting."""
import os
import subprocess
import sys
import threading

import pytest
import torch
import torch.nn.functional as TF

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.layers import MLP, CrossEntropyLoss
from shallowspeed_b200.ops import functional as F
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.parallel.comm import ProcessGrid, ThreadFabric
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule, Worker
from shallowspeed_b200.utils import assert_sync, get_model_hash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
GBS, N_MU, LR, STEPS = 128, 4, 0.05, 4
_X, _Y = synthetic_mnist(n=GBS * STEPS)


def _torch_ce(z, t, batch):
    """torch's loss and its autograd gradient: F.cross_entropy with probability targets, summed, over the batch."""
    z = z.detach().clone().requires_grad_(True)
    loss = TF.cross_entropy(z, t, reduction="sum") / batch
    loss.backward()
    return loss.detach(), z.grad


def _logits(rows=24, classes=10, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, classes, generator=g, dtype=torch.float64) * 3.0, g


@pytest.mark.parametrize("soft", [False, True], ids=["one-hot", "soft"])
def test_refs_match_torch_cross_entropy(soft):
    z, g = _logits()
    if soft:
        t = torch.rand(z.shape, generator=g, dtype=torch.float64)
        t = t / t.sum(1, keepdim=True) * 0.9                        # sum(t) != 1 as well: the rule holds for any t
    else:
        t = TF.one_hot(torch.randint(0, z.shape[1], (z.shape[0],), generator=g), z.shape[1]).double()
    loss, grad = _torch_ce(z, t, 64)
    assert torch.allclose(F.cross_entropy_ref(z, t, 64), loss, rtol=1e-13, atol=0)
    assert torch.allclose(F.cross_entropy_grad_ref(z, t, 64), grad, rtol=1e-12, atol=1e-16)
    assert torch.allclose(F.row_softmax_ref(z), torch.softmax(z, -1), rtol=1e-13, atol=0)
    dz, p, lv = F.loss_head_backward(z, t, 64, loss="cross_entropy")
    assert torch.equal(dz, F.cross_entropy_grad_ref(z, t, 64)) and torch.equal(lv, F.cross_entropy_ref(z, t, 64))
    assert torch.equal(p, F.row_softmax_ref(z))
    # the dispatching entry points take the reference on the CPU
    assert torch.equal(F.cross_entropy(z, t, 64), lv) and torch.equal(F.cross_entropy_grad(z, t, 64), dz)
    assert torch.equal(F.row_softmax(z), p)


def test_far_row_keeps_its_own_softmax():
    """A row whose logits lie 200 below another row's: the micro-batch-max softmax of the MSE contract underflows it to
    0 (and +1e-7 makes up its loss); the per-row contract keeps torch's values."""
    z, g = _logits(rows=8)
    z[3] -= 200.0
    t = TF.one_hot(torch.randint(0, z.shape[1], (z.shape[0],), generator=g), z.shape[1]).double()
    loss, grad = _torch_ce(z, t, 8)
    assert torch.allclose(F.cross_entropy_ref(z, t, 8), loss, rtol=1e-13, atol=0)
    assert torch.allclose(F.cross_entropy_grad_ref(z, t, 8), grad, rtol=1e-12, atol=1e-16)
    assert float(F.row_softmax_ref(z)[3].sum()) == pytest.approx(1.0, abs=1e-15)
    assert float(F.softmax_ref(z)[3].sum()) < 1e-40                 # what the global-max contract would give the row


# ------------------------------------------------------------------ the VM against torch autograd
def _torch_train(steps, relu_logits=False):
    """``steps`` SGD steps of nn.Linear + ReLU + F.cross_entropy from the MLP's initial weights on the batches the VM
    reads (batch b = rows [b * GBS, (b + 1) * GBS)); returns ([W, b] of every layer, the last step's loss)."""
    init = MLP(SIZES, 0, 1, GBS, loss="cross_entropy")
    ref = [(torch.nn.Parameter(l._params["W"].data.clone()), torch.nn.Parameter(l._params["b"].data.reshape(-1).clone()))
           for l in init.linears]
    for step in range(steps):
        rows = slice(step * GBS, (step + 1) * GBS)
        a, t = torch.as_tensor(_X[rows]).float(), torch.as_tensor(_Y[rows]).float()
        for i, (W, b) in enumerate(ref):
            a = a @ W.T + b
            if i < len(ref) - 1 or relu_logits:
                a = torch.relu(a)
        loss = TF.cross_entropy(a, t, reduction="sum") / GBS
        loss.backward()
        with torch.no_grad():
            for W, b in ref:
                W -= LR * W.grad
                b -= LR * b.grad
                W.grad, b.grad = None, None
    return [p.detach() for pair in ref for p in pair], float(loss.detach())


def _assert_params_close(got, ref, tol=2e-6):
    assert len(got) == len(ref)
    for x, y in zip(got, ref):
        assert float((x.reshape(y.shape) - y).abs().max()) < tol


def test_vm_step_matches_torch_autograd():
    model = MLP(SIZES, 0, 1, GBS, loss="cross_entropy")
    assert isinstance(model.loss_layer, CrossEntropyLoss) and model.loss == "cross_entropy"
    opt = SGD(model.parameters(), LR, arena=model.arena)
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(_X, _Y)
    worker = Worker(None, None, model, ds, opt)
    worker.execute(NaiveParallelSchedule(N_MU, 1, 0), 0)
    ref, loss = _torch_train(1)
    assert worker.batch_loss() == pytest.approx(loss, rel=1e-5)
    _assert_params_close([p.data for p in model.parameters()], ref)


def test_forward_output_is_the_row_softmax():
    model = MLP([20, 16, 5], 0, 1, 8, loss="cross_entropy")
    x = torch.randn(8, 20)
    z = torch.relu(x @ model.linears[0]._params["W"].data.T + model.linears[0]._params["b"].data)
    z = z @ model.linears[1]._params["W"].data.T + model.linears[1]._params["b"].data
    assert torch.allclose(model.forward(x), torch.softmax(z, -1), rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------ Python VM layouts
def run_layout(dp, pp, sched_cls, sizes=SIZES, steps=STEPS):
    dp_fabrics = [ThreadFabric(dp) for _ in range(pp)]
    pp_fabrics = [ThreadFabric(pp) for _ in range(dp)]
    results, errors = {}, []

    def rank_main(rank):
        try:
            torch.set_num_threads(1)
            grid = ProcessGrid(dp, pp, rank)
            dp_comm = dp_fabrics[grid.stage].comm(grid.replica)
            pp_comm = pp_fabrics[grid.replica].comm(grid.stage)
            model = MLP(sizes, grid.stage, pp, GBS, loss="cross_entropy")
            opt = SGD(model.parameters(), LR, arena=model.arena)
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


@pytest.mark.parametrize("dp,pp,cls", [(2, 1, NaiveParallelSchedule), (4, 1, GPipeSchedule), (1, 2, GPipeSchedule),
                                       (1, 4, PipeDreamSchedule), (2, 2, GPipeSchedule)])
def test_vm_layouts_match_sequential(sequential, dp, pp, cls):
    _assert_params_close(run_layout(dp, pp, cls), sequential)


def test_sequential_matches_torch_autograd(sequential):
    _assert_params_close(sequential, _torch_train(STEPS)[0], tol=5e-6)


@pytest.mark.parametrize("dp", [1, 2])
def test_vm_pp8_loss_only_last_stage(dp):
    """pp = 8 on 8 sizes: stage 7 holds nothing but the loss, and the last Linear (on stage 6) keeps its ReLU, as in the
    reference's partitioner - so the model is torch's with a ReLU on the logits."""
    assert MLP(SIZES, 7, 8, GBS, loss="cross_entropy").linears == []
    _assert_params_close(run_layout(dp, 8, GPipeSchedule), _torch_train(STEPS, relu_logits=True)[0], tol=5e-6)


def test_cross_entropy_changes_the_trajectory(sequential):
    """The layouts above do not train the MSE model by mistake."""
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena)
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(_X, _Y)
    worker = Worker(None, None, model, ds, opt)
    for b in range(STEPS):
        worker.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    assert max(float((p.data - q).abs().max()) for p, q in zip(model.parameters(), sequential)) > 1e-4


# ------------------------------------------------------------------ validation, CLI, checkpoints
@pytest.mark.parametrize("bad", ["cross-entropy", "CE", "nll", ""])
def test_unknown_loss_raises(bad):
    with pytest.raises(ValueError, match="loss"):
        MLP(SIZES, 0, 1, GBS, loss=bad)
    with pytest.raises(ValueError, match="loss"):
        F.loss_head_backward(torch.zeros(2, 3), torch.zeros(2, 3), 2, loss=bad)


def test_trainer_rejects_unknown_loss():
    from shallowspeed_b200.parallel.engine import Trainer

    with pytest.raises(ValueError, match="loss"):
        Trainer(SIZES, device="cpu", loss="hinge")


def test_mse_is_the_default():
    m = MLP(SIZES, 0, 1, GBS)
    assert m.loss == "mse" and type(m.loss_layer).__name__ == "MSELoss"
    assert MLP(SIZES, 0, 2, GBS, loss="cross_entropy").loss == "cross_entropy"   # every stage records it
    assert MLP(SIZES, 0, 2, GBS, loss="cross_entropy").loss_layer is None


def _cli(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable, "train.py"] + args, cwd=ROOT, env=env, capture_output=True, text=True,
                          timeout=timeout)


def test_train_cli_loss_flag_and_resume(tmp_path):
    base = ["--device", "cpu", "--engine", "python", "--no-eval", "--synthetic"]
    r = _cli(base + ["--steps", "2", "--loss", "cross-entropy", "--save", str(tmp_path / "ce")])
    assert r.returncode == 0, r.stderr[-2000:]
    assert "CrossEntropyLoss()" in r.stdout
    assert torch.load(tmp_path / "ce" / "stage0of1.pt")["hparams"]["loss"] == "cross_entropy"
    r = _cli(base + ["--steps", "2", "--save", str(tmp_path / "mse")])
    assert r.returncode == 0, r.stderr[-2000:]
    assert torch.load(tmp_path / "mse" / "stage0of1.pt")["hparams"]["loss"] == "mse"
    # a cross-entropy run continues a cross-entropy checkpoint, and refuses an MSE one
    r = _cli(base + ["--steps", "3", "--loss", "cross-entropy", "--resume", str(tmp_path / "ce")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _cli(base + ["--steps", "3", "--loss", "cross-entropy", "--resume", str(tmp_path / "mse")])
    assert r.returncode != 0 and "checkpoint was written with loss='mse'" in (r.stderr + r.stdout)
    r = _cli(base + ["--steps", "1", "--loss", "ce"])
    assert r.returncode != 0 and "--loss" in r.stderr


def test_checkpoint_without_loss_key_loads_as_mse(tmp_path):
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    m = MLP(SIZES, 0, 1, GBS)
    save_stage(m, tmp_path, 0, 1, step=3, hparams={"lr": LR})     # a checkpoint from before the loss setting
    assert "loss" not in torch.load(tmp_path / "stage0of1.pt")["hparams"]
    assert load_stage(MLP(SIZES, 0, 1, GBS), tmp_path, 0, 1, expect_hparams={"lr": LR, "loss": "mse"}) == 3
    with pytest.raises(ValueError, match="loss"):
        load_stage(MLP(SIZES, 0, 1, GBS, loss="cross_entropy"), tmp_path, 0, 1,
                   expect_hparams={"lr": LR, "loss": "cross_entropy"})
    # round trip of a cross-entropy checkpoint
    ce = MLP(SIZES, 0, 1, GBS, loss="cross_entropy")
    ce.arena.weights.add_(0.5)
    save_stage(ce, tmp_path / "ce", 0, 1, step=5, hparams={"lr": LR, "loss": "cross_entropy"})
    back = MLP(SIZES, 0, 1, GBS, loss="cross_entropy")
    assert load_stage(back, tmp_path / "ce", 0, 1, expect_hparams={"lr": LR, "loss": "cross_entropy"}) == 5
    assert torch.equal(back.arena.weights, ce.arena.weights)
