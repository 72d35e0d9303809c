"""GELU, SiLU and tanh hidden activations: the torch oracle (f and the gate f') against autograd, the gated modules with
and without dropout, sequential == DP == PP == DP x PP in the Python VM, and train.py (run, resume, refusals)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as TF

from shallowspeed_b200.layers import MLP
from shallowspeed_b200.ops import functional as F
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule

from test_equivalence import SIZES, _close, run_layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMOOTH = ["gelu", "silu", "tanh"]
TORCH_F = {"gelu": lambda z: TF.gelu(z, approximate="none"), "silu": TF.silu, "tanh": torch.tanh}
P, SEED = 0.3, 0x1234_5678_9ABC_DEF0


# ------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("kind", SMOOTH)
def test_activation_ref_matches_autograd_in_fp64(kind):
    z = torch.cat([torch.linspace(-12.0, 12.0, 2001, dtype=torch.float64),
                   torch.tensor([-1e4, -200.0, -40.0, 40.0, 200.0, 1e4, 0.0], dtype=torch.float64)])
    zg = z.clone().requires_grad_(True)
    ref = TORCH_F[kind](zg)
    (dref,) = torch.autograd.grad(ref.sum(), zg)
    a, g = F.activation_ref(kind, z)
    assert torch.allclose(a, ref.detach(), rtol=1e-14, atol=1e-14)
    assert torch.allclose(g, dref, rtol=1e-12, atol=1e-14)
    assert bool(torch.isfinite(g).all()) and bool(torch.isfinite(a).all())


@pytest.mark.parametrize("kind", SMOOTH)
def test_activation_ref_is_finite_in_fp32_at_large_magnitudes(kind):
    z = torch.tensor([-3e38, -1e6, -104.0, -89.0, -20.0, 20.0, 89.0, 104.0, 1e6, 3e38], dtype=torch.float32)
    a, g = F.activation_ref(kind, z)
    assert bool(torch.isfinite(g).all())
    assert torch.allclose(g, F.activation_ref(kind, z.double())[1].float(), atol=1e-6)


def test_unknown_activation_names_are_refused():
    for bad in ("leaky_relu", "GELU", "", None, 1):
        with pytest.raises(ValueError):
            F.check_activation(bad)
    with pytest.raises(ValueError):
        MLP(SIZES, 0, 1, 128, activation="elu")
    from shallowspeed_b200.models.layers import Linear

    with pytest.raises(ValueError):
        Linear(4, 3, activation="swish")


def test_trainer_refuses_an_unknown_activation():
    from shallowspeed_b200.parallel.engine import Trainer

    with pytest.raises(ValueError):
        Trainer(SIZES, activation="gelu_tanh", device="cpu")


# ------------------------------------------------------------------ modules
@pytest.mark.parametrize("kind", SMOOTH)
@pytest.mark.parametrize("p", [0.0, 0.4])
def test_linear_forward_and_backward_match_autograd(kind, p):
    from shallowspeed_b200.models.layers import Linear

    lin = Linear(6, 5, activation=kind)
    assert type(lin.activation).__name__ == {"gelu": "GELU", "silu": "SiLU", "tanh": "Tanh"}[kind]
    lin.arena.weights = lin.arena.weights.double()
    lin.arena.grads = lin.arena.grads.double()
    lin._bind()
    gen = torch.Generator().manual_seed(3)
    lin._params["b"].data.copy_(torch.randn(1, 5, dtype=torch.float64, generator=gen))
    x = torch.randn(3, 6, dtype=torch.float64, generator=gen) * 3
    g = torch.randn(3, 5, dtype=torch.float64, generator=gen)
    keep = torch.ones(3, 5, dtype=torch.bool)
    s = 1.0
    if p > 0:
        s = F.dropout_scale(p)
        lin.dropout = (p, 5, 0, s)
        lin.dropout_rows = (torch.arange(3), 2)
        keep = F.dropout_mask(p, 5, 0, 2, torch.arange(3), 5)
        assert 0 < int(keep.sum()) < keep.numel()
    W = lin._params["W"].data.clone().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    ref = TORCH_F[kind](xr @ W.T + lin._params["b"].data) * keep * s
    ref_dx, ref_dw = torch.autograd.grad((g * ref).sum(), (xr, W))
    lin.zero_grad()
    out = lin.forward(x)
    assert torch.allclose(out, ref.detach(), rtol=1e-13, atol=1e-13)
    dx = lin.backward(g)
    assert torch.allclose(dx, ref_dx, rtol=1e-12, atol=1e-13)
    assert torch.allclose(lin._params["W"].grad, ref_dw, rtol=1e-12, atol=1e-13)


def test_relu_default_is_unchanged():
    a = MLP(SIZES, 0, 1, 128)
    b = MLP(SIZES, 0, 1, 128, activation="relu")
    assert a.activation == b.activation == "relu"
    assert all(type(x.activation).__name__ == "ReLU" for x in a.linears[:-1]) and a.linears[-1].activation is None
    x = torch.randn(8, 784, generator=torch.Generator().manual_seed(0))
    assert torch.equal(a.forward(x), b.forward(x))


def test_pp8_stage_six_keeps_the_activation():
    m = MLP(SIZES, 6, 8, 128, activation="silu")
    assert [type(x.activation).__name__ for x in m.linears] == ["SiLU"]
    last = MLP(SIZES, 7, 8, 128, activation="silu")
    assert last.linears == [] or all(x.activation is None for x in last.linears)


# ------------------------------------------------------------------ sequential == DP == PP == DP x PP (dropout on)
def _run_layout(kind, dp, pp, cls, steps=4):
    import test_equivalence as E

    orig_mlp = E.MLP
    orig_worker_execute = E.Worker.execute

    def mlp(*a, **k):
        return orig_mlp(*a, activation=kind, dropout=P, dropout_seed=SEED, **k)

    def execute(self, sched, batch_id):
        self.model.dropout_step = batch_id
        return orig_worker_execute(self, sched, batch_id)

    E.MLP, E.Worker.execute = mlp, execute
    try:
        return E.run_layout(dp, pp, cls, steps=steps)
    finally:
        E.MLP, E.Worker.execute = orig_mlp, orig_worker_execute


_SEQ = {}


def _sequential(kind):
    if kind not in _SEQ:
        _SEQ[kind] = _run_layout(kind, 1, 1, NaiveParallelSchedule)
    return _SEQ[kind]


@pytest.mark.parametrize("kind", SMOOTH)
@pytest.mark.parametrize("dp,pp,cls", [
    (2, 1, NaiveParallelSchedule), (1, 2, GPipeSchedule), (1, 4, PipeDreamSchedule), (2, 2, GPipeSchedule),
])
def test_layout_matches_sequential(kind, dp, pp, cls):
    _close(_run_layout(kind, dp, pp, cls), _sequential(kind))


@pytest.mark.parametrize("kind", SMOOTH)
def test_activation_changes_training(kind):
    plain = run_layout(1, 1, NaiveParallelSchedule, steps=2)
    import test_equivalence as E

    orig = E.MLP
    E.MLP = lambda *a, **k: orig(*a, activation=kind, **k)
    try:
        other = E.run_layout(1, 1, NaiveParallelSchedule, steps=2)
    finally:
        E.MLP = orig
    assert any(not torch.equal(a, b) for a, b in zip(plain, other))


# ------------------------------------------------------------------ train.py
def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


CLI = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic"]


def test_train_cli_resume_is_bitwise_and_refuses_a_mismatch(tmp_path):
    act = ["--activation", "gelu", "--dropout", "0.2"]
    for args in (["--steps", "6", "--save", str(tmp_path / "full")], ["--steps", "3", "--save", str(tmp_path / "part")],
                 ["--steps", "6", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(CLI + act + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 6 and a["hparams"]["activation"] == "gelu"
    assert torch.equal(a["weights"], b["weights"])
    for other in (["--activation", "silu", "--dropout", "0.2"], ["--dropout", "0.2"]):
        r = _run(CLI + other + ["--steps", "6", "--resume", str(tmp_path / "part")])
        assert r.returncode != 0 and "checkpoint was written with activation" in (r.stderr + r.stdout)


def test_train_cli_checkpoint_without_the_key_resumes_as_relu(tmp_path):
    r = _run(CLI + ["--steps", "2", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    path = tmp_path / "part" / "stage0of1.pt"
    ck = torch.load(path)
    assert ck["hparams"]["activation"] == "relu"
    del ck["hparams"]["activation"]
    torch.save(ck, path)
    r = _run(CLI + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(CLI + ["--activation", "tanh", "--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with activation" in (r.stderr + r.stdout)


def test_train_cli_rejects_an_unknown_activation():
    r = _run(CLI + ["--activation", "elu", "--steps", "1"])
    assert r.returncode != 0 and "ValueError" in r.stderr and "unknown activation" in r.stderr
