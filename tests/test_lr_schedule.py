"""Learning-rate schedules on the CPU: every family against ``torch.optim.lr_scheduler`` step by step in fp64, the
Python VM under warmup + cosine against ``torch.optim.SGD`` + ``SequentialLR``, an ``lr == 0`` step, and ``train.py``
with a schedule (run, resume mid-schedule, refusals)."""
import math
import os
import subprocess
import sys

import pytest
import torch

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.layers import MLP
from shallowspeed_b200.lr_schedule import LRSchedule, to_fp32
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.pipe import NaiveParallelSchedule, Worker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
GBS, N_MU = 128, 4
BASE = 0.05
S = torch.optim.lr_scheduler


# ------------------------------------------------------------------ every family against torch
def _torch_rates(make, steps, base=BASE):
    """fp64 rates of ``steps`` optimizer steps under the torch scheduler ``make(opt)``."""
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=base)
    sched = make(opt)
    out = []
    for _ in range(steps):
        out.append(opt.param_groups[0]["lr"])
        opt.step()
        sched.step()
    return out


def _warm(opt, main, W, f):
    return S.SequentialLR(opt, [S.LinearLR(opt, start_factor=f, end_factor=1.0, total_iters=W), main], milestones=[W])


T, W, F = 40, 5, 0.25
CASES = {
    "constant": (dict(kind="constant"), lambda o: S.ConstantLR(o, factor=1.0, total_iters=0)),
    "step": (dict(kind="step", step_size=7, gamma=0.5), lambda o: S.StepLR(o, step_size=7, gamma=0.5)),
    "cosine": (dict(kind="cosine", total_steps=T, min_lr=1e-3), lambda o: S.CosineAnnealingLR(o, T_max=T, eta_min=1e-3)),
    "cosine-to-0": (dict(kind="cosine", total_steps=T), lambda o: S.CosineAnnealingLR(o, T_max=T, eta_min=0.0)),
    "linear": (dict(kind="linear", total_steps=T, min_lr=5e-3),
               lambda o: S.LinearLR(o, start_factor=1.0, end_factor=5e-3 / BASE, total_iters=T)),
    "warmup": (dict(kind="constant", warmup_steps=W, warmup_start_factor=F),
               lambda o: S.LinearLR(o, start_factor=F, end_factor=1.0, total_iters=W)),
    "warmup+step": (dict(kind="step", warmup_steps=W, warmup_start_factor=F, step_size=6, gamma=0.3),
                    lambda o: _warm(o, S.StepLR(o, step_size=6, gamma=0.3), W, F)),
    "warmup+cosine": (dict(kind="cosine", total_steps=T, warmup_steps=W, warmup_start_factor=F, min_lr=2e-3),
                      lambda o: _warm(o, S.CosineAnnealingLR(o, T_max=T - W, eta_min=2e-3), W, F)),
    "warmup+linear": (dict(kind="linear", total_steps=T, warmup_steps=W, warmup_start_factor=F),
                      lambda o: _warm(o, S.LinearLR(o, start_factor=1.0, end_factor=0.0, total_iters=T - W), W, F)),
}


@pytest.mark.filterwarnings("ignore::UserWarning")
@pytest.mark.parametrize("case", sorted(CASES))
def test_every_family_matches_torch_lr_scheduler(case):
    kw, make = CASES[case]
    sch = LRSchedule(BASE, **kw)
    # the whole horizon; torch's cosine is periodic past T_max, this one holds min_lr, so compare up to the horizon
    ref = _torch_rates(make, T + 1)
    for i, r in enumerate(ref):
        got = sch.exact(i)
        assert math.isclose(got, r, rel_tol=1e-12, abs_tol=1e-12 * BASE), (case, i, got, r)
        assert sch(i) == to_fp32(got)
    if "cosine" in case or "linear" in case:
        assert sch.exact(T + 7) == sch.min_lr                   # held past the horizon


def test_rate_is_rounded_to_fp32_once():
    sch = LRSchedule(0.1, "cosine", total_steps=9, warmup_steps=2)
    for i in range(12):
        v = sch(i)
        assert v == float(torch.tensor(sch.exact(i), dtype=torch.float64).to(torch.float32))
    assert LRSchedule(0.006)(12345) == float(torch.tensor(0.006, dtype=torch.float32))


@pytest.mark.parametrize("kw", [
    dict(base_lr=-0.1), dict(base_lr=float("nan")), dict(base_lr=float("inf")), dict(kind="exp"),
    dict(warmup_steps=-1), dict(warmup_steps=1.5), dict(warmup_steps=2, warmup_start_factor=0.0),
    dict(warmup_steps=2, warmup_start_factor=1.5), dict(kind="cosine"), dict(kind="cosine", total_steps=3, warmup_steps=3),
    dict(kind="linear", total_steps=10, min_lr=1.0), dict(kind="cosine", total_steps=10, min_lr=-1e-3),
    dict(kind="step"), dict(kind="step", step_size=0), dict(kind="step", step_size=3, gamma=0.0),
    dict(kind="step", step_size=3, gamma=2.0), dict(total_steps=-5),
])
def test_bad_arguments_raise_value_error(kw):
    kw = {"base_lr": BASE, **kw}
    with pytest.raises(ValueError):
        LRSchedule(**kw)


def test_bad_step_raises_and_spec_round_trips():
    sch = LRSchedule(BASE, "cosine", total_steps=20, warmup_steps=3, min_lr=1e-4)
    with pytest.raises(ValueError):
        sch(-1)
    again = LRSchedule(BASE, **sch.spec())
    assert [again(i) for i in range(25)] == [sch(i) for i in range(25)]
    assert LRSchedule(BASE).spec() == {"kind": "constant"}


def test_sgd_lr_setter_is_validated():
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), BASE, arena=model.arena)
    opt.lr = 0.0
    assert opt.lr == 0.0
    for bad in (-1.0, float("nan")):
        with pytest.raises(ValueError):
            opt.lr = bad
    assert opt.lr == 0.0


# ------------------------------------------------------------------ the Python VM against torch.optim.SGD + SequentialLR
_X, _Y = synthetic_mnist(n=GBS * 8)
MOM = dict(momentum=0.9, weight_decay=1e-3, nesterov=True)


class _TorchStep:
    """The VM's OptimizerStep done by torch.optim.SGD + a torch scheduler on parameters that share the arena's storage."""

    def __init__(self, model, make_sched):
        self.params = list(model.parameters())
        self.ref = [torch.nn.Parameter(p.data) for p in self.params]        # same storage: torch updates the arena
        self.opt = torch.optim.SGD(self.ref, lr=BASE, **MOM)
        self.sched = make_sched(self.opt)

    def step(self):
        for p, r in zip(self.params, self.ref):
            r.grad = p.grad
        self.opt.step()
        self.sched.step()


def _vm(optimizer_for, steps, schedule=None):
    model = MLP(SIZES, 0, 1, GBS)
    opt = optimizer_for(model)
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(_X, _Y)
    worker = Worker(None, None, model, ds, opt)
    for b in range(steps):
        if schedule is not None:
            opt.lr = schedule(b)
        worker.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    return [p.data.clone() for p in model.parameters()], model


@pytest.mark.filterwarnings("ignore::UserWarning")
def test_vm_follows_warmup_cosine_like_torch():
    steps, warm = 8, 3
    sch = LRSchedule(BASE, "cosine", total_steps=steps, warmup_steps=warm, warmup_start_factor=0.2, min_lr=1e-3)
    ours, _ = _vm(lambda m: SGD(m.parameters(), BASE, arena=m.arena, **MOM), steps, sch)
    theirs, _ = _vm(lambda m: _TorchStep(m, lambda o: _warm(o, S.CosineAnnealingLR(o, T_max=steps - warm, eta_min=1e-3),
                                                             warm, 0.2)), steps)
    for a, b in zip(ours, theirs):
        assert float((a - b).abs().max()) < 1e-6
    const, _ = _vm(lambda m: SGD(m.parameters(), BASE, arena=m.arena, **MOM), steps)
    assert max(float((a - b).abs().max()) for a, b in zip(ours, const)) > 1e-4    # the schedule changed the trajectory


def test_lr_zero_step_keeps_weights_and_advances_momentum():
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), BASE, arena=model.arena, **MOM)
    gen = torch.Generator().manual_seed(3)
    model.arena.grads.copy_(torch.randn(model.arena.grads.shape, generator=gen))
    opt.step()
    w, v = model.arena.weights.clone(), model.arena.momentum.clone()
    g = torch.randn(model.arena.grads.shape, generator=gen)
    model.arena.grads.copy_(g)
    opt.lr = 0.0
    opt.step()
    assert torch.equal(model.arena.weights, w)
    n = model.arena.numel
    want = v[:n] * MOM["momentum"] + (g[:n] + w[:n] * MOM["weight_decay"])
    assert torch.allclose(model.arena.momentum[:n], want, rtol=1e-6, atol=1e-7)
    assert not torch.equal(model.arena.momentum, v)


# ------------------------------------------------------------------ train.py
def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


BASE_CLI = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic", "--momentum", "0.9"]
COSINE = ["--lr-schedule", "cosine", "--warmup-steps", "2", "--lr-total-steps", "6"]


def test_train_cli_schedule_resume_is_bitwise(tmp_path):
    r = _run(BASE_CLI + ["--steps", "6", "--lr-schedule", "cosine", "--warmup-steps", "2", "--save", str(tmp_path / "a")])
    assert r.returncode == 0, r.stderr[-2000:]
    for args in (["--steps", "6", "--save", str(tmp_path / "full")], ["--steps", "3", "--save", str(tmp_path / "part")],
                 ["--steps", "6", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(BASE_CLI + COSINE + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    c = torch.load(tmp_path / "a" / "stage0of1.pt")
    assert a["step"] == b["step"] == 6 and a["hparams"] == b["hparams"] == c["hparams"]
    assert a["hparams"]["lr_schedule"] == {"kind": "cosine", "warmup_steps": 2, "warmup_start_factor": 1 / 3,
                                           "total_steps": 6, "min_lr": 0.0}
    assert torch.equal(a["weights"], b["weights"]) and torch.equal(a["momentum"], b["momentum"])
    assert torch.equal(a["weights"], c["weights"])           # the horizon defaults to the run's total steps
    # another schedule is refused, as another base rate is
    for other in (["--lr-schedule", "linear", "--warmup-steps", "2", "--lr-total-steps", "6"],
                  ["--lr-schedule", "cosine", "--warmup-steps", "1", "--lr-total-steps", "6"], []):
        r = _run(BASE_CLI + other + ["--steps", "6", "--resume", str(tmp_path / "part")])
        assert r.returncode != 0 and "checkpoint was written with lr_schedule" in (r.stderr + r.stdout)


def test_train_cli_checkpoint_without_schedule_resumes_as_constant(tmp_path):
    r = _run(BASE_CLI + ["--steps", "2", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    path = tmp_path / "part" / "stage0of1.pt"
    ck = torch.load(path)
    del ck["hparams"]["lr_schedule"]                       # as written before schedules existed
    torch.save(ck, path)
    r = _run(BASE_CLI + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(BASE_CLI + COSINE + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with lr_schedule" in (r.stderr + r.stdout)


def test_train_cli_rejects_a_bad_schedule():
    r = _run(BASE_CLI + ["--steps", "2", "--lr-schedule", "step"])
    assert r.returncode != 0 and "step_size" in r.stderr
