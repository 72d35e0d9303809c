"""Exponential moving average of the weights on the CPU: validation, the alpha sequence, the reference lerp against
fp64 and torch's AveragedModel, the optimizer's update on every path, the Python VM's layouts, checkpoints and the CLI."""
import os
import subprocess
import sys
import threading

import pytest
import torch

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.layers import MLP
from shallowspeed_b200.ops.functional import check_ema_decay, ema_alpha, ema_lerp_ref
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.parallel.comm import ProcessGrid, ThreadFabric
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule, Worker
from shallowspeed_b200.utils import assert_sync, get_model_hash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
GBS, N_MU, LR = 128, 4, 0.05
_X, _Y = synthetic_mnist(n=GBS * 6)
MOM = dict(momentum=0.9, weight_decay=1e-3, nesterov=True)


@pytest.mark.parametrize("bad", [0.0, 1.0, -0.5, 1.5, float("nan"), True, "0.9", [0.9]])
def test_bad_ema_decay_raises(bad):
    with pytest.raises(ValueError):
        check_ema_decay(bad)
    model = MLP(SIZES, 0, 1, GBS)
    with pytest.raises(ValueError):
        SGD(model.parameters(), LR, arena=model.arena, ema_decay=bad)


def test_no_ema_by_default_costs_nothing():
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena)
    assert opt.ema_decay is None and opt.ema_alpha is None and model.arena.ema is None


def test_alpha_sequence():
    assert ema_alpha(0.999, 0) == 1.0
    for n in (1, 2, 1000):
        a = ema_alpha(0.999, n)
        assert a == float(torch.tensor(1 - 0.999, dtype=torch.float64).float())
    assert ema_alpha(0.3, 5) == float(torch.tensor(0.7, dtype=torch.float64).float()) and ema_alpha(0.3, 5) >= 0.5
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena, ema_decay=0.99)
    assert opt.ema_updates == 0 and opt.ema_alpha == 1.0
    opt.step()
    assert opt.ema_updates == 1 and opt.ema_alpha == ema_alpha(0.99, 1)
    opt.ema_updates = 0
    assert opt.ema_alpha == 1.0
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError):
            opt.ema_updates = bad


@pytest.mark.parametrize("alpha", [1.0, float(1 - torch.tensor(0.999).item()), 0.001, 0.3, 0.5, 0.7])
def test_lerp_ref_against_fp64(alpha):
    gen = torch.Generator().manual_seed(3)
    e = torch.randn(4096, generator=gen)
    w = e + 0.01 * torch.randn(4096, generator=gen)
    got = ema_lerp_ref(e, w, alpha)
    a = torch.tensor(alpha, dtype=torch.float32).double()
    exact = e.double() + a * (w.double() - e.double())
    # three roundings, each within u = 2^-24 relative of its own result: w - e, the product with alpha (or 1 - alpha,
    # exact for alpha >= 0.5) and the final sum, so |err| <= u * (|result| + 2 * min(alpha, 1 - alpha) * |w - e|) (+ u^2)
    d = (w.double() - e.double()).abs()
    u = 2.0 ** -24
    bound = u * (exact.abs() + 2 * min(float(a), 1 - float(a)) * d) * (1 + 4 * u)
    assert bool(((got.double() - exact).abs() <= bound).all())
    if alpha == 1.0:
        assert torch.equal(got, w)


def test_lerp_ref_matches_torch_averaged_model():
    """torch's AveragedModel with get_ema_multi_avg_fn, driven through the same weight sequence.  torch's
    _foreach_lerp_ may contract the formula, and the difference of one update carries into the next, so the two agree
    to within 8 ulp of the tensor's largest magnitude (near-zero elements can differ by many of their own ulp)."""
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

    decay = 0.9
    gen = torch.Generator().manual_seed(4)
    net = torch.nn.Linear(64, 32)
    avg = AveragedModel(net, multi_avg_fn=get_ema_multi_avg_fn(decay))
    mine = [p.detach().clone() for p in net.parameters()]
    for n in range(6):
        with torch.no_grad():
            for p in net.parameters():
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
        avg.update_parameters(net)
        for e, p in zip(mine, net.parameters()):
            e.copy_(ema_lerp_ref(e, p.detach(), ema_alpha(decay, n)))
    for e, p in zip(mine, avg.module.parameters()):
        scale = float(p.detach().abs().max())
        assert float((e - p.detach()).abs().max()) <= 8 * 2.0 ** -24 * scale


@pytest.mark.parametrize("opt_kw", [{}, MOM])
def test_ema_equals_weights_at_construction_and_after_the_first_update(opt_kw):
    model = MLP(SIZES, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena, ema_decay=0.999, **opt_kw)
    arena = model.arena
    for i, (_, k) in enumerate(arena.blocks):
        assert torch.equal(arena.ema_block(i)[:, : k + 1], arena.block(i)[:, : k + 1])
        assert not bool(arena.ema_block(i)[:, k + 1:].any())          # padding is zero
    arena.grads.copy_(torch.randn(arena.grads.shape, generator=torch.Generator().manual_seed(5)))
    opt.step()
    assert torch.equal(arena.ema, arena.weights[: arena.numel])
    opt.step()
    assert not torch.equal(arena.ema, arena.weights[: arena.numel])


@pytest.mark.parametrize("arena_path", [True, False], ids=["arena", "per_parameter"])
@pytest.mark.parametrize("opt_kw", [{}, MOM], ids=["plain", "momentum"])
def test_ema_changes_no_weight_and_follows_the_reference(opt_kw, arena_path):
    """The weights of an EMA run are those of the same run without it, and the EMA is the reference lerp replayed over
    the run's own weight sequence, bit for bit."""
    runs = {}
    for decay in (None, 0.8):
        model = MLP(SIZES, 0, 1, GBS)
        opt = SGD(model.parameters(), LR, arena=model.arena if arena_path else None, ema_decay=decay, **opt_kw)
        params = list(model.parameters())
        ema = [p.data.clone() for p in params]                       # the reference, replayed
        gen = torch.Generator().manual_seed(6)
        ws = []
        for t in range(4):
            for p in params:
                p.grad.copy_(torch.randn(p.grad.shape, generator=gen))
            opt.step()
            ws.append([p.data.clone() for p in params])
            ema = [ema_lerp_ref(e, p.data, ema_alpha(0.8, t)) for e, p in zip(ema, params)]
        if decay is not None:
            assert opt.ema_updates == 4
            if arena_path:
                got = [model.arena.ema.as_strided(p.data.shape, p.data.stride(), p.data.storage_offset()) for p in params]
            else:
                got = opt.ema_buffers
            assert all(torch.equal(a, b) for a, b in zip(got, ema))
        runs[decay] = ws
    for a, b in zip(runs[None], runs[0.8]):
        assert all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------ Python VM: layouts
def run_ema_layout(dp, pp, sched_cls, steps=4, opt_kw=None, decay=0.9):
    """The EMA arenas of every stage (taken from replica 0) after ``steps`` VM steps; replicas must agree bitwise."""
    opt_kw = opt_kw or {}
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
            opt = SGD(model.parameters(), LR, arena=model.arena, ema_decay=decay, **opt_kw)
            ds = Dataset(None, GBS, GBS // dp // N_MU)
            ds.local_batch_size = GBS // dp
            ds.from_arrays(_X[grid.replica::dp], _Y[grid.replica::dp])
            worker = Worker(dp_comm, pp_comm, model, ds, opt)
            sched = sched_cls(N_MU, pp, grid.stage)
            for b in range(steps):
                worker.execute(sched, b)
            assert_sync(dp_comm, get_model_hash(model))
            results[rank] = (model, opt.ema_updates)
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
        assert results[rank][1] == steps
        assert torch.equal(results[rank][0].arena.ema, results[g.stage][0].arena.ema), "DP replicas' EMA diverged"
    # per Linear: (weights block, EMA block) of every stage in model order
    out = []
    for s in range(pp):
        m = results[s][0]
        for i in range(len(m.arena.blocks)):
            k = m.arena.blocks[i][1]
            out.append((m.arena.block(i)[:, : k + 1].clone(), m.arena.ema_block(i)[:, : k + 1].clone()))
    return out


@pytest.fixture(scope="module", params=[{}, MOM], ids=["plain", "momentum"])
def ema_sequential(request):
    return request.param, run_ema_layout(1, 1, NaiveParallelSchedule, opt_kw=request.param)


@pytest.mark.parametrize("dp,pp,cls", [(2, 1, NaiveParallelSchedule), (1, 2, GPipeSchedule), (1, 2, PipeDreamSchedule),
                                       (2, 2, GPipeSchedule)])
def test_vm_layouts_ema_match_sequential(ema_sequential, dp, pp, cls):
    opt_kw, seq = ema_sequential
    got = run_ema_layout(dp, pp, cls, opt_kw=opt_kw)
    assert len(got) == len(seq)
    for (w, e), (w0, e0) in zip(got, seq):
        assert float((w - w0).abs().max()) < 2e-6          # the tolerance the weights already meet across layouts
        assert float((e - e0).abs().max()) < 2e-6
    # non-vacuous: after 4 steps at decay 0.9 the EMA is not the weights
    assert max(float((w - e).abs().max()) for w, e in seq) > 1e-5


# ------------------------------------------------------------------ checkpoints and the CLI
def test_checkpoint_refuses_another_decay(tmp_path):
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    model = MLP(SIZES, 0, 1, GBS)
    SGD(model.parameters(), LR, arena=model.arena, ema_decay=0.9)
    save_stage(model, tmp_path, 0, 1, step=3, hparams=dict(lr=LR, ema_decay=0.9), ema=model.arena.ema)
    fresh = MLP(SIZES, 0, 1, GBS)
    SGD(fresh.parameters(), LR, arena=fresh.arena, ema_decay=0.9)
    fresh.arena.ema.zero_()
    assert load_stage(fresh, tmp_path, 0, 1, expect_hparams=dict(lr=LR, ema_decay=0.9)) == 3
    assert torch.equal(fresh.arena.ema, model.arena.ema)
    for other in (0.99, None):
        with pytest.raises(ValueError, match="ema_decay"):
            load_stage(MLP(SIZES, 0, 1, GBS), tmp_path, 0, 1, expect_hparams=dict(lr=LR, ema_decay=other))
    # a checkpoint without the key counts as written without an EMA
    save_stage(model, tmp_path / "old", 0, 1, step=1, hparams=dict(lr=LR))
    load_stage(MLP(SIZES, 0, 1, GBS), tmp_path / "old", 0, 1, expect_hparams=dict(lr=LR, ema_decay=None))
    with pytest.raises(ValueError, match="ema_decay"):
        load_stage(MLP(SIZES, 0, 1, GBS), tmp_path / "old", 0, 1, expect_hparams=dict(lr=LR, ema_decay=0.9))


def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_train_cli_prints_ema_accuracy_and_resumes_bitwise(tmp_path):
    base = ["train.py", "--device", "cpu", "--engine", "python", "--synthetic", "--ema-decay", "0.99"]
    r = _run(base + ["--steps", "3", "--log-json", str(tmp_path / "log.jsonl")])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.splitlines()
    acc = [i for i, s in enumerate(lines) if "Accuracy:" in s]
    assert acc and all(lines[i + 1].startswith("EMA accuracy: ") and lines[i + 1].endswith("%") for i in acc)
    import json

    evals = [json.loads(s) for s in open(tmp_path / "log.jsonl") if '"eval"' in s]
    assert evals and all("ema_accuracy" in e for e in evals)
    for args in (["--steps", "4", "--save", str(tmp_path / "full")], ["--steps", "2", "--save", str(tmp_path / "part")],
                 ["--steps", "4", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(base + ["--no-eval"] + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["hparams"]["ema_decay"] == 0.99 and a["step"] == b["step"] == 4
    assert torch.equal(a["weights"], b["weights"]) and torch.equal(a["ema"], b["ema"])
    assert not torch.equal(a["ema"], a["weights"])
    r = _run(base[:-1] + ["0.9", "--no-eval", "--steps", "4", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "ema_decay" in (r.stderr + r.stdout)


@pytest.mark.parametrize("bad", ["0", "1", "-0.1", "1.5"])
def test_train_cli_rejects_bad_decay(bad):
    r = _run(["train.py", "--device", "cpu", "--steps", "1", "--no-eval", "--synthetic", "--ema-decay", bad])
    assert r.returncode != 0 and "ema_decay" in r.stderr
