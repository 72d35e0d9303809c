"""Dropout on the hidden layers: the Philox4x32-10 generator against its known answers and a scalar implementation, the
mask contract (drop rate, scale, independence from the DP layout), the dropped Linear's backward, the model partition,
sequential == DP == PP == DP x PP in the Python VM, and train.py (run, resume, refusals)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from shallowspeed_b200.layers import MLP
from shallowspeed_b200.ops import functional as F
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule

from test_equivalence import SIZES, _close, run_layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, SEED = 0.3, 0x1234_5678_9ABC_DEF0


# ------------------------------------------------------------------ the generator
KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


def philox_scalar(c, k):
    """Philox4x32-10 on Python ints, written from the round definition."""
    c, (k0, k1) = list(c), k
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k1, p0 & 0xFFFFFFFF]
    return tuple(c)


@pytest.mark.parametrize("case", range(len(KAT)))
def test_philox_known_answers(case):
    ctr, key, want = KAT[case]
    assert philox_scalar(ctr, key) == want
    assert tuple(int(w) for w in F.philox4x32_10(ctr, key)) == want


def test_torch_philox_matches_scalar_on_random_counters():
    rng = random.Random(7)
    ctrs = [[rng.getrandbits(32) for _ in range(4)] for _ in range(300)]
    keys = [[rng.getrandbits(32) for _ in range(2)] for _ in range(300)]
    t = lambda i, src: torch.tensor([x[i] for x in src], dtype=torch.int64)
    got = F.philox4x32_10(tuple(t(i, ctrs) for i in range(4)), tuple(t(i, keys) for i in range(2)))
    for j in range(300):
        assert tuple(int(w[j]) for w in got) == philox_scalar(ctrs[j], keys[j])


# ------------------------------------------------------------------ the mask contract
@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_drop_fraction_and_scale(p):
    keep = F.dropout_mask(p, 99, layer=2, step=5, samples=torch.arange(1000), n_features=1000)
    n = keep.numel()
    dropped = n - int(keep.sum())
    sigma = (n * p * (1 - p)) ** 0.5
    assert abs(dropped - n * p) < 5 * sigma
    assert F.dropout_threshold(p) == int(np.floor(p * 2.0 ** 32))
    assert F.dropout_scale(p) == float(np.float32(1.0 / (1.0 - p)))
    x = torch.rand(4, 8) + 0.5
    k = F.dropout_mask(p, 99, 0, 0, torch.arange(4), 8)
    assert torch.equal(F.dropout_ref(x, k, F.dropout_scale(p)), torch.where(k, x * np.float32(F.dropout_scale(p)), 0.0))


def test_threshold_decides_on_word_zero():
    samples, feats = torch.arange(16), 24
    u = F.philox4x32_10((torch.arange(feats).view(1, -1), samples.view(-1, 1), 3, 11), (SEED & 0xFFFFFFFF, SEED >> 32))[0]
    assert torch.equal(F.dropout_mask(P, SEED, 3, 11, samples, feats), u >= F.dropout_threshold(P))
    # the step counter wraps at 2^32
    assert torch.equal(F.dropout_mask(P, SEED, 3, 11 + 2 ** 32, samples, feats), u >= F.dropout_threshold(P))


@pytest.mark.parametrize("dp", [2, 4, 8])
def test_mask_of_a_sample_does_not_depend_on_the_dp_layout(dp):
    batch, feats = 64, 40
    full = F.dropout_mask(P, SEED, 1, 4, torch.arange(batch), feats)
    for r in range(dp):
        n = torch.arange(batch // dp)
        shard = F.dropout_mask(P, SEED, 1, 4, n * dp + r, feats)
        assert torch.equal(shard, full[r::dp])


def test_masks_change_with_the_step_and_the_layer():
    a = F.dropout_mask(P, SEED, 1, 0, torch.arange(32), 64)
    assert not torch.equal(a, F.dropout_mask(P, SEED, 1, 1, torch.arange(32), 64))
    assert not torch.equal(a, F.dropout_mask(P, SEED, 2, 0, torch.arange(32), 64))
    assert not torch.equal(a, F.dropout_mask(P, SEED + 1, 1, 0, torch.arange(32), 64))


@pytest.mark.parametrize("kw", [dict(dropout=-0.1), dict(dropout=1.0), dict(dropout=float("nan")), dict(dropout="0.2"),
                                dict(dropout_seed=-1), dict(dropout_seed=2 ** 64), dict(dropout_seed=1.5)])
def test_bad_arguments_raise_value_error(kw):
    with pytest.raises(ValueError):
        MLP(SIZES, 0, 1, 128, **kw)


def test_dropout_step_is_validated():
    m = MLP(SIZES, 0, 1, 128, dropout=0.2)
    m.dropout_step = 7
    assert m.dropout_step == 7
    for bad in (-1, 1.0, True, "3"):
        with pytest.raises(ValueError):
            m.dropout_step = bad


# ------------------------------------------------------------------ the model
@pytest.mark.parametrize("pp", [1, 2, 4, 8])
def test_partition_drops_every_relu_linear_and_never_the_logits(pp):
    for stage in range(pp):
        m = MLP(SIZES, stage, pp, 128, dropout=0.25, dropout_seed=3)
        for lin in m.linears:
            if lin.activation is not None:
                assert lin.dropout[:2] == (0.25, 3) and lin.activation.dropout_scale == F.dropout_scale(0.25)
            else:
                assert lin.dropout is None
        if stage == pp - 1 and m.linears:   # pp = 8: the last stage holds only the loss head
            assert m.linears[-1].activation is None and m.linears[-1].dropout is None
    # pp = 8: stage 6 ends in the 123 -> 10 Linear, which carries a ReLU there and is dropped
    m6 = MLP(SIZES, 6, 8, 128, dropout=0.25)
    assert m6.linears[-1].out_dims == 10 and m6.linears[-1].dropout is not None and m6.linears[-1].dropout[2] == 6


def test_forward_matches_the_oracle_and_eval_does_not_drop():
    torch.manual_seed(0)
    m = MLP(SIZES, 0, 2, 128, dropout=P, dropout_seed=SEED)   # 784 -> 128 -> 127 -> 126 -> 125, all ReLU
    m.dropout_step = 9
    m.dropout_shard = (1, 2)
    x = torch.rand(16, 784)
    out = m.forward(x, mubatch_id=3)
    a = x
    s = F.dropout_scale(P)
    samples = (3 * 16 + torch.arange(16)) * 2 + 1
    for lin in m.linears:
        a = F.relu_ref(F.linear_ref(a, lin._params["W"].data, lin._params["b"].data))
        a = F.dropout_ref(a, F.dropout_mask(P, SEED, lin.dropout[2], 9, samples, a.shape[1]), s)
    assert torch.equal(out, a)
    m.backward(torch.zeros_like(out), mubatch_id=3)
    m.eval()
    plain = x
    for lin in m.linears:
        plain = F.relu_ref(F.linear_ref(plain, lin._params["W"].data, lin._params["b"].data))
    assert torch.equal(m.forward(x, mubatch_id=3), plain)


def test_dropped_linear_backward_matches_finite_differences():
    """fp64: d/dx and d/dW of sum(g * dropout(relu(x W^T + b))) for a fixed mask, against central differences."""
    from shallowspeed_b200.models.layers import Linear

    lin = Linear(6, 5)
    lin.arena.weights = lin.arena.weights.double()
    lin.arena.grads = lin.arena.grads.double()
    lin._bind()
    s = F.dropout_scale(0.4)
    lin.dropout = (0.4, 5, 0, s)
    lin.activation.dropout_scale = s
    lin.dropout_rows = (torch.arange(3), 2)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(3, 6, dtype=torch.float64, generator=gen)
    g = torch.randn(3, 5, dtype=torch.float64, generator=gen)
    keep = F.dropout_mask(0.4, 5, 0, 2, torch.arange(3), 5)
    assert 0 < int(keep.sum()) < keep.numel()

    def f(xv, wv):
        return float((g * F.dropout_ref(F.relu_ref(F.linear_ref(xv, wv, lin._params["b"].data)), keep, s)).sum())

    lin.zero_grad()
    lin.forward(x)
    dx = lin.backward(g)
    W = lin._params["W"].data.clone()
    eps = 1e-6
    for i in range(3):
        for j in range(6):
            e = torch.zeros_like(x)
            e[i, j] = eps
            assert abs((f(x + e, W) - f(x - e, W)) / (2 * eps) - float(dx[i, j])) < 1e-6
    for i in range(5):
        for j in range(6):
            e = torch.zeros_like(W)
            e[i, j] = eps
            assert abs((f(x, W + e) - f(x, W - e)) / (2 * eps) - float(lin._params["W"].grad[i, j])) < 1e-6


def _train_vm(dropout, steps=3, **kw):
    from test_equivalence import _make_dataset, GBS, LR, N_MU
    from shallowspeed_b200.pipe import Worker

    model = MLP(SIZES, 0, 1, GBS, **kw) if dropout is None else MLP(SIZES, 0, 1, GBS, dropout=dropout, **kw)
    opt = SGD(model.parameters(), LR, arena=model.arena)
    worker = Worker(None, None, model, _make_dataset(0, 1, GBS // N_MU), opt)
    for b in range(steps):
        if dropout is not None:
            model.dropout_step = b
        worker.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    return model.arena.weights.clone()


def test_p_zero_is_bit_identical_to_no_dropout():
    assert torch.equal(_train_vm(None), _train_vm(0.0, dropout_seed=5))


def test_dropout_changes_training_and_masks_follow_the_step():
    base = _train_vm(0.0)
    drop = _train_vm(0.3, dropout_seed=1)
    assert not torch.equal(base, drop)
    assert torch.equal(drop, _train_vm(0.3, dropout_seed=1))


# ------------------------------------------------------------------ sequential == DP == PP == DP x PP
def _run_dropout_layout(dp, pp, cls, steps=4):
    import test_equivalence as E

    orig_mlp = E.MLP
    orig_worker_execute = E.Worker.execute

    def mlp(*a, **k):
        return orig_mlp(*a, dropout=P, dropout_seed=SEED, **k)

    def execute(self, sched, batch_id):
        self.model.dropout_step = batch_id                 # one batch per step, from step 0
        return orig_worker_execute(self, sched, batch_id)

    E.MLP, E.Worker.execute = mlp, execute
    try:
        return E.run_layout(dp, pp, cls, steps=steps)
    finally:
        E.MLP, E.Worker.execute = orig_mlp, orig_worker_execute


@pytest.fixture(scope="module")
def sequential_dropout():
    return _run_dropout_layout(1, 1, NaiveParallelSchedule)


@pytest.mark.parametrize("dp,pp,cls", [
    (2, 1, NaiveParallelSchedule), (4, 1, GPipeSchedule),
    (1, 2, NaiveParallelSchedule), (1, 2, GPipeSchedule), (1, 2, PipeDreamSchedule),
    (1, 4, GPipeSchedule), (1, 4, PipeDreamSchedule),
    (2, 2, NaiveParallelSchedule), (2, 2, GPipeSchedule), (2, 2, PipeDreamSchedule),
])
def test_layout_matches_sequential_with_dropout(sequential_dropout, dp, pp, cls):
    _close(_run_dropout_layout(dp, pp, cls), sequential_dropout)


def test_dropout_layout_differs_from_plain(sequential_dropout):
    plain = run_layout(1, 1, NaiveParallelSchedule, steps=4)
    assert any(not torch.equal(a, b) for a, b in zip(plain, sequential_dropout))


# ------------------------------------------------------------------ train.py
def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


CLI = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic"]


def test_train_cli_smoke():
    r = _run(CLI + ["--dropout", "0.2", "--steps", "3"])
    assert r.returncode == 0, r.stderr[-2000:]


def test_train_cli_resume_is_bitwise_and_refuses_a_mismatch(tmp_path):
    drop = ["--dropout", "0.2", "--dropout-seed", "77"]
    for args in (["--steps", "6", "--save", str(tmp_path / "full")], ["--steps", "3", "--save", str(tmp_path / "part")],
                 ["--steps", "6", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(CLI + drop + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 6 and a["hparams"]["dropout"] == 0.2 and a["hparams"]["dropout_seed"] == 77
    assert torch.equal(a["weights"], b["weights"])
    for other in (["--dropout", "0.3", "--dropout-seed", "77"], ["--dropout", "0.2", "--dropout-seed", "78"], []):
        r = _run(CLI + other + ["--steps", "6", "--resume", str(tmp_path / "part")])
        assert r.returncode != 0 and "checkpoint was written with dropout" in (r.stderr + r.stdout)


def test_train_cli_checkpoint_without_dropout_resumes_as_p_zero(tmp_path):
    r = _run(CLI + ["--steps", "2", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    path = tmp_path / "part" / "stage0of1.pt"
    ck = torch.load(path)
    del ck["hparams"]["dropout"], ck["hparams"]["dropout_seed"]
    torch.save(ck, path)
    r = _run(CLI + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(CLI + ["--dropout", "0.1", "--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with dropout" in (r.stderr + r.stdout)


def test_train_cli_rejects_a_bad_rate():
    r = _run(CLI + ["--dropout", "1.0", "--steps", "1"])
    assert r.returncode != 0 and "dropout" in r.stderr
