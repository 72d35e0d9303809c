"""Shuffling the training set: the keyed Feistel permutation against a scalar implementation and pinned known answers, its
bijectivity, the rank-strided batch layout of a shuffled Dataset, sequential == DP == PP == DP x PP in the Python VM with
shuffling on, and train.py --shuffle (run, mid-epoch resume, refusals)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from shallowspeed_b200.dataset import Dataset, synthetic_mnist
from shallowspeed_b200.ops import functional as F
from shallowspeed_b200.pipe import GPipeSchedule, NaiveParallelSchedule, PipeDreamSchedule

from test_dropout import philox_scalar
from test_equivalence import GBS, _close, run_layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x1234_5678_9ABC_DEF0
NS = [1, 2, 3, 5, 127, 128, 129, 59500, 65536, 65537]
SEEDS = [0, 0x9E37_79B9_7F4A_7C15, 2 ** 64 - 1]       # the last two are >= 2^63
EPOCHS = [0, 1, 2 ** 32 - 1]


def shuffle_scalar(n, seed, epoch, q):
    """The permutation on Python ints, written from its definition."""
    w = 2
    while 2 ** w < n:
        w += 2
    h = w // 2
    mask = (1 << h) - 1
    x = q
    while True:
        L, R = x >> h, x & mask
        for i in range(6):
            f = philox_scalar((R, i, epoch & 0xFFFFFFFF, 0x53485546), (seed & 0xFFFFFFFF, seed >> 32))[0] & mask
            L, R = R, L ^ f
        x = (L << h) | R
        if x < n:
            return x


# ------------------------------------------------------------------ the permutation
def test_oracle_matches_the_scalar_definition():
    rng = random.Random(3)
    for n in NS:
        for seed in SEEDS + [rng.getrandbits(64)]:
            for epoch in EPOCHS + [rng.getrandbits(32)]:
                q = sorted({rng.randrange(n) for _ in range(12)})
                got = F.shuffle_index(n, seed, epoch, torch.tensor(q)).tolist()
                assert got == [shuffle_scalar(n, seed, epoch, v) for v in q], (n, seed, epoch)


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("seed", SEEDS)
def test_permutation_is_a_bijection(n, seed):
    for epoch in EPOCHS:
        p = F.shuffle_index(n, seed, epoch, torch.arange(n))
        assert p.dtype == torch.int64 and torch.equal(p.sort().values, torch.arange(n)), (n, seed, epoch)


def test_epochs_and_seeds_give_different_orders():
    q = torch.arange(59500)
    a = F.shuffle_index(59500, SEED, 0, q)
    assert not torch.equal(a, q)
    assert not torch.equal(a, F.shuffle_index(59500, SEED, 1, q))
    assert not torch.equal(a, F.shuffle_index(59500, SEED + 1, 0, q))
    assert not torch.equal(a, F.shuffle_index(59500, SEED ^ (1 << 63), 0, q))   # the seed's high word counts
    # the epoch is used mod 2^32
    assert torch.equal(F.shuffle_index(59500, SEED, 2 ** 32 + 1, q[:64]), F.shuffle_index(59500, SEED, 1, q[:64]))


# pinned outputs: a change of the definition (rounds, counter words, width rule, cycle walking) changes these
KAT = [(59500, SEED, 3, [9343, 19452, 32694, 27102, 5058, 31781, 11684, 45055, 47455, 58012, 48076, 42957, 19894, 27050,
                         51150, 24795]),
       (65537, 2 ** 64 - 1, 2 ** 32 - 1, [47270, 50258, 61500, 36177, 53723, 18812, 13078, 3532])]


@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case):
    n, seed, epoch, want = KAT[case]
    assert F.shuffle_index(n, seed, epoch, torch.arange(len(want))).tolist() == want
    assert [shuffle_scalar(n, seed, epoch, q) for q in range(len(want))] == want


@pytest.mark.parametrize("bad", [-1, 2 ** 64, 1.0, "3", True])
def test_bad_seeds_raise_value_error(bad):
    with pytest.raises(ValueError):
        Dataset(None, GBS, 32, shuffle_seed=bad)


def test_bad_positions_and_sizes_raise_value_error():
    for n, q in ((0, [0]), (2 ** 32, [0]), (10, [10]), (10, [-1])):
        with pytest.raises(ValueError):
            F.shuffle_index(n, 1, 0, torch.tensor(q))


def test_validation_set_is_never_shuffled():
    with pytest.raises(ValueError):
        Dataset(None, GBS, GBS, validation=True, shuffle_seed=1)
    ds = Dataset(None, GBS, GBS)
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError):
            ds.set_epoch(bad)


# ------------------------------------------------------------------ the Dataset
N_ROWS = 1000                      # 7 global batches of 128, 104 rows dropped per epoch
_X, _Y = synthetic_mnist(n=N_ROWS)


def _shuffled(rank, dp, seed=SEED, n_mu=4):
    ds = Dataset(None, GBS, GBS // dp // n_mu, shuffle_seed=seed)
    return ds.from_arrays(_X, _Y, DP_rank=rank, DP_size=dp)


@pytest.mark.parametrize("dp", [1, 2, 4])
def test_an_epoch_covers_distinct_samples_and_ranks_take_strided_parts(dp):
    full = _shuffled(0, 1)
    ranks = [_shuffled(r, dp) for r in range(dp)]
    for epoch in (0, 5):
        for ds in [full] + ranks:
            ds.set_epoch(epoch)
        assert full.get_num_batches() == N_ROWS // GBS == ranks[0].get_num_batches()
        seen = []
        for b in range(full.get_num_batches()):
            glob = full.sample_ids(b)
            assert torch.equal(glob, F.shuffle_index(N_ROWS, SEED, epoch, torch.arange(b * GBS, (b + 1) * GBS)))
            for r, ds in enumerate(ranks):
                ids = ds.sample_ids(b)
                assert torch.equal(ids, glob[r::dp])
                x, y = ds.load_batch(b)
                assert torch.equal(x, torch.from_numpy(_X)[ids]) and torch.equal(y, torch.from_numpy(_Y)[ids])
                for mu in range(ds.get_num_mubatches()):
                    rows = slice(mu * ds.mubatch_size, (mu + 1) * ds.mubatch_size)
                    assert torch.equal(ds.load_micro_batch_input(b, mu), x[rows])
                    assert torch.equal(ds.load_micro_batch_target(b, mu), y[rows])
                seen.append(ids)
        seen = torch.cat(seen)
        assert seen.numel() == N_ROWS // GBS * GBS == seen.unique().numel()


def test_epochs_drop_different_samples():
    ds = _shuffled(0, 1)
    kept = []
    for epoch in (0, 1):
        ds.set_epoch(epoch)
        kept.append(set(torch.cat([ds.sample_ids(b) for b in range(ds.get_num_batches())]).tolist()))
    assert kept[0] != kept[1]


def test_unshuffled_dataset_is_unchanged():
    """shuffle_seed=None keeps the rank-strided shard of the truncated file, and its sample ids are the positions."""
    for dp in (1, 2, 4):
        for r in range(dp):
            ds = Dataset(None, GBS, GBS // dp // 4, synthetic=True, n_samples=N_ROWS)
            ds.load(r, dp)
            assert not ds.shuffle
            full = N_ROWS - N_ROWS % GBS
            assert torch.equal(ds.input_X, torch.from_numpy(_X[r:full:dp]))
            for b in range(ds.get_num_batches()):
                q = b * GBS + torch.arange(GBS // dp) * dp + r
                assert torch.equal(ds.sample_ids(b), q)
                assert torch.equal(ds.load_batch(b)[0], torch.from_numpy(_X)[q])


def test_identity_permutation_reproduces_the_unshuffled_layout(monkeypatch):
    monkeypatch.setattr(F, "shuffle_index", lambda n, seed, epoch, q: torch.as_tensor(q, dtype=torch.int64))
    for dp in (1, 2):
        for r in range(dp):
            plain = Dataset(None, GBS, 16, synthetic=True, n_samples=N_ROWS)
            plain.load(r, dp)
            shuf = Dataset(None, GBS, 16, synthetic=True, n_samples=N_ROWS, shuffle_seed=7)
            shuf.load(r, dp)
            assert shuf.get_num_batches() == plain.get_num_batches()
            for b in range(plain.get_num_batches()):
                for a, c in zip(plain.load_batch(b), shuf.load_batch(b)):
                    assert torch.equal(a, c)
                for mu in range(plain.get_num_mubatches()):
                    assert torch.equal(plain.load_micro_batch_input(b, mu), shuf.load_micro_batch_input(b, mu))
                    assert torch.equal(plain.load_micro_batch_target(b, mu), shuf.load_micro_batch_target(b, mu))


# ------------------------------------------------------------------ sequential == DP == PP == DP x PP
STEPS = 9                          # crosses an epoch boundary (7 batches per epoch)


def _run_shuffled_layout(dp, pp, cls, seed=SEED, steps=STEPS):
    import test_equivalence as E

    orig_make, orig_execute = E._make_dataset, E.Worker.execute

    def make(dp_rank, dp_size, mubatch):
        ds = Dataset(None, GBS, mubatch, shuffle_seed=seed)
        return ds.from_arrays(_X, _Y, DP_rank=dp_rank, DP_size=dp_size)

    def execute(self, sched, step):
        n = self.dataset.get_num_batches()
        self.dataset.set_epoch(step // n)
        return orig_execute(self, sched, step % n)

    E._make_dataset, E.Worker.execute = make, execute
    try:
        return E.run_layout(dp, pp, cls, steps=steps)
    finally:
        E._make_dataset, E.Worker.execute = orig_make, orig_execute


@pytest.fixture(scope="module")
def sequential_shuffled():
    return _run_shuffled_layout(1, 1, NaiveParallelSchedule)


@pytest.mark.parametrize("dp,pp,cls", [
    (2, 1, NaiveParallelSchedule), (4, 1, GPipeSchedule),
    (1, 2, GPipeSchedule), (1, 4, PipeDreamSchedule),
    (2, 2, NaiveParallelSchedule), (2, 2, GPipeSchedule), (2, 2, PipeDreamSchedule),
])
def test_layout_matches_sequential_with_shuffling(sequential_shuffled, dp, pp, cls):
    _close(_run_shuffled_layout(dp, pp, cls), sequential_shuffled)


def test_shuffled_run_differs_from_unshuffled_and_from_another_seed(sequential_shuffled):
    import test_equivalence as E

    orig = E._make_dataset

    def make(dp_rank, dp_size, mubatch):     # the same 1000-row file, unshuffled
        ds = Dataset(None, GBS, mubatch)
        ds.local_batch_size = GBS // dp_size
        full = N_ROWS - N_ROWS % GBS
        return ds.from_arrays(_X[dp_rank:full:dp_size], _Y[dp_rank:full:dp_size])

    E._make_dataset = make
    try:
        plain = run_layout(1, 1, NaiveParallelSchedule, steps=N_ROWS // GBS)
    finally:
        E._make_dataset = orig
    shuffled = _run_shuffled_layout(1, 1, NaiveParallelSchedule, steps=N_ROWS // GBS)
    assert any(not torch.equal(a, b) for a, b in zip(plain, shuffled))
    other = _run_shuffled_layout(1, 1, NaiveParallelSchedule, seed=SEED + 1)
    assert any(not torch.equal(a, b) for a, b in zip(other, sequential_shuffled))


# ------------------------------------------------------------------ train.py
def _run(args, timeout=900):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


CLI = ["train.py", "--device", "cpu", "--engine", "python", "--no-eval", "--synthetic"]


def test_train_cli_smoke():
    r = _run(CLI + ["--shuffle", "--shuffle-seed", str(2 ** 64 - 1), "--steps", "3"])
    assert r.returncode == 0, r.stderr[-2000:]


def test_train_cli_resume_is_bitwise_and_refuses_a_mismatch(tmp_path):
    shuf = ["--shuffle", "--shuffle-seed", "77"]
    for args in (["--steps", "6", "--save", str(tmp_path / "full")], ["--steps", "3", "--save", str(tmp_path / "part")],
                 ["--steps", "6", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")]):
        r = _run(CLI + shuf + args)
        assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 6 and a["hparams"]["shuffle"] is True and a["hparams"]["shuffle_seed"] == 77
    assert torch.equal(a["weights"], b["weights"])
    for other in (["--shuffle", "--shuffle-seed", "78"], []):
        r = _run(CLI + other + ["--steps", "6", "--resume", str(tmp_path / "part")])
        assert r.returncode != 0 and "checkpoint was written with shuffle" in (r.stderr + r.stdout)
    # the same steps unshuffled give other weights
    r = _run(CLI + ["--steps", "6", "--save", str(tmp_path / "plain")])
    assert r.returncode == 0, r.stderr[-2000:]
    assert not torch.equal(a["weights"], torch.load(tmp_path / "plain" / "stage0of1.pt")["weights"])


def test_train_cli_checkpoint_without_shuffle_resumes_unshuffled(tmp_path):
    r = _run(CLI + ["--steps", "2", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    path = tmp_path / "part" / "stage0of1.pt"
    ck = torch.load(path)
    del ck["hparams"]["shuffle"], ck["hparams"]["shuffle_seed"]
    torch.save(ck, path)
    r = _run(CLI + ["--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(CLI + ["--shuffle", "--steps", "3", "--resume", str(tmp_path / "part")])
    assert r.returncode != 0 and "checkpoint was written with shuffle" in (r.stderr + r.stdout)


@pytest.mark.parametrize("seed", ["-1", str(2 ** 64)])
def test_train_cli_rejects_a_bad_seed(seed):
    r = _run(CLI + ["--shuffle", "--shuffle-seed", seed, "--steps", "1"])
    assert r.returncode != 0 and "shuffle_seed" in r.stderr
