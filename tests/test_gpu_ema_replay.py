"""The EMA in the data-parallel kernels and in pipeline stages, on one GPU, through the replays of test_gpu_dp_replay (a
replica of dp 1/2/4/8, its peers replayed from memory) and test_gpu_pp_replay (a pipeline stage, its neighbours'
boundary tiles and flags replayed).

Each case runs twice with the same inputs: as the replay builds it, and with ``ema_decay`` added to its optimizer.  The
replays run unchanged and check everything they check without EMA; around every step a wrapper of
``NativeWorker.step_from`` records the EMA before and after the step and the weights the step wrote.  Then:
  * the weights of every step equal those of the EMA-free run, bit for bit;
  * every EMA entry the replica owns is ``ema_lerp_ref(E0, W_after, alpha)`` bit for bit, every other entry (the peers'
    elements, the padding) is unchanged.  The flat-arena update passes over the padding as well, so there the padding
    follows the weights' (which the replays poison with NaN; in a real run it is zero and stays zero);
  * ``ema_state()`` contributes exactly the owned entries (shared ones from DP rank 0) to its all-reduce.
The decay 0.3 makes alpha 1 on the first step and 0.7 (the alpha >= 0.5 branch of the lerp) after it; one LL and one
flag case run at 0.999 for the other branch."""
import pytest
import torch

import test_gpu_dp_replay as DP
import test_gpu_pp_replay as PP
from shallowspeed_b200.ops.functional import ema_lerp_ref

pytestmark = pytest.mark.gpu


def _record(monkeypatch, decay, rec):
    """Wrap NativeWorker.step_from (and, with a decay, the optimizer the replay builds) for one run."""
    import shallowspeed_b200.optimizer as O
    from shallowspeed_b200.parallel import engine as E

    if decay is not None:
        base = O.SGD

        class EmaSGD(base):
            def __init__(self, *a, **kw):
                super().__init__(*a, ema_decay=decay, **kw)

        monkeypatch.setattr(O, "SGD", EmaSGD)
    orig = E.NativeWorker.step_from

    def step_from(self, sched, x, y):
        arena = self.model.arena
        torch.cuda.synchronize()
        e0 = arena.ema.clone() if arena.ema is not None else None
        alpha = self.optimizer.ema_alpha
        eng = orig(self, sched, x, y)
        eng.synchronize()
        torch.cuda.synchronize()
        # the flat-arena update (plan op "sgd") passes over the whole arena, padding included
        flat = any(line.split()[1] == "sgd" for line in eng.plan_text(0).splitlines() if line.strip())
        step = dict(W1=arena.weights[: arena.numel].clone(), E0=e0, alpha=alpha, model=self.model, flat=flat,
                    protos=list(eng.layer_protocols()), dp=self.dp_comm.Get_size(), rank=self.dp_comm.Get_rank())
        if e0 is not None:
            step["E1"] = arena.ema.clone()
            step["state"] = _state_contribution(self, monkeypatch)
        rec.append(step)
        return eng

    monkeypatch.setattr(E.NativeWorker, "step_from", step_from)


def _state_contribution(worker, monkeypatch):
    """What ``ema_state()`` feeds into its DP all-reduce on this replica (the all-reduce itself replaced by identity)."""
    import torch.distributed as dist

    if worker.dp_comm.Get_size() == 1:
        return worker.ema_state()
    with monkeypatch.context() as m:
        m.setattr(dist, "all_reduce", lambda t, op=None, group=None: None)
        m.setattr(worker.dp_comm, "group", None, raising=False)
        return worker.ema_state()


def _owned(model, protos, dp, rank, shared_to_rank0=False):
    from shallowspeed_b200.parallel.engine import owned_elements

    return owned_elements(model.arena, model.linears, protos, dp, rank, shared_to_rank0=shared_to_rank0).cuda()


def _real(arena):
    m = torch.zeros(arena.numel, dtype=torch.bool, device="cuda")
    for i, (o, k) in enumerate(arena.blocks):
        m[arena.offsets[i]: arena.offsets[i] + o * arena.lds[i]].view(o, arena.lds[i])[:, : k + 1] = True
    return m


def _same(a, b):
    """Bitwise equal, NaN where the other is NaN."""
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def _check(plain, ema):
    assert len(plain) == len(ema) > 0
    model = ema[0]["model"]
    real = _real(model.arena)
    for t, (a, b) in enumerate(zip(plain, ema)):
        assert torch.equal(a["W1"][real], b["W1"][real]), f"step {t + 1}: the EMA changed the weights"
        owned = _owned(model, b["protos"], b["dp"], b["rank"]) & real
        if b["flat"]:
            owned |= ~real
        want = ema_lerp_ref(b["E0"], b["W1"], b["alpha"])
        assert torch.equal(b["E1"][owned & real], want[owned & real]), f"step {t + 1}: an owned EMA entry differs"
        pad = owned & ~real                                    # NaN where the replay poisoned the weights' padding
        assert _same(b["E1"][pad], want[pad])
        assert torch.equal(b["E1"][~owned], b["E0"][~owned]), f"step {t + 1}: a non-owned EMA entry (or padding) changed"
        assert bool(owned.any()) and (b["alpha"] == 1.0) == (t == 0)
        mine = _owned(model, b["protos"], b["dp"], b["rank"], shared_to_rank0=True)
        n = model.arena.numel
        contribution = torch.where(mine, b["E1"], torch.zeros_like(b["E1"]))
        assert _same(b["state"].to(contribution.device)[:n], contribution[:n]), f"step {t + 1}: ema_state()"


def _twice(monkeypatch, decay, run):
    plain, ema = [], []
    with monkeypatch.context() as m:
        _record(m, None, plain)
        run(m)
    with monkeypatch.context() as m:
        _record(m, decay, ema)
        run(m)
    _check(plain, ema)


@pytest.mark.parametrize("dp,rank,stateful,decay", [(2, 1, False, 0.3), (2, 0, True, 0.3), (4, 2, False, 0.3),
                                                    (4, 3, True, 0.999), (8, 7, False, 0.3), (8, 5, True, 0.3)])
def test_ll_replay_ema(dp, rank, stateful, decay, monkeypatch):
    def run(m):
        DP._run(f"ll dp{dp} r{rank} gate1 fp32{' stateful' if stateful else ''}", DP.REF, dp, rank, "ll",
                env={"SSB_DP_GATE": "1"}, mb_rows=128 // dp // 4, n_mu=4, stateful=stateful, monkeypatch=m)

    _twice(monkeypatch, decay, run)


@pytest.mark.parametrize("sizes,dp,rank,shot,stateful,decay", [
    ("ref", 2, 1, "one-shot", False, 0.3), ("ref", 2, 0, "two-shot", False, 0.3), ("ref", 4, 1, "two-shot", True, 0.3),
    ("ref", 4, 0, "one-shot", True, 0.999), ("wide", 2, 1, "two-shot", True, 0.3), ("wide", 2, 0, "one-shot", False, 0.3)])
def test_flag_replay_ema(sizes, dp, rank, shot, stateful, decay, monkeypatch):
    env = {"SSB_DP_LL": "0", "SSB_DP_ONE_SHOT" if shot == "one-shot" else "SSB_DP_TWO_SHOT": "1"}

    def run(m):
        DP._run(f"flags {sizes} dp{dp} r{rank} {shot}{' stateful' if stateful else ''}",
                {"ref": DP.REF, "wide": DP.WIDE}[sizes], dp, rank, shot, env=env, stateful=stateful, monkeypatch=m)

    _twice(monkeypatch, decay, run)


@pytest.mark.parametrize("name", ["ref-one-shot", "ref-reduce-sgd-two-shot-stateful"])
def test_dp1_flag_protocol_ema(name, monkeypatch):
    sizes, proto, env, precision, st = DP.DP1[name]

    def run(m):
        DP._run(f"dp1 {name}", sizes, 1, 0, proto, env=env, precision=precision, stateful=st, monkeypatch=m)

    _twice(monkeypatch, 0.3, run)


# pipeline stages: the deferred grouped wave (default), the per-micro-batch accumulation + flat-arena update
# (SSB_PP_DEFER_WGRAD=0) and the layer-wise path; dp x pp stages under the LL wave and under dp_reduce_sgd, where the
# owned entries are owned_elements of the stage's own layers
PP_NAMES = ["ref-pp2-s0-naive", "ref-pp2-s1-1f1b-mb24-tf32", "ref-pp4-s2-gpipe-stateful", "ref-pp4-s3-1f1b",
            "ref-pp4-s2-no-defer", "ref-pp4-s0-no-chain", "wide-pp2-s1-gpipe", "ref-pp4-s1-dp4-r3-1f1b",
            "ref-pp4-s1-dp2-r1-no-defer"]


@pytest.mark.parametrize("name", PP_NAMES)
def test_pp_stage_replay_ema(name, monkeypatch):
    _twice(monkeypatch, 0.3, lambda m: PP._run(name, m))
