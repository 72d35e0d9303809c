"""Pipeline stages on ONE GPU, per element against fp64, by running one stage of a pp-way pipeline and replaying its
neighbours' boundary tiles and flags from memory.

Every message of the peer-memory pipeline transport (``runtime/pp_context.h``) is data at a known address stamped with
the step's epoch: a boundary tile in the consumer's receive slot ``act_in[mu]`` / ``dz_in[mu]``, its arrival flag, and
the credit that hands a producer its slots back.  Before a step the test writes what the two neighbours would have sent
stage s: the input tiles of every micro-batch (non-first stage), the received gradients (non-last stage, training),
every arrival flag s polls set to the step's epoch e and both of s's credits set to e - 1.  Every wait the stage performs
is then satisfied before the launch, and nothing depends on a second process.  The real engine (``NativeWorker._build``
with ``pp_transport="peer"`` and a stand-in pipeline communicator of size pp and rank s) runs s against neighbour contexts
that are plain allocations of this process (``PpContext.open_local``).  Their receive slots hold NaN and every word of
their flag arrays a sentinel that is never an epoch; after the step the test reads back what s sent into them.

Checked per element and per micro-batch, from the engine's own buffers (the oracles of ``test_gpu_chain.py``,
``test_gpu_gemm.py`` and ``test_gpu_cross_entropy.py``), so errors cannot cascade:
* forward: every layer from the kernel's act[l - 1]; on a non-first stage act[0] IS the injected receive slot;
* loss head (last stage): probabilities, dz_L and the loss of every micro-batch, MSE and cross-entropy;
* received gradient (non-last stage): dz[L] bit-equal to the injected tile masked by relu'(act[L]), the copy the
  weight-gradient GEMMs read;
* dgrad chain, layer 1 included on non-first stages; on the first stage dz[0] is never written;
* update: the deferred wave over all rows of the stage, or per-micro-batch weight gradients accumulating through memory
  ((n_mu - 1) more fp32 roundings) and a separate SGD pass; plain or stateful, at each step's learning rate;
* outbound tiles: slot mu of the neighbour bit-equal to micro-batch mu of my act[L] / dz[0] (a wrong micro-batch
  resolution or a row offset fails here), and nothing written into the slots nobody sends to;
* outbound flags: exactly the neighbours' arrival flags of the n_mu micro-batches and the one credit per neighbour hold e,
  every other neighbour word still the sentinel, my own flags untouched.

dp x pp (``dp`` / ``rank`` of a case): the stage is also replica ``rank`` of a dp-way group (a stand-in DP communicator,
``comm_mode="fused"``, peer DpContexts of this process), and the DP half of ``test_gpu_dp_replay.py`` runs next to the
pipeline half: ``dp_prefill`` writes the DP peers' LL lines or partial tiles and flags before every step, ``dp_check``
replaces the local update check (5.) with the owned updates against the reduced fp64 oracle, the copied or untouched
peer elements, every outbound LL line or staging tile and flag, and the momentum ownership, all from the stage's own act
(act[0] IS the injected receive slot) and dz (dz[L] IS the masked receive slot, or, for a residual last layer, the
engine's own gated copy).  The plan must run the deferred LL wave (``dp_ll``, every layer ``DP_PROTO_LL``) or one
``dp_reduce_sgd`` per layer behind per-micro-batch weight gradients, one DP epoch bump and one pipeline epoch bump; both
epochs advance by one per step.  The stage's MLP and the loss-head oracle scale by the global batch mb * n_mu * dp; the
injected peer partials take the scale of the stage's own (from its input and received gradient).  The Linear-less last
stage of pp = 8 runs its head with a DpContext without layers: no DP kernel, nothing sent to the peers, both epochs
advance.  The residual GELU stage with dropout is checked per element by ``test_gpu_residual.check_residual_layers``
with the masks of samples (mu * mb + n) * dp + rank at the stage's layer_base.

Measured on an H100 80GB HBM3 (700 W): the worst err / bound of the 16 dp x pp cases is 0.499 (the update of
wide-pp2-s1-dp4-r3-gpipe), of all cases 0.887 (the tf32 update of ref-pp2-s1-1f1b-mb24-tf32); the whole file, CPU
tests included, runs in 39 s.

Not covered here, and left to ``test_gpu_multi.py``: concurrent neighbours and peers, real waiting on credits and flags
(every wait is satisfied before the launch), NVLink visibility ordering, the NCCL and NVLS transports, and
``optimizer_state()`` / ``ema_state()`` assembled across both groups.
"""
import gc
import math
import zlib

import pytest
import torch

from test_gpu_chain import (FP32_ULP, HEAD_RTOL, LOGIT_SPREAD, RTOL, _gather, _init_weights, _pitched, _poison,
                            dgrad_oracle, excess, fwd_oracle, head_oracle)
from test_gpu_cross_entropy import ce_head_oracle
from test_gpu_dp_replay import (_StandInComm, _device_view, dp_check, dp_peer_data, dp_prefill, dp_setup, flag_geometry,
                                local_dp_context, ll_tiles)
from test_gpu_gemm import grad_oracle, rtol_for, sgd_oracle
from test_gpu_residual import check_residual_layers

REF = [784, 128, 127, 126, 125, 124, 123, 10]     # the reference model; pp = 4 cuts it at the ragged 127 / 125
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]  # layer-wise GEMMs, 520-wide boundaries at pp = 2
RES_SIZES = [784, 48, 48, 48, 48, 48, 48, 10]      # pp = 4 stage 1: two residual layers, one on each boundary
FEATURES = dict(activation="gelu", dropout=0.3, dropout_seed=0x5EED_0F_0DD_5EED, residual=True)
LR, MU, WD = 0.5, 0.9, 5e-4
LR_STEPS = (0.5, 0.25, 0.375)                       # the case that changes opt.lr between steps (exact in fp32)
STEPS = 3                                           # the epoch advances, credits come back, the staging set alternates
DZ_SCALE = 1e-2                                     # injected gradients: updates of ~1e-2 against weights of ~1e-1
SENTINEL = 0x0BADF1A6                               # a neighbour flag word nobody may write; never an epoch here
SMALL_TILE_F4 = 2048                                # kPpSmallTileF4 (pp_context.h): one-CTA push up to 32 KB
NAN = float("nan")
WORST = {}


def _C():
    from shallowspeed_b200 import _C as mod

    return mod


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ================================================================================================== the case grid
def _case(sizes, pp, s, sched, mb=32, n_mu=4, env=None, precision="fp32", stateful=False, loss="mse", push=None, dp=1,
          rank=0, model=None):
    """``push``: which push kernel the unfolded transport must reach in its outbound directions ("small" / "multi").
    ``dp`` / ``rank``: the stage is DP replica ``rank`` of ``dp`` (its peers replayed as in test_gpu_dp_replay).
    ``model``: MLP keywords (activation, dropout, residual) of the feature cases."""
    return dict(sizes=sizes, pp=pp, s=s, sched=sched, mb=mb, n_mu=n_mu, env=env or {}, precision=precision,
                stateful=stateful, loss=loss, push=push, dp=dp, rank=rank, model=model or {})


UNFOLD = {"SSB_PP_FOLD": "0"}
CASES = {
    # reference model, pp = 2: folded boundaries (single-chunk and multi-chunk stores), every schedule
    "ref-pp2-s0-naive": _case(REF, 2, 0, "naive", n_mu=2),
    "ref-pp2-s1-naive": _case(REF, 2, 1, "naive", n_mu=2),
    "ref-pp2-s0-gpipe-mb24-tf32": _case(REF, 2, 0, "gpipe", mb=24, precision="tf32"),
    "ref-pp2-s1-1f1b-mb24-tf32": _case(REF, 2, 1, "1f1b", mb=24, precision="tf32"),
    # the unfolded transport: one-CTA pushes at mb 32, multi-CTA pushes (shared completion counter) at mb 128
    "ref-pp2-s0-unfolded": _case(REF, 2, 0, "1f1b", env=UNFOLD, push="small"),
    "ref-pp2-s1-unfolded": _case(REF, 2, 1, "1f1b", env=UNFOLD, push="small"),
    "ref-pp2-s0-unfolded-mb128": _case(REF, 2, 0, "gpipe", mb=128, n_mu=2, env=UNFOLD, push="multi"),
    "ref-pp2-s1-unfolded-mb128": _case(REF, 2, 1, "gpipe", mb=128, n_mu=2, env=UNFOLD, push="multi"),
    # reference model, pp = 4: every stage; the middle ones cut at 127 / 125
    "ref-pp4-s0-1f1b": _case(REF, 4, 0, "1f1b"),
    "ref-pp4-s1-1f1b-mb100": _case(REF, 4, 1, "1f1b", mb=100, n_mu=2),
    "ref-pp4-s2-gpipe-stateful": _case(REF, 4, 2, "gpipe", stateful=True),
    "ref-pp4-s3-1f1b": _case(REF, 4, 3, "1f1b"),
    "ref-pp4-s3-gpipe-ce": _case(REF, 4, 3, "gpipe", n_mu=2, loss="cross_entropy"),
    "ref-pp4-s1-naive-nmu1-mb64": _case(REF, 4, 1, "naive", mb=64, n_mu=1),
    "ref-pp4-s2-gpipe-nmu12": _case(REF, 4, 2, "gpipe", mb=24, n_mu=12),
    "ref-pp4-s1-no-defer-nmu12": _case(REF, 4, 1, "1f1b", mb=24, n_mu=12, env={"SSB_PP_DEFER_WGRAD": "0"}),
    "ref-pp4-s2-no-defer": _case(REF, 4, 2, "naive", env={"SSB_PP_DEFER_WGRAD": "0"}),
    # layer-wise path (GEMM per layer, OP_RELU_MASK on the received gradient, stand-alone loss head)
    "ref-pp4-s0-no-chain": _case(REF, 4, 0, "gpipe", env={"SSB_NO_CHAIN": "1"}, push="small"),
    "ref-pp4-s1-no-chain-mb24": _case(REF, 4, 1, "naive", mb=24, n_mu=2, env={"SSB_NO_CHAIN": "1"}, push="small"),
    "ref-pp4-s3-no-chain": _case(REF, 4, 3, "1f1b", env={"SSB_NO_CHAIN": "1"}, push="small"),
    # inference on first, middle and last stages (the forward-only flag branch of the chain kernel)
    "ref-pp4-s0-inference": _case(REF, 4, 0, "inference"),
    "ref-pp4-s1-inference": _case(REF, 4, 1, "inference"),
    "ref-pp4-s2-inference-unfolded": _case(REF, 4, 2, "inference", env=UNFOLD, push="small"),
    "ref-pp4-s3-inference": _case(REF, 4, 3, "inference"),
    # pp = 8: a one-Linear middle stage, and the last stage without any Linear (loss head only)
    "ref-pp8-s3-1f1b": _case(REF, 8, 3, "1f1b"),
    "ref-pp8-s7-1f1b": _case(REF, 8, 7, "1f1b", push="small"),
    "ref-pp8-s7-inference": _case(REF, 8, 7, "inference"),
    # wide model, pp = 2: layer-wise GEMMs, 520-wide boundaries moved by the multi-CTA push in both directions
    "wide-pp2-s0-gpipe": _case(WIDE, 2, 0, "gpipe", n_mu=2, push="multi"),
    "wide-pp2-s1-gpipe": _case(WIDE, 2, 1, "gpipe", n_mu=2, push="multi"),
    # dp x pp: the stage is replica `rank` of a dp-way group; its DP peers are replayed next to its pipeline neighbours.
    # The deferred LL wave (folded): X is act_in on a non-first stage, dZ the masked dz_in on a non-last one
    "ref-pp2-s0-dp2-r1-gpipe": _case(REF, 2, 0, "gpipe", dp=2, rank=1),
    "ref-pp2-s1-dp2-r0-1f1b": _case(REF, 2, 1, "1f1b", dp=2, rank=0),
    "ref-pp2-s1-dp2-r0-1f1b-ce": _case(REF, 2, 1, "1f1b", n_mu=2, loss="cross_entropy", dp=2, rank=0),
    "ref-pp4-s1-dp4-r3-1f1b": _case(REF, 4, 1, "1f1b", dp=4, rank=3),
    "ref-pp4-s2-dp8-r5-gpipe-stateful": _case(REF, 4, 2, "gpipe", stateful=True, dp=8, rank=5),
    "ref-pp4-s2-dp2-r1-unfolded": _case(REF, 4, 2, "1f1b", env=UNFOLD, push="small", dp=2, rank=1),
    # per-micro-batch weight gradients through memory, then one dp_reduce_sgd per layer (LL zones allocated, unused)
    "ref-pp4-s1-dp2-r1-no-defer": _case(REF, 4, 1, "1f1b", env={"SSB_PP_DEFER_WGRAD": "0"}, dp=2, rank=1),
    # the flag protocol on a stage
    "ref-pp4-s1-dp4-r2-flags-two-shot-stateful": _case(REF, 4, 1, "gpipe", env={"SSB_DP_LL": "0", "SSB_DP_TWO_SHOT": "1"},
                                                       stateful=True, dp=4, rank=2),
    "ref-pp4-s0-dp4-r1-flags-one-shot": _case(REF, 4, 0, "1f1b", env={"SSB_DP_LL": "0"}, dp=4, rank=1),
    "ref-pp4-s3-dp2-r1-no-chain": _case(REF, 4, 3, "1f1b", env={"SSB_NO_CHAIN": "1"}, push="small", dp=2, rank=1),
    # a one-Linear stage, and the stage without any Linear: a DpContext with no layers
    "ref-pp8-s3-dp2-r1-1f1b": _case(REF, 8, 3, "1f1b", dp=2, rank=1),
    "ref-pp8-s7-dp2-r1-1f1b": _case(REF, 8, 7, "1f1b", push="small", dp=2, rank=1),
    # layer-wise GEMMs: one-shot and two-shot layers, multi-CTA pushes
    "wide-pp2-s0-dp2-r1-gpipe": _case(WIDE, 2, 0, "gpipe", n_mu=2, push="multi", dp=2, rank=1),
    "wide-pp2-s1-dp4-r3-gpipe": _case(WIDE, 2, 1, "gpipe", n_mu=2, push="multi", dp=4, rank=3),
    # residual GELU layers with dropout on both boundaries: the skip gradient is dz_in, the wgrad reads dz[L].  dp 4, so
    # that rank 1 owns LL rows of the 48-wide layers (rows 32 .. 47; at dp 2 it would own none)
    "res-pp4-s1-dp4-r1-gelu-drop": _case(RES_SIZES, 4, 1, "1f1b", dp=4, rank=1, model=FEATURES),
    "res-pp4-s1-dp4-r1-gelu-drop-no-chain": _case(RES_SIZES, 4, 1, "1f1b", env={"SSB_NO_CHAIN": "1"}, push="small", dp=4,
                                                 rank=1, model=FEATURES),
}


def _local(c):
    from shallowspeed_b200.layers import stage_sizes

    return stage_sizes(c["sizes"], c["s"], c["pp"])


def _lds(local):
    """(ld_in, ld_out) of a stage: every boundary row is padded to 8 floats (pipe_engine.cpp, alloc_buffers)."""
    return -(-local[0] // 8) * 8, -(-local[-1] // 8) * 8


# ================================================================================================== message checks
def flag_layout(buffers):
    """{range name: (first word, words)} of a PpContext's flag array, from the pointers ``buffers()`` reports."""
    base = buffers["flags"][0]
    return {k: ((buffers[k][0] - base) // 4, buffers[k][1] // 4)
            for k in ("act_arrived", "dz_arrived", "act_credit", "dz_credit")}


def own_flags(layout, words, n_mu, e):
    """The flag array of the stage under test before step ``e``: every arrival flag it polls at e, both credits at
    e - 1, everything else 0."""
    f = torch.zeros(words, dtype=torch.int32)
    for name in ("act_arrived", "dz_arrived"):
        f[layout[name][0]: layout[name][0] + n_mu] = e
    for name in ("act_credit", "dz_credit"):
        f[layout[name][0]] = e - 1
    return f


def neighbour_flags(layout, words, n_mu, e, side, training):
    """What the flag array of neighbour ``side`` ("prev" / "next") must hold after step ``e``: the arrival flags of
    the tiles the stage sent it and the credit of the slots it consumed from it at e, every other word the sentinel."""
    f = torch.full((words,), SENTINEL, dtype=torch.int32)
    if side == "next":
        f[layout["act_arrived"][0]: layout["act_arrived"][0] + n_mu] = e     # my act pushes land in its act_in
        if training:
            f[layout["dz_credit"][0]] = e                                    # I consumed its dz pushes
    else:
        if training:
            f[layout["dz_arrived"][0]: layout["dz_arrived"][0] + n_mu] = e
        f[layout["act_credit"][0]] = e                                       # I consumed its act pushes
    return f


def check_flags(got, want, what):
    bad = (got != want).nonzero().flatten().tolist()
    assert not bad, f"{what}: {len(bad)} flag words differ, first at word {bad[0]}: {int(got[bad[0]])} != {int(want[bad[0]])}"


def check_tiles(slots, tiles, cols, what):
    """Slot mu of a receive buffer ([n_mu, mb, ld]) bit-equal to my tile of micro-batch mu ([n_mu, mb, >= cols]) on the
    valid columns."""
    got = slots[:, :, :cols].float().contiguous().view(torch.int32)
    want = tiles[:, :, :cols].float().contiguous().view(torch.int32)
    bad = (got != want).nonzero().tolist()
    assert not bad, f"{what}: {len(bad)} elements differ, first at (micro-batch, row, column) {tuple(bad[0])}"


def check_received_grad(dz_L, act_L, injected, cols, what):
    """dz[L] after the step bit-equal to the injected gradient masked by relu'(act[L]) on the valid columns."""
    want = torch.where(act_L[..., :cols] > 0, injected[..., :cols].float(), torch.zeros((), dtype=torch.float32))
    got = dz_L[..., :cols].float().contiguous().view(torch.int32)
    bad = (got != want.contiguous().view(torch.int32)).nonzero().tolist()
    assert not bad, f"{what}: {len(bad)} elements differ from the masked received gradient, first at {tuple(bad[0])}"


def _nan_pad(tile, ld):
    out = torch.full((tile.shape[0], ld), NAN, dtype=torch.float32)
    out[:, : tile.shape[1]] = tile
    return out


def _plan(text):
    return [line.split() for line in text.splitlines() if line.strip()]


def check_plan(text, n_mu, folded, deferred, first, last, training):
    """The lowered plan of one staging set: no push / wait kernels when the boundaries are folded into the chain
    launches, otherwise one push per micro-batch and outbound direction and one wait per micro-batch and inbound
    direction; one epoch bump and one credit per step; the grouped weight-gradient wave exactly when it is deferred."""
    ops = _plan(text)
    count = lambda name: sum(1 for o in ops if o[1] == name)                                 # noqa: E731
    per_mu = lambda name: sorted(int(t[3:]) for o in ops if o[1] == name for t in o if t.startswith("mu="))  # noqa: E731
    n_out = (0 if last else 1) + (0 if first or not training else 1)
    n_in = (0 if first else 1) + (0 if last or not training else 1)
    if folded:
        assert count("pp_push") == 0 and count("pp_wait") == 0, text
    else:
        assert per_mu("pp_push") == sorted(list(range(n_mu)) * n_out), text
        assert per_mu("pp_wait") == sorted(list(range(n_mu)) * n_in), text
    assert count("pp_bump_epoch") == 1 and count("pp_credit") == 1, text
    assert (count("wgrad_group") == 1) == deferred and count("wgrad_group") <= 1, text


def _note(case, res):
    worst = max(res, key=res.get)
    WORST[case] = (res[worst], worst)
    print(f"\n[pp-replay] {case}: max err/bound {res[worst]:.3g} ({worst})")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, (case, bad)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for case, (v, what) in WORST.items():
        print(f"[pp-replay] worst err/bound {v:.3g} ({what})  {case}")


# ================================================================================================== the stage
class _Ctx:
    """Device tensors over one PpContext's buffers."""

    def __init__(self, ctx, n_mu, mb, ld_in, ld_out):
        b = ctx.buffers()
        self.act_in = _device_view(b["act_in"], "<f4").view(n_mu, mb, ld_in)
        self.dz_in = _device_view(b["dz_in"], "<f4").view(n_mu, mb, ld_out)
        self.flags = _device_view(b["flags"], "<i4")
        self.epoch = _device_view(b["epoch"], "<i4")
        self.act_in_ptr = b["act_in"][0]
        self.layout = flag_layout(b)


SCHEDULES = {"naive": "NaiveParallelSchedule", "gpipe": "GPipeSchedule", "1f1b": "PipeDreamSchedule",
             "inference": "InferenceSchedule"}


def _build_stage(c, monkeypatch):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E

    C = _C()
    pp, s, mb, n_mu, dp = c["pp"], c["s"], c["mb"], c["n_mu"], c["dp"]
    model = MLP(c["sizes"], s, pp, mb * n_mu * dp, loss=c["loss"], **c["model"]).to("cuda")
    rule = dict(momentum=MU, weight_decay=WD, nesterov=True) if c["stateful"] else {}
    opt = SGD(model.parameters(), LR, arena=model.arena, **rule)
    ctxs = {"dp": []}

    def make_pp_context(comm, eng, n_mu, mb_rows, is_first, is_last):
        # make_pp_context with neighbours that are contexts of this process instead of CUDA IPC mappings
        ld_in, ld_out = eng.boundary_lds()
        me = C.PpContext(int(n_mu), int(mb_rows), int(ld_in), int(ld_out), bool(is_first), bool(is_last))
        prev = None if is_first else C.PpContext(int(n_mu), int(mb_rows), int(ld_in), int(ld_in), comm.rank == 1, False)
        nxt = None if is_last else C.PpContext(int(n_mu), int(mb_rows), int(ld_out), int(ld_out), False,
                                               comm.rank + 2 == comm.size)
        me.open_local(prev, nxt)
        ctxs.update(me=me, prev=prev, next=nxt)
        torch.cuda.synchronize()
        return me

    monkeypatch.setattr(E, "make_nccl_comm", lambda comm: None)
    monkeypatch.setattr(E, "make_pp_context", make_pp_context)
    monkeypatch.setattr(E, "make_dp_context", local_dp_context(ctxs["dp"]))

    class _Shape:
        mubatch_size = mb

    w = E.NativeWorker(_StandInComm(dp, c["rank"]) if dp > 1 else None, _StandInComm(pp, s), model, _Shape(), opt,
                       comm_mode="fused", precision=c["precision"], pp_transport="peer")
    return w, model, opt, ctxs


def _ll_on(c, local):
    """Whether the stage's DpContext allocates LL landing zones (dp_context.cpp)."""
    tiles = sum(_C().dp_ll_tiles(i, o) for i, o in zip(local[:-1], local[1:]))
    return c["dp"] > 1 and c["env"].get("SSB_DP_LL", "1") != "0" and 0 < tiles <= 128


def _dp_protocol(c, local, deferred):
    """"ll" when the deferred wave runs the LL kernel, else the flag protocols of the stage's layers ("one-shot",
    "two-shot" or both, "+"-joined; "" for a stage without layers)."""
    if deferred and c["dp"] > 1:
        return "ll"
    geom = flag_geometry(local, c["dp"], two_shot="SSB_DP_TWO_SHOT" in c["env"], one_shot="SSB_DP_ONE_SHOT" in c["env"])
    return "+".join(n for n, on in (("one-shot", any(g["one_shot"] for g in geom)),
                                    ("two-shot", any(not g["one_shot"] for g in geom))) if on)


def _stage_grad_scale(local, relu, Ws, x, t, dz_top, n_mu, batch, loss):
    """Per layer of a stage, the mean |weight gradient| of a plain fp64 ReLU backward pass from the stage input ``x``
    and, on a non-last stage, the received gradient ``dz_top`` (else the loss head of the targets ``t``): the scale of
    the injected peer partials."""
    L, acts = len(local) - 1, [x.double()]
    for l in range(L):
        acts.append(fwd_oracle(acts[-1], Ws[l][:, :-1], Ws[l][:, -1], relu[l], 0.0)[0])
    if dz_top is None:
        mb, oracle = x.shape[0] // n_mu, ce_head_oracle if loss == "cross_entropy" else head_oracle
        dz = torch.cat([oracle(acts[L][mu * mb:(mu + 1) * mb], t[mu * mb:(mu + 1) * mb], batch, 0.0)[1][0]
                        for mu in range(n_mu)])
    else:
        dz = dz_top.double() * ((acts[L] > 0).double() if relu[-1] else 1.0)
    out = [None] * L
    for l in range(L, 0, -1):
        out[l - 1] = float(torch.cat([dz.T @ acts[l - 1], dz.sum(0)[:, None]], 1).abs().mean())
        if l > 1:
            dz = dgrad_oracle(dz, Ws[l - 1][:, :-1], acts[l - 1] if relu[l - 2] else torch.ones_like(acts[l - 1]), 0.0)[0]
    return out


def _run(name, monkeypatch):
    from shallowspeed_b200 import pipe

    c = CASES[name]
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    pp, s, mb, n_mu, precision, dp, rank = c["pp"], c["s"], c["mb"], c["n_mu"], c["precision"], c["dp"], c["rank"]
    local = _local(c)
    L, rows = len(local) - 1, mb * n_mu
    batch = rows * dp                                       # the global batch the loss head scales by
    feat = bool(c["model"])                                 # gated, dropped, residual layers: check_residual_layers
    first, last, training = s == 0, s == pp - 1, c["sched"] != "inference"
    ld_in, ld_out = _lds(local)
    w, model, opt, ctxs = _build_stage(c, monkeypatch)
    sched = getattr(pipe, SCHEDULES[c["sched"]])(n_mu, pp, s)
    eng = w.engine_for(sched)
    arena = model.arena
    gen = _gen(name)
    rtol = RTOL[precision]
    relu = [lin.activation is not None for lin in model.linears]

    # ---- the path this case is meant to exercise
    chain = "SSB_NO_CHAIN" not in c["env"] and c["sizes"] is not WIDE and L >= 1
    assert eng.uses_chain() == chain
    folded = chain and c["env"].get("SSB_PP_FOLD", "1") != "0"
    deferred = (chain and training and c["env"].get("SSB_PP_DEFER_WGRAD", "1") != "0"
                and (dp == 1 or _ll_on(c, local)))
    for st in (0, 1):
        check_plan(eng.plan_text(st), n_mu, folded, deferred and dp == 1, first, last, training)
    d = None
    if dp > 1:
        # the DP kernel of the plan: the deferred LL wave, or one dp_reduce_sgd per layer behind the final backward
        C = _C()
        protos, proto = list(eng.layer_protocols()), _dp_protocol(c, local, deferred)
        assert ctxs["dp"][rank].ll_tiles() == (len(ll_tiles(local)) if _ll_on(c, local) else 0)
        d = dp_setup(ctxs["dp"], rank, proto, local, c["env"], arena, protos)
        for st in (0, 1):
            text = eng.plan_text(st)
            ops = [o[1] for o in _plan(text)]
            assert ops.count("bump_epoch") == 1 and "fused_wgrad_dp" not in ops, text
            if proto == "ll":
                assert ops.count("dp_ll") == 1 and "dp_reduce_sgd" not in ops, text
            else:
                assert ops.count("dp_reduce_sgd") == L and "dp_ll" not in ops, text
        if proto == "ll":
            assert protos == [C.DP_PROTO_LL] * L
        else:
            got = ctxs["dp"][rank].layer_geometry()
            assert len(got) == len(d["geom"]) == L
            for g, h in zip(d["geom"], got):
                assert all(g[key] == h[key] for key in g), (g, h)
            assert protos == [C.DP_PROTO_ALL if g["one_shot"] else C.DP_PROTO_TWO_SHOT for g in d["geom"]]
    assert tuple(eng.boundary_lds()) == (ld_in, ld_out)
    if c["push"] is not None:
        assert not folded
        tiles = ([mb * ld_out] if not last else []) + ([mb * ld_in] if not first and training else [])
        assert all((n // 4 > SMALL_TILE_F4) == (c["push"] == "multi") for n in tiles), (tiles, c["push"])

    me = _Ctx(ctxs["me"], n_mu, mb, ld_in, ld_out)
    nb = {side: _Ctx(ctxs[side], n_mu, mb, ld_in if side == "prev" else ld_out, ld_in if side == "prev" else ld_out)
          for side in ("prev", "next") if ctxs[side] is not None}
    for mu in range(n_mu):
        if not first:
            assert eng.act(mu, 0).data_ptr() == me.act_in_ptr + 4 * mu * mb * ld_in, "act[0] is not the receive slot"

    # ---- data of every step
    xs = [torch.randn(rows, local[0], generator=gen) for _ in range(STEPS)]
    if not first:
        for x in xs:
            x.clamp_(min=0.0)                               # a ReLU output: non-negative, about half exact zeros
            if L == 0:                                      # the tile is the logits: keep the softmax contract's span
                for xm in x.view(n_mu, mb, -1):
                    xm.mul_(LOGIT_SPREAD / float(xm.max()))
    ts = [torch.nn.functional.one_hot(torch.randint(0, local[-1], (rows,), generator=gen), local[-1]).float()
          for _ in range(STEPS)]
    dzs = [torch.randn(rows, local[-1], generator=gen) * DZ_SCALE for _ in range(STEPS)]
    if L > 0:
        Ws, bs = _init_weights(local, xs[0], n_mu, gen, activation=model.activation)
        for i, (W, b) in enumerate(zip(Ws, bs)):
            arena.weight_view(i).copy_(W)
            arena.bias_view(i).copy_(b[None, :])
            if c["stateful"]:
                o, k = arena.blocks[i]
                arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen).cuda() * 1e-3
    _poison(eng, model, local, rows, training, gated=feat)
    if first and training:
        _pitched(eng.dz(0, 0), rows).fill_(NAN)            # the first stage never produces dz[0]
    lrs = LR_STEPS if c["stateful"] else (LR,) * STEPS
    words = me.flags.numel()

    res = {}
    for step in range(STEPS):
        p = f"s{step + 1}."
        e = int(me.epoch[0].item()) + 1
        W0 = [arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(arena.blocks)]
        V0 = [arena.momentum_block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(arena.blocks)] \
            if c["stateful"] else [torch.zeros_like(W) for W in W0]
        W0_flat = arena.weights.detach().clone()
        model.dropout_step = step
        if d is not None:
            # the peers' partials at the scale of this stage's own (the stage's input and received gradient)
            dp_epoch = int(d["me"].epoch[0].item()) + 1
            scale = _stage_grad_scale(local, relu, W0, xs[step], ts[step], None if last else dzs[step], n_mu, batch,
                                      c["loss"])
            P, Wc = dp_peer_data(d, gen, arena.blocks, scale, W0, lrs[step])
        torch.cuda.synchronize()
        # ---- inbound: what the neighbours send; my flags: every poll satisfied, both credits at e - 1
        if not first:
            me.act_in.copy_(_nan_pad(xs[step], ld_in).view(n_mu, mb, ld_in).cuda())
        if not last and training:
            me.dz_in.copy_(_nan_pad(dzs[step], ld_out).view(n_mu, mb, ld_out).cuda())
        mine = own_flags(me.layout, words, n_mu, e)
        me.flags.copy_(mine.cuda())
        # ---- outbound targets: NaN slots, sentinel flags
        for ctx in nb.values():
            ctx.act_in.fill_(NAN)
            ctx.dz_in.fill_(NAN)
            ctx.flags.fill_(SENTINEL)
        if d is not None:
            dp_prefill(d, P, Wc, dp_epoch)
        torch.cuda.synchronize()

        opt.lr = lrs[step]
        w.step_from(sched, xs[step].pin_memory() if first else None, ts[step].pin_memory() if last else None)
        eng.synchronize()
        torch.cuda.synchronize()
        assert int(me.epoch[0].item()) == e
        loss = eng.last_loss() if last and training else None

        act = [xs[step].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
        if not first:
            assert torch.equal(_gather(lambda mu: eng.act(mu, 0), n_mu), act[0]), "act[0] differs from the injected tile"
        dz = [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(L + 1)] if training else None

        # ---- non-vacuity
        for l in range(0 if not first else 1, L + 1):
            if not feat and (l == 0 or relu[l - 1]):
                frac = float((act[l] > 0).double().mean())
                assert 0.05 <= frac <= 0.95, f"step {step + 1}: {frac:.3f} of act[{l}] is positive"
        if training:
            for l in range(0 if not first else 1, L + 1):
                assert float(dz[l].abs().max()) > 0.0, f"step {step + 1}: dz[{l}] is all zero"

        # ---- 1. forward, every layer from the kernel's own input (feature cases: check_residual_layers below)
        for l in range(1, L + 1 if not feat else 1):
            W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
            ref, bound = fwd_oracle(act[l - 1], W, b, relu[l - 1], rtol)
            res[p + f"fwd{l}"] = excess(act[l], ref, bound)

        # ---- 2. loss head, per micro-batch
        if last:
            probs = _gather(eng.probs, n_mu)
            loss_ref = loss_bound = 0.0
            oracle = ce_head_oracle if c["loss"] == "cross_entropy" else head_oracle
            for mu in range(n_mu):
                r = slice(mu * mb, (mu + 1) * mb)
                (pr, bp), (g, bg), (lv, bl) = oracle(act[L][r], ts[step][r], batch, HEAD_RTOL)
                res[p + "probs"] = max(res.get(p + "probs", 0.0), excess(probs[r], pr, bp))
                if training:
                    res[p + "dzL"] = max(res.get(p + "dzL", 0.0), excess(dz[L][r], g, bg))
                loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
            if training:
                res[p + "loss"] = abs(loss - loss_ref) / loss_bound if math.isfinite(loss) else math.inf

        if training:
            # ---- 3. the received gradient, masked in place (a residual last layer keeps it: dz_in stays unmodified)
            if not last and not feat:
                check_received_grad(dz[L].float().view(n_mu, mb, -1), act[L].float().view(n_mu, mb, -1),
                                    dzs[step].view(n_mu, mb, -1), local[-1], f"step {step + 1}: dz[{L}]")
            elif not last:
                assert torch.equal(me.dz_in.cpu()[..., : local[-1]], dzs[step].view(n_mu, mb, -1)), "dz_in was modified"
            if feat:
                # every activated, dropped, residual layer per element, with the masks of the replica's samples
                # (mu * mb + n) * dp + rank at the stage's layer_base; the received gradient as the skip gradient g[L]
                got = check_residual_layers(eng, model, W0_flat, xs[step], n_mu, mb, precision, lrs[step], step=step,
                                            g_in=None if last else dzs[step].view(n_mu, mb, -1),
                                            samples_of=lambda mu: (mu * mb + torch.arange(mb)) * dp + rank)
                res.update({p + k: v for k, v in got.items()})
            # ---- 4. dgrad chain (layer 1 unmasked, and only on non-first stages)
            for l in range(L, 0 if not first else 1, -1):
                if feat:
                    break
                mask = act[l - 1] if l >= 2 else torch.ones_like(act[0])
                ref, bound = dgrad_oracle(dz[l], W0[l - 1][:, :-1], mask, rtol)
                res[p + f"dgrad{l}"] = excess(dz[l - 1], ref, bound)
            if first:
                assert bool(torch.isnan(_pitched(eng.dz(0, 0), rows)).all()), "the first stage wrote dz[0]"
            # ---- 5. the update at this step's learning rate: local, or through the DP kernel with the peers replayed
            own, own_b = [], []
            for i, (o, k) in enumerate(arena.blocks):
                if deferred:
                    g, gb = grad_oracle(dz[i + 1], act[i], rtol_for(precision, rows))
                else:       # one wgrad GEMM per micro-batch accumulating into G: n_mu - 1 more fp32 roundings
                    g, gb = grad_oracle(dz[i + 1], act[i], rtol_for(precision, mb))
                    mag, _ = grad_oracle(dz[i + 1].abs(), act[i].abs(), 0.0)
                    gb = gb + (n_mu - 1) * FP32_ULP * mag
                own.append(g)
                own_b.append(gb)
                if d is not None:
                    continue
                st = c["stateful"]
                Wr, bW, Vr, bV = sgd_oracle(g, gb, W0[i], V0[i], lrs[step], MU if st else 0.0, WD if st else 0.0, st)
                res[p + f"upd{i + 1}"] = excess(arena.block(i)[:, : k + 1].cpu(), Wr, bW)
                if st:
                    res[p + f"mom{i + 1}"] = excess(arena.momentum_block(i)[:, : k + 1].cpu(), Vr, bV)
                assert bool(torch.isnan(arena.block(i)[:, k + 1:]).all()), f"the padding of layer {i + 1}'s weights changed"
            if d is not None:
                dp_check(d, res, step, arena, own, own_b, P, Wc, W0, V0, lrs[step], c["stateful"], dp_epoch)

        # ---- 6. outbound tiles, read from the neighbours' memory
        if "next" in nb:
            check_tiles(nb["next"].act_in.cpu(), act[L].float().view(n_mu, mb, -1), local[-1],
                        f"step {step + 1}: next.act_in")
            assert bool(torch.isnan(nb["next"].dz_in).all()), "a tile landed in the successor's dz_in"
        if "prev" in nb:
            if training:
                check_tiles(nb["prev"].dz_in.cpu(), dz[0].float().view(n_mu, mb, -1), local[0],
                            f"step {step + 1}: prev.dz_in")
            else:
                assert bool(torch.isnan(nb["prev"].dz_in).all()), "inference wrote into the predecessor's dz_in"
            assert bool(torch.isnan(nb["prev"].act_in).all()), "a tile landed in the predecessor's act_in"

        # ---- 7. outbound flags; my own flags untouched
        for side, ctx in nb.items():
            check_flags(ctx.flags.cpu(), neighbour_flags(ctx.layout, words, n_mu, e, side, training),
                        f"step {step + 1}: flags of {side}")
        check_flags(me.flags.cpu(), mine, f"step {step + 1}: my own flags")
    _note(name, res)
    eng.synchronize()
    del eng, w
    gc.collect()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_pp_stage_replay(name, monkeypatch):
    _run(name, monkeypatch)


# ================================================================================================== CPU side
def test_grid_reaches_every_stage_and_transport_branch():
    """The case list reaches every stage position, schedule, transport form, push kernel, micro-batch shape, precision
    and optimizer the pipeline path distinguishes; ``_C.chain_eligible`` confirms which stages run the chain kernel."""
    C = _C()
    seen = {k: set() for k in ("pos", "sched", "form", "push", "mb", "prec", "opt", "loss")}
    stages = set()
    for name, c in CASES.items():
        local = _local(c)
        L, pp, s = len(local) - 1, c["pp"], c["s"]
        first, last, training = s == 0, s == pp - 1, c["sched"] != "inference"
        layers = list(zip(local[:-1], local[1:]))
        eligible = L >= 1 and C.chain_eligible(layers, c["mb"], local[-1], last, c["precision"] == "fp32")
        assert eligible == (c["sizes"] is not WIDE and L >= 1), name
        chain = eligible and "SSB_NO_CHAIN" not in c["env"]
        folded = chain and c["env"].get("SSB_PP_FOLD", "1") != "0"
        stages.add((tuple(c["sizes"]), pp, s))
        seen["pos"].add("first" if first else "last" if last else "middle")
        seen["sched"].add(c["sched"] if training else f"inference-{'first' if first else 'last' if last else 'middle'}")
        seen["form"].add("folded" if folded else "layer-wise" if not chain else "unfolded")
        if chain and training and c["env"].get("SSB_PP_DEFER_WGRAD") == "0":
            seen["form"].add("no-defer")
        if not folded:
            ld_in, ld_out = _lds(local)
            if not last:
                seen["push"].add(("act", c["mb"] * ld_out // 4 > SMALL_TILE_F4))
            if not first and training:
                seen["push"].add(("dz", c["mb"] * ld_in // 4 > SMALL_TILE_F4))
        if folded:
            seen["mb"].add("single-chunk" if c["mb"] <= 32 else "multi-chunk")
        seen["mb"] |= {f"mb{c['mb']}", f"n_mu{c['n_mu']}"} | ({"n_mu>streams"} if c["n_mu"] > 8 else set())
        seen["prec"].add((c["precision"], folded))
        seen["opt"].add(("stateful" if c["stateful"] else "plain", "middle" if not first and not last else "edge"))
        seen["loss"].add(c["loss"])
        if L == 0:
            assert last and pp == 8 and c["sizes"] is REF
        if c["model"]:
            assert c["sizes"] is RES_SIZES and c["dp"] > 1
    assert {(tuple(REF), pp, s) for pp in (2, 4) for s in range(pp)} <= stages
    assert {(tuple(REF), 8, 3), (tuple(REF), 8, 7), (tuple(WIDE), 2, 0), (tuple(WIDE), 2, 1)} <= stages
    assert len(_local(CASES["ref-pp8-s3-1f1b"])) == 2 and len(_local(CASES["ref-pp8-s7-1f1b"])) == 1
    assert [_local(CASES[n])[0] for n in ("ref-pp4-s1-1f1b-mb100", "ref-pp4-s2-gpipe-stateful")] == [127, 125]
    assert seen["pos"] == {"first", "middle", "last"}
    assert seen["sched"] == {"naive", "gpipe", "1f1b", "inference-first", "inference-middle", "inference-last"}
    assert seen["form"] == {"folded", "unfolded", "layer-wise", "no-defer"}
    assert seen["push"] == {(d, multi) for d in ("act", "dz") for multi in (False, True)}
    assert {"single-chunk", "multi-chunk", "mb24", "mb100", "mb128", "n_mu1", "n_mu12", "n_mu>streams"} <= seen["mb"]
    assert {("fp32", True), ("fp32", False), ("tf32", True)} == seen["prec"]
    assert ("stateful", "middle") in seen["opt"]
    assert seen["loss"] == {"mse", "cross_entropy"}


def _dp_path(c):
    """(protocol, DP kernel, launch form) a dp > 1 case must reach, from the shape rules alone: ``_C.chain_eligible``
    for the chain kernel, the LL zone rule and ``flag_geometry`` for the protocol."""
    C = _C()
    local = _local(c)
    L, last = len(local) - 1, c["s"] == c["pp"] - 1
    chain = (L >= 1 and "SSB_NO_CHAIN" not in c["env"]
             and C.chain_eligible(list(zip(local[:-1], local[1:])), c["mb"], local[-1], last, c["precision"] == "fp32"))
    deferred = chain and c["env"].get("SSB_PP_DEFER_WGRAD", "1") != "0" and _ll_on(c, local)
    proto = _dp_protocol(c, local, deferred)
    form = "layer-wise" if not chain else "folded" if c["env"].get("SSB_PP_FOLD", "1") != "0" else "unfolded"
    kernel = "dp_ll" if proto == "ll" else "dp_reduce_sgd" if L else "none"
    return proto, kernel, form


DP_CASES = [n for n, c in CASES.items() if c["dp"] > 1]


def test_dp_grid_reaches_every_position_protocol_and_form():
    """The dp x pp cases reach every stage position, every DP protocol (LL, one-shot, two-shot, each through its kernel),
    dp 2, 4 and 8, every launch form, the per-micro-batch wgrad path, the flag protocol on a stage, momentum, both
    losses, the one-Linear and the Linear-less stage and the residual feature stage, with ranks off zero."""
    seen = {k: set() for k in ("pos", "proto", "kernel", "dp", "form", "misc")}
    for name in DP_CASES:
        c = CASES[name]
        local = _local(c)
        L, first, last = len(local) - 1, c["s"] == 0, c["s"] == c["pp"] - 1
        proto, kernel, form = _dp_path(c)
        assert c["sched"] != "inference" and 0 <= c["rank"] < c["dp"], name
        seen["pos"].add("first" if first else "last" if last else "middle")
        seen["proto"] |= set(proto.split("+")) - {""}
        seen["kernel"].add(kernel)
        seen["dp"].add(c["dp"])
        seen["form"].add(form)
        seen["misc"] |= {f"L={L}" for L in (0, 1) if len(local) - 1 == L}
        seen["misc"] |= {k for k, on in (("stateful", c["stateful"]), ("ce", c["loss"] == "cross_entropy"),
                                         ("res", bool(c["model"])), ("rank>0", c["rank"] > 0),
                                         ("no-defer", c["env"].get("SSB_PP_DEFER_WGRAD") == "0" and form != "layer-wise"),
                                         ("flags-on-chain", proto != "ll" and form != "layer-wise" and L > 0)) if on}
        if proto == "ll":
            assert form != "layer-wise" and kernel == "dp_ll"
        if c["model"]:
            assert form in ("folded", "layer-wise") and not first and not last
    assert seen["pos"] == {"first", "middle", "last"}
    assert seen["proto"] == {"ll", "one-shot", "two-shot"}
    assert seen["kernel"] == {"dp_ll", "dp_reduce_sgd", "none"}
    assert seen["dp"] == {2, 4, 8}
    assert seen["form"] == {"folded", "unfolded", "layer-wise"}
    assert seen["misc"] == {"L=0", "L=1", "stateful", "ce", "res", "rank>0", "no-defer", "flags-on-chain"}
    # every protocol at every position it can run at: LL needs the chain kernel
    pairs = {(("first" if c["s"] == 0 else "last" if c["s"] == c["pp"] - 1 else "middle"), p)
             for c in map(CASES.get, DP_CASES) for p in _dp_path(c)[0].split("+") if p}
    assert {(pos, p) for pos in ("first", "middle", "last") for p in ("ll", "one-shot")} <= pairs, pairs
    assert {("first", "two-shot"), ("middle", "two-shot"), ("last", "two-shot")} <= pairs, pairs


@pytest.mark.parametrize("name", DP_CASES)
def test_dp_prefill_covers_exactly_the_polled_lines_and_flags(name):
    """For the local layers, dp and rank of every dp x pp case: the LL or flag prefill covers exactly what the replica
    polls (test_gpu_dp_replay's checks on the stage's geometry)."""
    from test_gpu_dp_replay import check_flag_prefill, check_ll_prefill

    c = CASES[name]
    local = _local(c)
    proto, _kernel, _form = _dp_path(c)
    if proto == "ll":
        check_ll_prefill(local, c["dp"], c["rank"])
    else:
        check_flag_prefill(local, c["dp"], c["rank"], dict(two_shot="SSB_DP_TWO_SHOT" in c["env"],
                                                          one_shot="SSB_DP_ONE_SHOT" in c["env"]))


def _emulated_stage(seed=0):
    """A correct middle stage of n_mu = 3 micro-batches after step e, emulated on the CPU: its outbound tiles in the
    neighbours' slots, its masked received gradient and every flag array, on a made-up flag layout (the checks take the
    layout from ``PpContext.buffers()`` on the GPU)."""
    g = torch.Generator().manual_seed(seed)
    n_mu, mb, cols, ld, e, words = 3, 5, 7, 8, 6, 48
    layout = {"act_arrived": (0, 16), "dz_arrived": (16, 16), "act_credit": (32, 1), "dz_credit": (40, 1)}
    act_L = torch.randn(n_mu, mb, cols, generator=g).clamp_min(0.0)
    dz_0 = torch.randn(n_mu, mb, cols, generator=g)
    injected = torch.randn(n_mu, mb, cols, generator=g)
    dz_L = torch.where(act_L > 0, injected, torch.zeros(()))
    nxt = torch.full((n_mu, mb, ld), NAN)
    nxt[..., :cols] = act_L
    prv = torch.full((n_mu, mb, ld), NAN)
    prv[..., :cols] = dz_0
    flags = {side: neighbour_flags(layout, words, n_mu, e, side, True) for side in ("prev", "next")}
    mine = own_flags(layout, words, n_mu, e)
    return dict(n_mu=n_mu, cols=cols, e=e, words=words, layout=layout, act_L=act_L, dz_0=dz_0, injected=injected,
                dz_L=dz_L, next=nxt, prev=prv, flags=flags, mine=mine, mine_after=mine.clone())


def _check_emulated(t):
    check_tiles(t["next"], t["act_L"], t["cols"], "next.act_in")
    check_tiles(t["prev"], t["dz_0"], t["cols"], "prev.dz_in")
    check_received_grad(t["dz_L"], t["act_L"], t["injected"], t["cols"], "dz[L]")
    for side in ("prev", "next"):
        check_flags(t["flags"][side], neighbour_flags(t["layout"], t["words"], t["n_mu"], t["e"], side, True), side)
    check_flags(t["mine_after"], t["mine"], "mine")


def test_checks_reject_injected_faults():
    """The message checks accept an emulated correct stage and reject each plausible transport fault."""
    _check_emulated(_emulated_stage())

    def slot_of_next_mu(t):              # the outbound slot mu holds micro-batch mu + 1
        t["next"][0] = t["next"][1]

    def shifted_row(t):                  # one tile stored one row down
        t["prev"][1, 1:] = t["prev"][1, :-1].clone()

    def flipped_mask(t):                 # one mask element of the received gradient flipped
        i = (t["act_L"] == 0).nonzero()[0].tolist()
        t["dz_L"][tuple(i)] = t["injected"][tuple(i)]

    def kept_mask(t):                    # a positive activation's gradient dropped
        i = (t["act_L"] > 0).nonzero()[0].tolist()
        t["dz_L"][tuple(i)] = 0.0

    def flag_at_sentinel(t):             # one arrival flag never raised
        t["flags"]["next"][t["layout"]["act_arrived"][0] + 2] = SENTINEL

    def flag_stale(t):                   # one arrival flag raised with the previous epoch
        t["flags"]["prev"][t["layout"]["dz_arrived"][0] + 1] = t["e"] - 1

    def credit_wrong_neighbour(t):       # the act credit stored into the successor instead of the predecessor
        t["flags"]["prev"][t["layout"]["act_credit"][0]] = SENTINEL
        t["flags"]["next"][t["layout"]["act_credit"][0]] = t["e"]

    def credit_wrong_word(t):            # the dz credit stored into the successor's act credit word
        t["flags"]["next"][t["layout"]["dz_credit"][0]] = SENTINEL
        t["flags"]["next"][t["layout"]["act_credit"][0]] = t["e"]

    def own_flag_written(t):             # the stage wrote its own credit
        t["mine_after"][t["layout"]["act_credit"][0]] = t["e"]

    def stray_flag(t):                   # an arrival flag raised for a micro-batch that does not exist
        t["flags"]["next"][t["layout"]["act_arrived"][0] + t["n_mu"]] = t["e"]

    for fault in (slot_of_next_mu, shifted_row, flipped_mask, kept_mask, flag_at_sentinel, flag_stale,
                  credit_wrong_neighbour, credit_wrong_word, own_flag_written, stray_flag):
        t = _emulated_stage()
        fault(t)
        with pytest.raises(AssertionError):
            _check_emulated(t)


def _emulated_dpxpp_stage(fault=None):
    """Replica 1 of dp = 4 of stage 1 of a pp = 4 model with residual GELU layers and dropout, one step emulated on the
    CPU (fp64, stored in fp32) with its peer's partials, its LL update, its flags and, for the loss scale, a last stage's
    head.  ``fault`` injects one plausible dp x pp fault; the result is what the GPU test reads back from the engine."""
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.ops import functional as F
    from test_gpu_chain import act_ref

    sizes, pp, st, dp, rank, n_mu, mb, lr, step, e = [20, 48, 48, 48, 48, 48, 48, 4], 4, 1, 4, 1, 2, 3, 0.5, 4, 6
    rows = n_mu * mb
    model = MLP(sizes, st, pp, rows * dp, **FEATURES)
    L = len(model.linears)
    g = torch.Generator().manual_seed(1)
    arena = model.arena
    blocks = [torch.randn(o, k + 1, generator=g, dtype=torch.float64).float().double() * 0.3 for o, k in arena.blocks]
    W0 = torch.zeros(arena.numel)
    for i, (o, k) in enumerate(arena.blocks):
        W0[arena.offsets[i]: arena.offsets[i] + o * arena.lds[i]].view(o, -1)[:, : k + 1] = blocks[i].float()
    x = torch.randn(rows, 48, generator=g).clamp_min(0.0)          # act_in
    x_stage = torch.randn(rows, 48, generator=g)                    # what the staging buffer holds
    g_in = torch.randn(rows, 48, generator=g) * 1e-2                # dz_in
    s = F.dropout_scale(FEATURES["dropout"])
    src_rank = 0 if fault == "rank0-masks" else rank
    base = 1 if fault == "layer-base" else 0
    acts, gates = [x.double()], [None]
    for l, lin in enumerate(model.linears, start=1):
        z = acts[-1] @ blocks[l - 1][:, :-1].T + blocks[l - 1][:, -1]
        keep = torch.cat([F.dropout_mask(FEATURES["dropout"], FEATURES["dropout_seed"], lin.dropout[2] + base, step,
                                         (mu * mb + torch.arange(mb)) * dp + src_rank, lin.out_dims) for mu in range(n_mu)])
        f, f1, _ = act_ref("gelu", z)
        acts.append((acts[-1] + torch.where(keep, f * s, 0.0)).float().double())
        gates.append(torch.where(keep, f1 * s, 0.0).float())           # a dropped gate is +0
    dz = [None] * (L + 1)
    dz[L] = g_in if fault == "dz-is-dz_in" else g_in * gates[L]      # fp32 multiply, out of place
    gl = g_in.double()
    for l in range(L, 0, -1):
        pre = dz[l].double() @ blocks[l - 1][:, :-1] + gl
        dz[l - 1] = (pre * gates[l - 1].double()).float() if l > 1 else pre.float()
        gl = pre
    # the update: own partial [dz.T @ act | colsum] + the peers', plain SGD on the rows this replica owns (LL: rows
    # 32 .. 63 of every 128-row tile)
    P = {p: [torch.randn(o, k + 1, generator=g) * 1e-2 for o, k in arena.blocks] for p in range(dp) if p != rank}
    own, own_b, W1 = [], [], []
    for i, (o, k) in enumerate(arena.blocks):
        a_used = x_stage if fault == "staging-x" and i == 0 else acts[i]
        dz_used = g_in if fault == "unmasked-dz" and i == L - 1 else dz[i + 1]
        gr, gb = grad_oracle(dz[i + 1], acts[i], RTOL["fp32"])
        used = torch.cat([dz_used.double().T @ a_used.double(), dz_used.double().sum(0)[:, None]], 1)
        tot = used + sum(P[p][i].double() for p in P if not (fault == "dropped-peer" and p == 3))
        own.append(gr)
        own_b.append(gb)
        W1.append((blocks[i] - lr * tot).float())
    owned = [(torch.arange(o)[:, None] % 128 // (128 // dp) == rank).expand(o, k + 1) for o, k in arena.blocks]
    # a last stage's loss head: dz of the logits scaled by 1 / (mb * n_mu * dp)
    logits = torch.randn(mb, 4, generator=g, dtype=torch.float64) * 5
    t = torch.nn.functional.one_hot(torch.randint(0, 4, (mb,), generator=g), 4).double()
    dz_head = head_oracle(logits, t, rows * (1 if fault == "loss-scale" else dp), 0.0)[1][0].float()
    # flags: one credit per neighbour, my arrival flags into the successor's act_arrived
    layout = {"act_arrived": (0, 16), "dz_arrived": (16, 16), "act_credit": (32, 1), "dz_credit": (40, 1)}
    flags = {side: neighbour_flags(layout, 48, n_mu, e, side, True) for side in ("prev", "next")}
    if fault == "no-credit":
        flags["prev"][layout["act_credit"][0]] = SENTINEL

    class Eng:
        def act(self, mu, l):
            return acts[l][mu * mb:(mu + 1) * mb].float()

        def dz(self, mu, l):
            return dz[l][mu * mb:(mu + 1) * mb]

        def gate(self, mu, l):
            return gates[l][mu * mb:(mu + 1) * mb]

        def g(self, mu, l):
            assert l == L
            return g_in[mu * mb:(mu + 1) * mb]

        def uses_chain(self):
            return True

    return dict(eng=Eng(), model=model, W0=W0, x=x, g_in=g_in, n_mu=n_mu, mb=mb, dp=dp, rank=rank, step=step, lr=lr,
                blocks=blocks, own=own, own_b=own_b, P=P, W1=W1, owned=owned, logits=logits, t=t, dz_head=dz_head,
                batch=rows * dp, layout=layout, flags=flags, e=e)


def _check_emulated_dpxpp(t):
    """The GPU test's checks of a dp x pp stage, applied to an emulated one."""
    from test_gpu_dp_replay import check_owned_update

    n_mu, mb, dp, rank = t["n_mu"], t["mb"], t["dp"], t["rank"]
    check_residual_layers(t["eng"], t["model"], t["W0"], t["x"], n_mu, mb, "fp32", t["lr"], step=t["step"],
                          g_in=t["g_in"].view(n_mu, mb, -1), samples_of=lambda mu: (mu * mb + torch.arange(mb)) * dp + rank)
    res = {}
    for i, blk in enumerate(t["blocks"]):
        assert bool(t["owned"][i].any())
        check_owned_update(t["W1"][i], t["own"][i], t["own_b"][i], [t["P"][p][i] for p in t["P"]], blk, None, None,
                           t["lr"], False, t["owned"][i], res, "%s" + str(i + 1))
    (_, _), (g, bg), _ = head_oracle(t["logits"], t["t"], t["batch"], HEAD_RTOL)
    res["dzL"] = excess(t["dz_head"], g, bg)
    assert all(v <= 1.0 for v in res.values()), res
    for side in ("prev", "next"):
        check_flags(t["flags"][side], neighbour_flags(t["layout"], 48, n_mu, t["e"], side, True), side)


def test_dpxpp_checks_reject_injected_faults():
    """The checks of a dp x pp stage accept an emulated correct stage and reject each fault of the composition: the own
    partial from the staging buffer instead of act_in, the LL wave reading the received gradient unmasked, dz[L] of a
    residual last layer replaced by dz_in, a loss scale without the dp factor, rank 0's dropout masks on rank 1, the
    stage's layer_base off by one, a peer partial dropped, and a pipeline credit not returned."""
    _check_emulated_dpxpp(_emulated_dpxpp_stage())
    for fault in ("staging-x", "unmasked-dz", "dz-is-dz_in", "loss-scale", "rank0-masks", "layer-base", "dropped-peer",
                  "no-credit"):
        with pytest.raises(AssertionError):
            _check_emulated_dpxpp(_emulated_dpxpp_stage(fault))


def test_plan_check_counts_pushes_and_waits_per_micro_batch():
    """``check_plan`` on hand-written plans: a correct unfolded middle stage passes; a missing push of one micro-batch,
    a push of the wrong micro-batch, a folded plan with a wait, and a second credit are rejected."""
    def plan(ops):
        return "".join(f"{i} {op}\n" for i, op in enumerate(ops))

    ok = ["pp_bump_epoch stream=0", "record_event stream=0 event=0"]
    ok += [f"pp_wait stream=1 mu={mu}" for mu in range(2)] + [f"pp_push stream=1 mu={mu}" for mu in range(2)]
    ok += [f"pp_wait stream=1 mu={mu}" for mu in range(2)] + [f"pp_push stream=1 mu={mu}" for mu in range(2)]
    ok += ["wgrad_group stream=10", "pp_credit stream=0"]
    check_plan(plan(ok), 2, False, True, False, False, True)
    bad = [ok[:5] + ok[6:], [o.replace("mu=1", "mu=0") if o.startswith("pp_push") else o for o in ok], ok + ok[-1:]]
    for b in bad:
        with pytest.raises(AssertionError):
            check_plan(plan(b), 2, False, True, False, False, True)
    with pytest.raises(AssertionError):
        check_plan(plan(ok), 2, True, True, False, False, True)
    with pytest.raises(AssertionError):
        check_plan(plan(ok), 2, False, False, False, False, True)
