"""The one-GPU engine (pp = 1, dp = 1) per element against fp64 at EVERY step of a six-step run, in both input-staging
sets, at up to 128 micro-batches, in fp32, tf32 and bf16, with and without residual layers, the EMA of the weights,
learning-rate schedules and shuffled epochs.

``PipeEngine`` plans two complete steps, one per staging set, each captured into a graph of its own with its own
device state (the x / y staging buffers, the learning-rate slot, the dropout-step slot, the EMA-alpha slot, the pinned
loss slot), and ``run()`` alternates them while the momentum and the EMA carry over.  The micro-batch index reaches the
row offsets of every buffer, the chain kernel's ``mu_base``, the dropout rows, the loss slot (stride
``max(n_mu, 16)``), the targets and the stream map (at most 8 micro-batch streams, so past 8 micro-batches several
share one).  Every step of every case below is checked by ``check_step`` from the engine's own buffers, with the
oracles of ``test_gpu_chain.py``, ``test_gpu_gemm.py``, ``test_gpu_cross_entropy.py``, ``test_gpu_bf16.py`` and
``test_gpu_residual.py``, so errors cannot cascade from step to step:

* staging: set i % 2 holds step i's x and targets bitwise and NaN in its padding, the other set step i - 1's inputs,
  and ``fill_set()`` alternates; a shuffled case runs as train.py runs it (``NativeWorker.execute`` on a
  device-resident ``Dataset(shuffle_seed=...)``, ``set_epoch`` at each epoch's first batch, two epochs of three
  batches), and its sets hold the rows ``shuffle_index`` picks for the step's epoch and batch;
* every layer of every micro-batch (``check_layers``: forward, gates, dropped elements +0, dgrad; residual models
  ``check_residual_layers``: the skip added unrounded, g_l, and the nil features, where the skip and g_l stand alone
  and are bounded by one rounding) with the masks of the step's dropout step; in bf16 every product from the
  bf16-rounded operands (``test_gpu_bf16.bf``, ``RTOL_BF16``); the loss head (probabilities, dz_L, and the step's
  loss against the sum over micro-batches);
* the update at the step's own rate (hand-picked rates, or the rate ``LRSchedule`` gives the step, which train.py
  hands the optimizer before it; 0.0 leaves W bitwise unchanged and V still advances), plain or stateful, deferred /
  coalesced or accumulated per micro-batch through memory; the momentum per element; NaN still in the weights'
  padding;
* the EMA: every real entry, bias column included, is ``ema_lerp_ref(E0, W1, alpha)`` bit for bit, with the alpha of
  the optimizer's update count at that step; its padding is untouched where the update is fused into a wgrad epilogue
  (the grouped wgrad of the chain forms, the per-layer epilogue of the layer-wise forms) and follows the weights'
  padding under the flat pass (``layerwise-per-mb``); and the weights and momentum of every step equal, bit for bit,
  those of the same case run without EMA;
* non-vacuity at every step: 5-95 % of every hidden activation positive (of a residual layer's branch), every dz
  non-zero, live units dropped under dropout, |z| > 9 reached under a smooth activation, the skip and g_l checked at
  a nil feature of every residual layer, the EMA away from the weights, the rate changing across the warm-up steps.

An EMA case starts from an EMA away from the weights and from a resumed update count, so step 0 already runs with
alpha < 1.  The engine takes whatever alpha its caller hands it per step; the cases change the decay every step
(EMA_DECAYS), so that the alpha slot of either staging set is rewritten at every step and both branches of the lerp
(alpha >= 0.5 and alpha < 0.5) run in one run.

The device-timed and the pipelined steps of ``bench.py`` never synchronise with the host; for a subset of cases the
same run is replayed through ``Trainer.step_async`` (device-resident inputs) and ``Trainer.step_pipelined`` (pinned host
memory, lagged losses), and once more with the plan walked eagerly instead of replayed from its CUDA graphs, each with
``Trainer.lr_schedule`` driving the rate; each must reproduce the checked run's weights, momentum, EMA and losses bit
for bit (the kernels sum in a fixed order), while the rate, the dropout step and the alpha change at every step.  The
evaluation engine of ``train.py`` (a second ``NativeWorker`` sharing the first, ordered behind it by
``NativeWorker._enter``) runs between two training steps without a host sync; its forward, probabilities and
``count_correct`` are checked against the weights of the step before it.  With an EMA, train.py's EMA evaluation runs
there as well: ``ema_state()`` copied into a second model's arena and run by that model's own inference worker, checked
against the EMA of that step (a residual model in its inference form: skips added, no gates).

The CPU tests check that the grid reaches every branch named above and that the checks reject a set of injected faults
in a six-step fp32 emulation of the engine (residual layers, momentum, the EMA, a schedule, shuffled epochs) while
they accept the clean emulation.

Worst err / bound over all six steps, measured on an H100 80GB HBM3 (700 W power limit), as fp32 / tf32 / bf16:

    chain with a cluster     0.57 / 0.95 / 0.58     residual      bf16 0.50
    chain on one CTA         0.43 / 0.71 / 0.42     residual fp32 0.85
    chain per micro-batch    0.50 / 0.89 / 0.49     residual      bf16 0.83
    layer-wise               0.50 / 0.97 / 0.50     residual tf32 0.95
    layer-wise per micro-b.  0.57 / 0.93 / 0.58     residual fp32 0.50
    split-K                  0.59 /  -   / 0.50     residual fp32 0.59

the interleaved evaluations 0.24 at most (the EMA of the bf16 residual model).  The residual worst values are g_l at a
nil feature (gskip) or the update.  Every case stays non-degenerate at these rates, the eager replays are bitwise the
graph runs, and the file takes 100 to 130 s there.
"""
import math
import re

import pytest
import torch

from shallowspeed_b200.lr_schedule import LRSchedule
from shallowspeed_b200.ops.functional import ema_alpha, ema_lerp_ref, shuffle_index
from test_gpu_bf16 import bf, grad_oracle_bf16, rtol_bf16
from test_gpu_chain import (ATOL, DROP_P, DROP_SEED, HEAD_RTOL, RTOL, U, _gather, _init_weights, _pitched, _poison,
                            check_layers, excess, head_oracle, rows_update_oracle)
from test_gpu_cross_entropy import ce_head_oracle
from test_gpu_gemm import FP32_ULP, MU, WD, WIDE, _gen, grad_oracle, rtol_for, sgd_oracle
from test_gpu_residual import (NIL_COL, NIL_ROW, _branch_nonvacuous, _init_res_weights, _residual_flags,
                               check_residual_layers)

REF = [784, 128, 127, 126, 125, 124, 123, 10]    # the reference model, the benchmark's flagship
ONE_CTA = [784, 32, 24, 10]                        # every layer at most 32 wide: one CTA per micro-batch
SPLITK = WIDE["1000-1500-777"]                     # layer-wise GEMMs with split-K forward and dgrad
RES_REF = [784, 128, 128, 128, 128, 10]            # the reference's widths made equal: C = 4, k-split layer 1 feeding
RES_ONE_CTA = [784, 32, 32, 32, 10]                # residual layers 2..4 (2..3 on one CTA)
RES_SPLITK = [1000, 1500, 1500, 10]                # a wide residual layer 2 with split-K forward and dgrad
BUILD_LR = 0.5
# the rate of each step, all exact in fp32.  Step 3 (set 1) needs no slot write: its set still holds 0.25 from step 1,
# while set 0 went to 0.375 in between.  Step 4 runs at 0.
LRS = (0.25, 0.25, 0.375, 0.25, 0.0, 0.375)
STEPS = len(LRS)
# each kind with a warm-up whose rate changes at every step; cosine and linear reach min_lr = 0 within the run, the
# constant one holds its base from step 2 on, so that step 4's set needs no slot write
SCHEDULES = {
    "cosine": LRSchedule(0.375, "cosine", total_steps=5, warmup_steps=2, warmup_start_factor=0.5),
    "linear": LRSchedule(0.375, "linear", total_steps=4, warmup_steps=1, warmup_start_factor=0.25),
    "step": LRSchedule(0.5, "step", warmup_steps=3, warmup_start_factor=0.25, step_size=1, gamma=0.5),
    "constant": LRSchedule(0.375, "constant", warmup_steps=2, warmup_start_factor=0.5),
}
EMA_DECAYS = (0.75, 0.3, 0.9, 0.5, 0.6, 0.2)      # alpha 0.25, 0.7, 0.1, 0.5, 0.4, 0.8: both branches of the lerp
EMA_RESUMED = 7                                    # the EMA update count an EMA case starts from
EMA_PAD = 7.0                                      # the EMA's padding: kept by a fused site, lerped by the flat pass
EPOCH_BATCHES = 3                                  # a shuffled case: two epochs of three batches
SHUFFLE_SEED, SHUFFLE_SPARE = 0x5F0_FF1E, 5        # SHUFFLE_SPARE rows past the last batch: dropped, another set each epoch
EVAL_AFTER = 2                                     # the interleaved evaluation runs between steps 2 and 3
V_SCALE = 1e-3                                     # the momentum a stateful case starts from

NO_CHAIN, NO_COALESCE = "SSB_NO_CHAIN", "SSB_NO_COALESCE"
FORMS = {                                          # form -> environment that selects it
    "chain-cluster": (), "chain-one-cta": (), "chain-per-mb": (NO_COALESCE,), "layerwise": (NO_CHAIN,),
    "layerwise-per-mb": (NO_CHAIN, NO_COALESCE), "splitk": (),
}


def _case(sizes, form, n_mu, mb, sched="naive", precision="fp32", loss="mse", activation="relu", dropout=0.0,
          drop_start=0, stateful=False, residual=False, ema=False, lr_schedule=None, shuffle=False, graph=True,
          replay=False, eval_mu=None):
    """``ema``: keep an EMA at the per-step decays EMA_DECAYS, from EMA_RESUMED updates; ``lr_schedule``: a SCHEDULES
    name (None: the rates LRS); ``shuffle``: stage shuffled epochs through ``NativeWorker.execute``; ``replay``: also
    run the unsynchronised replays; ``eval_mu``: also run the interleaved evaluation with this many micro-batches
    (None: not at all)."""
    return dict(sizes=sizes, form=form, n_mu=n_mu, mb=mb, sched=sched, precision=precision, loss=loss,
                activation=activation, dropout=dropout, drop_start=drop_start, stateful=stateful, residual=residual,
                ema_decay=EMA_DECAYS if ema else None, lr_schedule=lr_schedule, shuffle=shuffle, graph=graph,
                replay=replay, eval_mu=eval_mu)


GELU_DROP = dict(activation="gelu", dropout=DROP_P)
CASES = {
    # chain kernel, all micro-batches in one launch, 4 CTAs per micro-batch and a k-split first layer
    "chain-ref-3x24-tf32-ce": _case(REF, "chain-cluster", 3, 24, precision="tf32", loss="cross_entropy"),
    "chain-ref-4x32": _case(REF, "chain-cluster", 4, 32, replay=True, eval_mu=1),
    "chain-ref-9x8-gelu-drop-resumed": _case(REF, "chain-cluster", 9, 8, drop_start=1000, **GELU_DROP),
    "chain-ref-17x8-stateful": _case(REF, "chain-cluster", 17, 8, stateful=True, replay=True),
    "chain-ref-32x4-tf32-eager": _case(REF, "chain-cluster", 32, 4, precision="tf32", graph=False),
    "chain-ref-128x1": _case(REF, "chain-cluster", 128, 1),
    "chain-ref-4x32-ema-linear-drop": _case(REF, "chain-cluster", 4, 32, dropout=DROP_P, ema=True, lr_schedule="linear",
                                            replay=True, eval_mu=4),
    "chain-ref-9x8-bf16-stateful": _case(REF, "chain-cluster", 9, 8, precision="bf16", stateful=True),
    "res-chain-4x32-bf16-ema-cosine": _case(RES_REF, "chain-cluster", 4, 32, precision="bf16", residual=True, ema=True,
                                            lr_schedule="cosine", replay=True, eval_mu=2),
    # chain kernel, one CTA per micro-batch
    "chain-one-4x32-tf32": _case(ONE_CTA, "chain-one-cta", 4, 32, precision="tf32"),
    "chain-one-17x8-stateful": _case(ONE_CTA, "chain-one-cta", 17, 8, stateful=True),
    "chain-one-4x32-bf16-ema": _case(ONE_CTA, "chain-one-cta", 4, 32, precision="bf16", ema=True),
    "res-chain-one-17x8-silu-stateful-ema-linear": _case(RES_ONE_CTA, "chain-one-cta", 17, 8, activation="silu",
                                                         stateful=True, residual=True, ema=True, lr_schedule="linear"),
    # chain kernel, one launch per micro-batch, the weight gradients in one deferred wave
    "chain-per-mb-9x8-naive": _case(REF, "chain-per-mb", 9, 8, replay=True, eval_mu=9),
    "chain-per-mb-9x8-gpipe-gelu-drop": _case(REF, "chain-per-mb", 9, 8, sched="gpipe", **GELU_DROP),
    "chain-per-mb-9x8-pipedream-stateful-tf32": _case(REF, "chain-per-mb", 9, 8, sched="pipedream", stateful=True,
                                                     precision="tf32"),
    "chain-per-mb-17x8-gpipe": _case(REF, "chain-per-mb", 17, 8, sched="gpipe"),
    "chain-per-mb-9x8-bf16-ema-shuffled": _case(REF, "chain-per-mb", 9, 8, precision="bf16", ema=True, shuffle=True),
    "res-chain-per-mb-9x8-bf16-tanh-ce-stateful-ema": _case(RES_REF, "chain-per-mb", 9, 8, sched="gpipe",
                                                            precision="bf16", loss="cross_entropy", activation="tanh",
                                                            stateful=True, residual=True, ema=True),
    # layer-wise GEMMs over all micro-batches, SGD fused into the weight-gradient epilogue
    "layerwise-4x32": _case(REF, "layerwise", 4, 32, replay=True, eval_mu=1),
    "layerwise-17x8-gelu-drop-stateful-tf32": _case(REF, "layerwise", 17, 8, stateful=True, precision="tf32",
                                                    **GELU_DROP),
    "layerwise-4x32-bf16-ema": _case(REF, "layerwise", 4, 32, precision="bf16", ema=True),
    "res-layerwise-4x32-tf32-gelu-drop-resumed-stateful-step": _case(RES_REF, "layerwise", 4, 32, precision="tf32",
                                                                     drop_start=500, stateful=True, residual=True,
                                                                     lr_schedule="step", **GELU_DROP),
    # layer-wise GEMMs per micro-batch: weight gradients accumulate through memory, then a separate SGD pass
    "layerwise-per-mb-9x8-tf32-ce-eager": _case(REF, "layerwise-per-mb", 9, 8, precision="tf32", loss="cross_entropy",
                                                graph=False),
    "layerwise-per-mb-17x8-stateful": _case(REF, "layerwise-per-mb", 17, 8, sched="gpipe", stateful=True, replay=True),
    "layerwise-per-mb-9x8-bf16-stateful-ema": _case(REF, "layerwise-per-mb", 9, 8, precision="bf16", stateful=True,
                                                    ema=True),
    "res-layerwise-per-mb-9x8-ema-constant-shuffled": _case(RES_REF, "layerwise-per-mb", 9, 8, residual=True, ema=True,
                                                            lr_schedule="constant", shuffle=True),
    # wide layers: split-K forward and dgrad GEMMs
    "splitk-3x32-stateful": _case(SPLITK, "splitk", 3, 32, stateful=True),
    "splitk-3x32-bf16-ema": _case(SPLITK, "splitk", 3, 32, precision="bf16", ema=True),
    "res-splitk-2x32-stateful-ema": _case(RES_SPLITK, "splitk", 2, 32, stateful=True, residual=True, ema=True),
}
REPLAYS = [n for n, c in CASES.items() if c["replay"]]
EVALS = [n for n, c in CASES.items() if c["eval_mu"] is not None]
WORST = {}                    # (form, precision, "residual" or "") -> (worst err / bound, where)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for (form, precision, res), (v, what) in sorted(WORST.items()):
        print(f"[steps] worst err/bound {form:>16} {precision} {res:>8}: {v:.3g} ({what})")


def _bits(t):
    return t.detach().float().contiguous().cpu().view(torch.int32)


def _bit_equal(a, b):
    return torch.equal(_bits(a), _bits(b))


def _same(a, b):
    """Bitwise equal, NaN where the other is NaN."""
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def _blocks(model, flat):
    """The [out, in + 1] blocks (W | bias) of a flat weight arena, in fp64 on the CPU."""
    out = []
    for i, (o, k) in enumerate(model.arena.blocks):
        off, ld = model.arena.offsets[i], model.arena.lds[i]
        out.append(flat[off:off + o * ld].view(o, ld)[:, : k + 1].double().cpu())
    return out


def _real(arena):
    """Bool mask over the arena's ``numel`` entries: the weights and bias columns, not the padding."""
    m = torch.zeros(arena.numel, dtype=torch.bool, device=arena.weights.device)
    for i, (o, k) in enumerate(arena.blocks):
        m[arena.offsets[i]: arena.offsets[i] + o * arena.lds[i]].view(o, arena.lds[i])[:, : k + 1] = True
    return m


def _head(loss):
    return ce_head_oracle if loss == "cross_entropy" else head_oracle


def _rate(c, i):
    """The rate of step ``i``: its schedule's, an fp32 value, or the hand-picked LRS[i]."""
    return SCHEDULES[c["lr_schedule"]](i) if c["lr_schedule"] else LRS[i]


def _alpha(c, i):
    """The EMA alpha of step ``i`` (None without an EMA): update EMA_RESUMED + i at that step's decay."""
    return ema_alpha(c["ema_decay"][i], EMA_RESUMED + i) if c["ema_decay"] else None


# ================================================================================================== the per-step checks
def check_step(eng, model, c, st):
    """Every check of one step that just ran, from ``eng``'s buffers.  ``st``: the step's index ``i``, inputs ``x`` /
    ``t`` and those of the step before (``x_prev`` / ``t_prev``, None at step 0), ``lr``, dropout step ``dstep``, the
    flat weights ``W0`` and momentum ``V0`` (None: plain rule) before it, the loss the engine reported and the staging
    set ``fill`` it was filled into; with an EMA the flat EMA ``E0`` before the step and the step's ``alpha``; with a
    run of the same case without EMA next to it, its weights ``W_plain`` and momentum ``V_plain`` after the step.
    Returns {check: max err / bound}."""
    n_mu, mb, precision, i = c["n_mu"], c["mb"], c["precision"], st["i"]
    rows, L = n_mu * mb, len(model.linears)
    in_dim, out_dim = model.linears[0].in_dims, model.linears[-1].out_dims
    what = f"step {i}"

    # ---- staging: this step's set holds its inputs, the other set the previous step's, and the sets alternate
    assert st["fill"] == i % 2 and eng.fill_set() == (i + 1) % 2, (what, st["fill"], eng.fill_set())
    for s, (x, t) in ((i % 2, (st["x"], st["t"])), ((i + 1) % 2, (st["x_prev"], st["t_prev"]))):
        xs, ys = (v.cpu() for v in eng.staging(s))
        for buf, want, cols in ((xs, x, in_dim), (ys, t, out_dim)):
            got = buf[:, :cols]
            ok = _bit_equal(got, want) if want is not None else int(torch.count_nonzero(got)) == 0
            assert ok, f"{what}: staging set {s} does not hold the inputs of step {i if s == i % 2 else i - 1}"
            assert bool(buf[:, cols:].isnan().all()), f"{what}: the padding of staging set {s} changed"

    # ---- every layer of every micro-batch: forward, gates, dropped elements, dgrad (and the skips of a residual model)
    samples_of = lambda mu: mu * mb + torch.arange(mb)                                        # noqa: E731
    if c["residual"]:
        res = check_residual_layers(eng, model, st["W0"], st["x"], n_mu, mb, precision, st["lr"], step=st["dstep"],
                                    samples_of=samples_of, check_update=False)
    else:
        res = check_layers(eng, model, st["W0"], st["x"], n_mu, mb, precision, st["lr"], samples_of, step=st["dstep"],
                           check_update=False)
    act = [st["x"].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
    dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
    blocks = _blocks(model, st["W0"])

    # ---- non-vacuity
    if c["residual"]:
        _branch_nonvacuous(model, blocks, act, model.activation, model.dropout)
        for l, lin in enumerate(model.linears, start=1):
            if lin.residual:       # the nil features: the skip alone in the forward, g_l alone in the dgrad
                assert f"skip{l}" in res and (l == 1 or f"gskip{l}" in res), (what, l, sorted(res))
    else:
        for l in range(1, L):
            frac = float((act[l] > 0).double().mean())
            assert 0.05 <= frac <= 0.95, f"{what} layer {l}: {frac:.3f} of the activations are positive"
            if model.activation != "relu":
                z = act[l - 1] @ blocks[l - 1][:, :-1].T + blocks[l - 1][:, -1]
                assert bool((z.abs() > 9).any()), f"{what} layer {l}: no pre-activation beyond |z| = 9"
    for l in range(1, L + 1):
        assert float(dz[l].abs().max()) > 0.0, f"{what}: dz[{l}] is all zero"

    # ---- loss head, per micro-batch; the engine sums the micro-batch losses in fp32
    probs = _gather(eng.probs, n_mu)
    t = st["t"]
    loss_ref = loss_bound = 0.0
    for mu in range(n_mu):
        r = slice(mu * mb, (mu + 1) * mb)
        (p, bp), (g, bg), (lv, bl) = _head(c["loss"])(act[L][r], t[r], rows, HEAD_RTOL)
        res["probs"] = max(res.get("probs", 0.0), excess(probs[r], p, bp))
        res["dzL"] = max(res.get("dzL", 0.0), excess(dz[L][r], g, bg))
        loss_ref, loss_bound = loss_ref + lv, loss_bound + bl + n_mu * U * abs(lv)
    res["loss"] = abs(st["loss"] - loss_ref) / loss_bound if math.isfinite(st["loss"]) else math.inf

    # ---- the update at this step's rate; in bf16 the gradient from the rounded operands
    lr, stateful = st["lr"], st["V0"] is not None
    per_mb_wgrad = c["form"] == "layerwise-per-mb"
    if precision == "bf16":
        g_oracle, g_rtol = grad_oracle_bf16, rtol_bf16
    else:
        g_oracle, g_rtol = grad_oracle, (lambda k: rtol_for(precision, k))
    W1 = model.arena.weights.detach()
    V1 = model.arena.momentum.detach() if stateful else None
    blocks1 = _blocks(model, W1)
    vblocks0 = _blocks(model, st["V0"]) if stateful else None
    vblocks1 = _blocks(model, V1) if stateful else None
    for l in range(1, L + 1):
        if stateful or per_mb_wgrad or precision == "bf16":
            if per_mb_wgrad:       # one wgrad GEMM per micro-batch accumulating into G: n_mu - 1 more fp32 roundings
                g, gb = g_oracle(dz[l], act[l - 1], g_rtol(mb))
                mag, _ = g_oracle(dz[l].abs(), act[l - 1].abs(), 0.0)
                gb = gb + (n_mu - 1) * FP32_ULP * mag
            else:
                g, gb = g_oracle(dz[l], act[l - 1], g_rtol(rows))
            mu_, wd, nest = (MU, WD, True) if stateful else (0.0, 0.0, False)
            v0 = vblocks0[l - 1] if stateful else torch.zeros_like(blocks[l - 1])
            Wr, bW, Vr, bV = sgd_oracle(g, gb, blocks[l - 1], v0, lr, mu_, wd, nest)
            res[f"upd{l}"] = excess(blocks1[l - 1], Wr, bW + ATOL)      # ATOL: a nil weight stays 0 at rate 0
            if stateful:
                res[f"mom{l}"] = excess(vblocks1[l - 1], Vr, bV + ATOL)
        else:
            ref, bound = rows_update_oracle(dz[l], act[l - 1], blocks[l - 1], lr, RTOL[precision])
            res[f"upd{l}"] = excess(blocks1[l - 1] - blocks[l - 1], ref, bound)
        k = model.arena.blocks[l - 1][1]
        assert bool(model.arena.block(l - 1)[:, k + 1:].isnan().all()), f"{what}: the padding of layer {l}'s weights changed"
    if lr == 0.0:                      # the parameters only: a NaN in the padding may come back with other bits
        for l in range(L):
            assert _bit_equal(blocks1[l], blocks[l]), f"{what}: lr 0 changed the weights of layer {l + 1}"
            if stateful:
                assert not _bit_equal(vblocks1[l], vblocks0[l]), f"{what}: layer {l + 1}'s momentum stood still at lr 0"

    # ---- the EMA: the reference lerp towards the new weights, bit for bit; training untouched by it
    n = model.arena.numel
    real = _real(model.arena)
    if st.get("E0") is not None:
        W1f, E1, E0 = W1[:n], model.arena.ema.detach(), st["E0"]
        want = ema_lerp_ref(E0, W1f, st["alpha"])
        assert torch.equal(E1[real], want[real]), f"{what}: an EMA entry is not lerp(E0, W1, {st['alpha']})"
        if per_mb_wgrad:                 # the flat pass runs over the whole arena: the padding follows the weights'
            assert _same(E1[~real], want[~real]), f"{what}: the flat pass left the EMA's padding behind"
        else:
            assert _same(E1[~real], E0[~real]), f"{what}: a fused EMA update wrote into the padding"
        frac = float((E1[real] != W1f[real]).double().mean())
        assert frac > 0.5, f"{what}: the EMA equals the weights on {1 - frac:.3f} of the entries"
    if st.get("W_plain") is not None:
        assert torch.equal(W1[:n][real], st["W_plain"][:n][real]), f"{what}: the EMA changed the weights"
        if stateful:
            assert torch.equal(V1[:n][real], st["V_plain"][:n][real]), f"{what}: the EMA changed the momentum"

    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, (what, bad)
    key = (c["form"], precision, "residual" if c["residual"] else "")
    worst = max(res, key=res.get)
    if c["form"] in FORMS and res[worst] > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (res[worst], f"{worst} at {what} of {c['name']}")
    return res


def check_eval(veng, model, W, x, t, n_mu, mb, precision, loss, count):
    """The evaluation engine's forward per layer from its own act[l - 1] at the flat weights ``W``
    (``check_residual_layers`` in its inference form: the skips of a residual model added, no gates), its probabilities
    per micro-batch, and ``count`` against argmax(probs) == argmax(t) over the rows (first maximum wins)."""
    L = len(model.linears)
    blocks = _blocks(model, W)
    act = [x.double()] + [_gather(lambda mu, l=l: veng.act(mu, l), n_mu) for l in range(1, L + 1)]
    res = {f"eval-{k}": v for k, v in check_residual_layers(veng, model, W, x, n_mu, mb, precision, 0.0,
                                                               training=False).items()}
    if model.residual:
        _branch_nonvacuous(model, blocks, act, model.activation, 0.0)
    else:
        for l in range(1, L):
            frac = float((act[l] > 0).double().mean())
            assert 0.05 <= frac <= 0.95, f"eval layer {l}: {frac:.3f} of the activations are positive"
    probs = _gather(veng.probs, n_mu)
    for mu in range(n_mu):
        r = slice(mu * mb, (mu + 1) * mb)
        (p, bp), _, _ = _head(loss)(act[L][r], t[r], n_mu * mb, HEAD_RTOL)
        res["eval-probs"] = max(res.get("eval-probs", 0.0), excess(probs[r], p, bp))
    want = int((probs.argmax(1) == t.argmax(1)).sum())
    assert count == want, f"count_correct {count}, argmax(probs) == argmax(targets) on {want} rows"
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


# ================================================================================================== GPU side
def _state(name):
    """Initial weights, momentum, EMA and the batches of case ``name``, from a generator of its own.  A shuffled case
    draws a dataset of EPOCH_BATCHES batches and SHUFFLE_SPARE rows, and step i's batch is the rows ``shuffle_index``
    picks for batch i % EPOCH_BATCHES of epoch i // EPOCH_BATCHES."""
    c = CASES[name]
    sizes, rows = c["sizes"], c["n_mu"] * c["mb"]
    gen = _gen("steps", name)
    state = {}
    if c["shuffle"]:
        n = EPOCH_BATCHES * rows + SHUFFLE_SPARE
        x_all = torch.randn(n, sizes[0], generator=gen)
        t_all = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (n,), generator=gen), sizes[-1]).float()
        pos = torch.arange(rows)
        ids = [shuffle_index(n, SHUFFLE_SEED, i // EPOCH_BATCHES, (i % EPOCH_BATCHES) * rows + pos) for i in range(STEPS)]
        xs, ts = [x_all[j] for j in ids], [t_all[j] for j in ids]
        state.update(x_all=x_all, t_all=t_all)
    else:
        xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(STEPS)]
        ts = [torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
              for _ in range(STEPS)]
    if c["residual"]:
        Ws, bs = _init_res_weights(sizes, _residual_flags(sizes), xs[0], c["n_mu"], gen, c["activation"])
    else:
        Ws, bs = _init_weights(sizes, xs[0], c["n_mu"], gen, c["activation"], far=c["activation"] != "relu")
    Vs = [torch.randn(o, i + 1, generator=gen) * V_SCALE for i, o in zip(sizes[:-1], sizes[1:])]
    xv = torch.randn(rows, sizes[0], generator=gen)
    tv = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    Es = [torch.cat([W, b[:, None]], 1) + 1e-2 * torch.randn(W.shape[0], W.shape[1] + 1, generator=gen)
          for W, b in zip(Ws, bs)]                                       # E0 != W0
    state.update(xs=xs, ts=ts, Ws=Ws, bs=bs, Vs=Vs, xv=xv, tv=tv, Es=Es)
    return state


def _trainer(c, state, monkeypatch, graph=None):
    """A Trainer of case ``c`` in its initial state, NaN in every padding column, on the path the case names
    (``graph``: overrides the case's use of CUDA graphs).  With an EMA: the EMA ``state["Es"]`` (EMA_PAD in its
    padding) and EMA_RESUMED updates behind it."""
    from shallowspeed_b200.parallel.engine import Trainer

    for k in FORMS[c["form"]]:
        monkeypatch.setenv(k, "1")
    sizes, n_mu, mb = c["sizes"], c["n_mu"], c["mb"]
    rule = dict(momentum=MU, weight_decay=WD, nesterov=True) if c["stateful"] else {}
    tr = Trainer(sizes, global_batch_size=n_mu * mb, n_mubatches=n_mu, lr=BUILD_LR, schedule=c["sched"],
                 precision=c["precision"], loss=c["loss"], activation=c["activation"], dropout=c["dropout"],
                 dropout_seed=DROP_SEED, use_graph=c["graph"] if graph is None else graph, residual=c["residual"],
                 ema_decay=c["ema_decay"][0] if c["ema_decay"] else None, **rule)
    model, eng = tr.model, tr.engine
    assert [lin.residual for lin in model.linears] == (_residual_flags(sizes) if c["residual"] else [False] * len(sizes[1:]))
    for i, (W, b) in enumerate(zip(state["Ws"], state["bs"])):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
        if c["stateful"]:
            model.arena.momentum_block(i)[:, : W.shape[1] + 1] = state["Vs"][i].cuda()
    if c["ema_decay"]:
        tr.optimizer.ema_updates = EMA_RESUMED
        model.arena.ema.fill_(EMA_PAD)
        for i, E in enumerate(state["Es"]):
            model.arena.ema_block(i)[:, : E.shape[1]] = E.cuda()
    _assert_path(eng, c)
    rows = n_mu * mb
    _poison(eng, model, sizes, rows, True, gated=c["activation"] != "relu" or c["residual"])
    for s in (0, 1):
        xs, ys = eng.staging(s)
        xs[:, sizes[0]:] = float("nan")
        ys[:, sizes[-1]:] = float("nan")
    torch.cuda.synchronize()
    return tr


def _assert_path(eng, c):
    form, text = c["form"], eng.plan_text(0) + eng.plan_text(1)
    assert eng.uses_chain() == form.startswith("chain"), eng.describe()
    assert eng.coalesced() == (form not in ("chain-per-mb", "layerwise-per-mb")), eng.describe()
    if form == "chain-cluster":
        assert (eng.chain_cluster(), eng.chain_ksplit()) == (4, 2)
    elif form == "chain-one-cta":
        assert (eng.chain_cluster(), eng.chain_ksplit()) == (1, 1)
    elif form == "chain-per-mb":
        assert text.count("wgrad_group") == 2, text                    # the deferred wave, once per staging set
    elif form == "layerwise-per-mb":
        assert text.count(" sgd ") == 2, text                          # the separate SGD pass, once per staging set
    splitk = int(eng.describe().split("splitk_gemms=")[1].split(",")[0])
    if form == "splitk":
        assert splitk > 0, eng.describe()
    if not form.startswith("chain") and form != "layerwise-per-mb":
        assert "wgrad_group" not in text and " sgd " not in text, text   # SGD fused into each wgrad epilogue
    if c["residual"]:
        assert "res=1" in text, text
    if c["ema_decay"]:
        assert f"ema={c['ema_decay'][0]:g}" in eng.describe(), eng.describe()
    mus = {int(m) for m in re.findall(r"mu=(\d+)", text)}
    assert mus == (set(range(c["n_mu"])) if form.endswith("per-mb") else mus & {0}), (mus, text)


def _dataset(c, state):
    """A shuffled case's training set as train.py keeps it: the whole file on the device, ``Dataset(shuffle_seed=...)``."""
    from shallowspeed_b200.dataset import Dataset

    rows = c["n_mu"] * c["mb"]
    ds = Dataset(None, rows, c["mb"], device="cuda", shuffle_seed=SHUFFLE_SEED)
    return ds.from_arrays(state["x_all"], state["t_all"], DP_rank=0, DP_size=1)


def _renil(tr, i):
    """Before step i > 0 of a residual model: zero the nil rows and columns of every residual layer again (the update
    moved them), on the engine's main stream, which its next run forks from, so no host sync is needed."""
    model = tr.model
    if i == 0 or not model.residual:
        return
    with torch.cuda.stream(torch.cuda.ExternalStream(tr.engine.main_stream(), device=model.arena.weights.device)):
        for j, lin in enumerate(model.linears):
            if lin.residual:
                model.arena.weight_view(j)[:, NIL_COL] = 0.0
                model.arena.weight_view(j)[NIL_ROW(lin.out_dims)] = 0.0
                model.arena.bias_view(j)[:, NIL_ROW(lin.out_dims)] = 0.0


def _train_step(tr, c, i, x, t, ds=None):
    """Step ``i`` as train.py runs it: the optimizer's rate (and EMA decay) and the model's dropout step set before the
    worker's step; from the shuffled dataset ``ds`` through ``execute``, else from ``x`` / ``t``."""
    tr.optimizer.lr = _rate(c, i)
    if c["ema_decay"]:
        tr.optimizer.ema_decay = c["ema_decay"][i]
    tr.model.dropout_step = c["drop_start"] + i
    if ds is not None:
        if i % EPOCH_BATCHES == 0:
            ds.set_epoch(i // EPOCH_BATCHES)
        tr.worker.execute(tr.schedule, i % EPOCH_BATCHES)
    else:
        tr.worker.step_from(tr.schedule, x, t)


_RECORDS = {}


def _checked_run(name, monkeypatch):
    """The case's six steps, each checked by ``check_step`` right after it (an EMA case next to the same run without
    EMA); returns the weights and EMA after every step, the final momentum and the loss of every step."""
    c = dict(CASES[name], name=name)
    state = _state(name)
    tr = _trainer(c, state, monkeypatch)
    plain = _trainer(dict(c, ema_decay=None), state, monkeypatch) if c["ema_decay"] else None
    ds = None
    if c["shuffle"]:
        ds = _dataset(c, state)
        for t_ in (tr, plain):
            if t_ is not None:
                t_.worker.dataset = ds          # the Trainer's worker, given the dataset train.py gives its worker
    eng, model = tr.engine, tr.model
    xh = [x.pin_memory() for x in state["xs"]]
    th = [t.pin_memory() for t in state["ts"]]
    rec = dict(W=[], E=[], losses=[])
    for i in range(STEPS):
        for t_ in (tr, plain):
            if t_ is not None:
                _renil(t_, i)
        torch.cuda.synchronize()
        W0 = model.arena.weights.detach().clone()
        V0 = model.arena.momentum.detach().clone() if c["stateful"] else None
        E0 = model.arena.ema.detach().clone() if c["ema_decay"] else None
        fill = eng.fill_set()
        _train_step(tr, c, i, xh[i], th[i], ds)
        loss = float(eng.last_loss())
        st = dict(i=i, x=state["xs"][i], t=state["ts"][i], x_prev=state["xs"][i - 1] if i else None,
                  t_prev=state["ts"][i - 1] if i else None, lr=_rate(c, i), dstep=c["drop_start"] + i, W0=W0, V0=V0,
                  E0=E0, alpha=_alpha(c, i), loss=loss, fill=fill)
        if plain is not None:
            _train_step(plain, c, i, xh[i], th[i], ds)
            assert float(plain.engine.last_loss()) == loss, f"step {i}: the EMA changed the loss"
            st.update(W_plain=plain.model.arena.weights.detach(),
                      V_plain=plain.model.arena.momentum.detach() if c["stateful"] else None)
            assert tr.optimizer.ema_updates == EMA_RESUMED + i + 1
        torch.cuda.synchronize()
        check_step(eng, model, c, st)
        if c["activation"] != "relu" or c["residual"]:
            for l in range(1, len(c["sizes"]) - 1):
                pad = _pitched(eng.gate(0, l), c["n_mu"] * c["mb"])[:, c["sizes"][l]:]
                assert bool(pad.isnan().all()), f"step {i} layer {l}: a kernel wrote into the gate's padding"
        rec["W"].append(model.arena.weights.detach().cpu().clone())
        rec["E"].append(model.arena.ema.detach().cpu().clone() if c["ema_decay"] else None)
        rec["losses"].append(loss)
    rec["V"] = model.arena.momentum.detach().cpu().clone() if c["stateful"] else None
    # the rate changed across the warm-up steps
    sched = SCHEDULES.get(c["lr_schedule"])
    if sched is not None:
        assert all(sched(j) != sched(j - 1) for j in range(1, sched.warmup_steps + 1)), c["lr_schedule"]
    return rec


def _record(name, monkeypatch):
    if name not in _RECORDS:
        _RECORDS[name] = _checked_run(name, monkeypatch)
    return _RECORDS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_every_step_matches_fp64(name, monkeypatch):
    _RECORDS[name] = _checked_run(name, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("name", REPLAYS)
def test_unsynchronised_and_eager_steps_are_bitwise_the_checked_run(name, monkeypatch):
    """The case replayed as ``bench.py`` runs it: ``step_async`` on device-resident inputs with no host sync, and
    ``step_pipelined`` + ``flush`` from pinned host memory; and once more with the plan walked eagerly instead of
    replayed from its graphs (the same kernels in the same order), each step through ``Trainer.step``.  The rate comes
    from ``Trainer.lr_schedule`` and the dropout step from the Trainer's step count.  Weights, momentum, EMA and losses
    equal the checked run's."""
    rec = _record(name, monkeypatch)
    c = CASES[name]
    assert c["graph"]
    state = _state(name)
    for mode in ("async", "pipelined", "eager"):
        tr = _trainer(c, state, monkeypatch, graph=mode != "eager")
        tr.lr_schedule = SCHEDULES[c["lr_schedule"]] if c["lr_schedule"] else LRS.__getitem__

        def before(i):
            _renil(tr, i)
            if c["ema_decay"]:
                tr.optimizer.ema_decay = c["ema_decay"][i]     # the caller's alpha sequence

        if mode == "eager":
            xh = [x.pin_memory() for x in state["xs"]]
            th = [t.pin_memory() for t in state["ts"]]
            losses = []
            for i in range(STEPS):
                before(i)
                losses.append(float(tr.step(xh[i], th[i])))
            want = rec["losses"]
        elif mode == "async":
            xd = [x.cuda() for x in state["xs"]]
            td = [t.cuda() for t in state["ts"]]
            for i in range(STEPS):
                before(i)
                tr.step_async(xd[i], td[i])
            tr.synchronize()
            losses = [float(tr.loss())]
            want = rec["losses"][-1:]
        else:
            xh = [x.pin_memory() for x in state["xs"]]
            th = [t.pin_memory() for t in state["ts"]]
            lagged = []
            for i in range(STEPS):
                before(i)
                lagged.append(tr.step_pipelined(xh[i], th[i]))
            lagged.append(tr.flush())
            tr.synchronize()
            assert lagged[0] is None
            losses = [float(v) for v in lagged[1:]]
            want = rec["losses"]
        torch.cuda.synchronize()
        assert _bit_equal(tr.model.arena.weights, rec["W"][-1]), f"{mode}: the weights differ from the checked run's"
        if c["stateful"]:
            assert _bit_equal(tr.model.arena.momentum, rec["V"]), f"{mode}: the momentum differs from the checked run's"
        if c["ema_decay"]:
            assert _bit_equal(tr.model.arena.ema, rec["E"][-1]), f"{mode}: the EMA differs from the checked run's"
            assert tr.optimizer.ema_updates == EMA_RESUMED + STEPS
        assert [_bits(torch.tensor(v)) for v in losses] == [_bits(torch.tensor(v)) for v in want], (mode, losses, want)
        del tr


@pytest.mark.gpu
@pytest.mark.parametrize("name", EVALS)
def test_evaluation_between_training_steps(name, monkeypatch):
    """train.py's evaluation engine (``NativeWorker(..., share=worker)``, ``InferenceSchedule``) between two training
    steps, nothing synchronised until the end: the training run is bitwise the checked one, and the evaluation reads the
    weights of the step before it.  With an EMA, train.py's EMA evaluation as well: ``ema_state()`` copied into a
    second model's arena, run by that model's own inference worker, and checked against the EMA of that step."""
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.models.mlp import MLP
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import InferenceSchedule

    rec = _record(name, monkeypatch)
    c = CASES[name]
    state = _state(name)
    tr = _trainer(c, state, monkeypatch)
    rows, n_ev = c["n_mu"] * c["mb"], c["eval_mu"]
    val = Dataset(None, rows, rows // n_ev, device="cuda")
    val.local_batch_size = rows
    val.from_arrays(state["xv"], state["tv"])
    sched = InferenceSchedule(n_ev, 1, 0)
    workers = [(tr.model, NativeWorker(None, None, tr.model, val, None, use_graph=c["graph"],
                                       precision=c["precision"], share=tr.worker))]
    if c["ema_decay"]:
        ema_model = MLP(c["sizes"], 0, 1, rows, loss=c["loss"], activation=c["activation"], residual=c["residual"])
        ema_model.to("cuda")
        workers.append((ema_model, NativeWorker(None, None, ema_model, val, None, use_graph=c["graph"],
                                                precision=c["precision"], share=tr.worker)))
    engines = []
    for model, vw in workers:
        veng = vw.engine_for(sched)                    # built (and synchronised) before the run
        assert veng.uses_chain() == c["form"].startswith("chain")
        _poison(veng, model, c["sizes"], rows, False)
        engines.append(veng)
    torch.cuda.synchronize()
    xh = [x.pin_memory() for x in state["xs"]]
    th = [t.pin_memory() for t in state["ts"]]
    for i in range(STEPS):
        _renil(tr, i)
        _train_step(tr, c, i, xh[i], th[i])
        if i == EVAL_AFTER:
            engines[0].reset_correct()
            workers[0][1].execute(sched, 0)
            if c["ema_decay"]:                         # train.py's evaluate(): ema_state() synchronises the worker
                ema_model, ew = workers[1]
                ema = tr.ema_state()
                ema_model.arena.weights[: ema_model.arena.numel].copy_(ema)
                engines[1].reset_correct()
                ew.execute(sched, 0)
    tr.worker.synchronize()
    for _, vw in workers:
        vw.synchronize()
    torch.cuda.synchronize()
    assert _bit_equal(tr.model.arena.weights, rec["W"][-1]), "the training run differs from the uninterrupted one"
    if c["ema_decay"]:
        assert _bit_equal(tr.model.arena.ema, rec["E"][-1]), "the EMA differs from the uninterrupted run's"
    mb = rows // n_ev
    evaluated = [("weights", rec["W"][EVAL_AFTER])] + ([("EMA", rec["E"][EVAL_AFTER])] if c["ema_decay"] else [])
    for (what, W), (model, vw), veng in zip(evaluated, workers, engines):
        res = check_eval(veng, model, W, state["xv"], state["tv"], n_ev, mb, c["precision"], c["loss"],
                         veng.count_correct())
        out0 = vw.output_buffers[0]
        assert out0.data_ptr() == veng.probs(0).data_ptr() and out0.shape == veng.probs(0).shape
        print(f"\n[steps] eval of the {what} of {name} ({n_ev} micro-batches): "
              + " ".join(f"{k}={v:.2g}" for k, v in res.items()))


# ================================================================================================== CPU side
def _slot_writes(values, initial):
    """Which steps must write their staging set's slot (PipeEngine::run: one slot per set for the rate, the dropout step
    and the EMA alpha, each rewritten only when it holds another value)."""
    held, out = [initial, initial], []
    for i, v in enumerate(values):
        out.append(held[i % 2] != v)
        held[i % 2] = v
    return out


SITES = {"chain-cluster": "grouped", "chain-one-cta": "grouped", "chain-per-mb": "grouped", "layerwise": "fused",
         "splitk": "fused", "layerwise-per-mb": "flat"}     # where the update (and the EMA) of each form runs


def test_grid_reaches_every_branch():
    from shallowspeed_b200 import _C
    from shallowspeed_b200.lr_schedule import KINDS
    from shallowspeed_b200.ops.functional import precision_code

    table = {"chain-cluster": {3, 4, 9, 17, 32, 128}, "chain-one-cta": {4, 17}, "chain-per-mb": {9, 17},
             "layerwise": {4, 17}, "layerwise-per-mb": {9, 17}, "splitk": {2, 3}}
    counts = {f: set() for f in FORMS}
    feats = {k: set() for k in ("stateful", "gelu-drop", "ce", "eager", "residual", "shuffle", "bf16-stateful",
                                "bf16-ema")}
    precisions = {p: set() for p in ("fp32", "tf32", "bf16")}
    forms = {site: set() for site in ("plain", "rule", "ema-plain", "ema-rule")}    # SgdForm (and rule) per site
    scheds, activations, losses, lr_kinds = set(), set(), set(), set()
    for name, c in CASES.items():
        f, n_mu, mb, pr = c["form"], c["n_mu"], c["mb"], c["precision"]
        counts[f].add(n_mu)
        precisions[pr].add(f)
        layers = list(zip(c["sizes"][:-1], c["sizes"][1:]))
        eligible = _C.chain_eligible(layers, mb, c["sizes"][-1], True, precision_code(pr))
        assert eligible == (f != "splitk"), name                       # layer-wise REF runs layer-wise by SSB_NO_CHAIN
        res = _residual_flags(c["sizes"])
        if f in ("chain-cluster", "chain-one-cta"):
            cl = _C.chain_cluster_size(layers, True, True, True, True, False, False)
            ksplit = cl > 1 and -(-c["sizes"][0] // 32) > 4
            assert (cl, ksplit) == ((4, True) if f == "chain-cluster" else (1, False)), name
            assert _C.chain_cluster_budget(mb, cl, precision_code(pr))[0]
            if c["residual"] and f == "chain-cluster":
                assert res[1] and not res[0], name                     # the k-split layer 1 feeds a residual layer
        if f == "splitk":
            assert c["sizes"] in (WIDE["1000-1500-777"], RES_SPLITK), name
        if f == "chain-per-mb":
            scheds.add((c["sched"], n_mu))
        if c["stateful"]:
            feats["stateful"].add(f)
        if c["activation"] == "gelu" and c["dropout"] == DROP_P:
            feats["gelu-drop"].add(f)
        if c["loss"] == "cross_entropy":
            feats["ce"].add(f)
        if not c["graph"]:
            feats["eager"].add(f)
        if c["residual"]:
            assert any(res), name
            feats["residual"].add(f)
        if c["shuffle"]:
            feats["shuffle"].add(f)
        if pr == "bf16" and c["stateful"]:
            feats["bf16-stateful"].add(f)
        if pr == "bf16" and c["ema_decay"]:
            feats["bf16-ema"].add(f)
        forms[("ema-" if c["ema_decay"] else "") + ("rule" if c["stateful"] else "plain")].add(SITES[f])
        activations.add(c["activation"])
        losses.add(c["loss"])
        lr_kinds.add(c["lr_schedule"])
        if c["replay"]:
            assert c["drop_start"] == 0, name                          # Trainer draws the masks of step _steps
            assert c["graph"], name                                    # the eager replay is the other plan walk
            assert not c["shuffle"], name                              # the replays stage the batches themselves
        if c["ema_decay"]:
            alphas = [_alpha(c, i) for i in range(STEPS)]
            assert alphas[0] < 1.0 and min(alphas) < 0.5 <= max(alphas), name   # resumed; both branches of the lerp
    assert counts == table, counts
    assert {("naive", 9), ("gpipe", 9), ("pipedream", 9), ("gpipe", 17)} <= scheds
    # more than 8 micro-batches (shared streams) in both per-micro-batch forms, more than 16 (the loss stride) in a
    # coalesced and a per-micro-batch form, and counts that are not powers of two
    assert all(max(counts[f]) > 8 for f in ("chain-per-mb", "layerwise-per-mb"))
    assert max(counts["chain-cluster"]) > 16 and max(counts["chain-per-mb"]) > 16
    assert any(n & (n - 1) for n in counts["chain-cluster"])
    # tf32 in every form the chain kernel or the layer-wise GEMMs run at their own widths, bf16 in every form
    assert precisions["tf32"] == set(FORMS) - {"splitk"} and precisions["bf16"] == set(FORMS), precisions
    assert sum(c["precision"] == "tf32" for c in CASES.values()) >= 6
    assert sum(c["precision"] == "bf16" for c in CASES.values()) >= 6
    assert feats["bf16-stateful"] and feats["bf16-ema"]
    assert feats["stateful"] == set(FORMS) and feats["residual"] == set(FORMS)
    # every update form at every site, the EMA with a plain rule and with momentum; the deferred wave with an EMA
    assert all(sites == {"grouped", "fused", "flat"} for sites in forms.values()), forms
    assert any(c["form"] == "chain-per-mb" and c["ema_decay"] for c in CASES.values())
    assert {"chain-cluster", "chain-per-mb"} <= feats["gelu-drop"] and feats["gelu-drop"] & {"layerwise", "layerwise-per-mb"}
    assert feats["ce"] & {"chain-cluster", "chain-one-cta", "chain-per-mb"} and feats["ce"] & {"layerwise", "layerwise-per-mb"}
    assert feats["eager"] & {"chain-cluster", "chain-one-cta", "chain-per-mb"} and feats["eager"] & {"layerwise", "layerwise-per-mb"}
    assert feats["shuffle"] & {"chain-cluster", "chain-one-cta", "chain-per-mb"} and feats["shuffle"] & {"layerwise", "layerwise-per-mb"}
    assert activations == {"relu", "gelu", "silu", "tanh"} and losses == {"mse", "cross_entropy"}
    assert any(c["drop_start"] > 0 and c["dropout"] > 0 for c in CASES.values())
    assert any(c["drop_start"] > 0 and c["dropout"] > 0 and c["residual"] for c in CASES.values())
    # each staging set runs at least two checked steps; an lr-0 step; a step whose set needs no slot write while the
    # other set changed in between
    assert STEPS >= 4
    assert 0.0 in LRS and all(float(torch.tensor(lr, dtype=torch.float32)) == lr for lr in LRS)
    writes = _slot_writes(LRS, BUILD_LR)
    assert any(not writes[i] and LRS[i - 1] != LRS[i] for i in range(2, STEPS)), writes
    # every schedule kind with a warm-up, at fp32 rates; a step at rate 0 and a step that needs no slot write
    assert lr_kinds == set(KINDS) | {None} and set(SCHEDULES) == set(KINDS)
    rates = {k: [s(i) for i in range(STEPS)] for k, s in SCHEDULES.items()}
    for k, s in SCHEDULES.items():
        assert s.kind == k and s.warmup_steps >= 1 and s.warmup_start_factor < 1.0, k
        assert all(float(torch.tensor(r, dtype=torch.float32)) == r for r in rates[k])
        assert all(rates[k][i] != rates[k][i - 1] for i in range(1, s.warmup_steps + 1)), k
    assert any(0.0 in r for r in rates.values())
    assert any(not all(_slot_writes(r, BUILD_LR)) for r in rates.values())
    # a shuffled case runs two epochs of three batches, and the epoch's spare rows differ
    assert STEPS >= 2 * EPOCH_BATCHES >= 6 and SHUFFLE_SPARE > 0
    # the replays: the bench-shaped reference case, a per-micro-batch and a layer-wise one, an EMA + schedule + dropout
    # case whose rate, dropout step and alpha slots are rewritten at every step, and a bf16 residual case
    assert "chain-ref-4x32" in REPLAYS and CASES["chain-ref-4x32"]["sizes"] == REF
    assert any(CASES[n]["form"].endswith("per-mb") for n in REPLAYS)
    assert any(CASES[n]["form"].startswith("layerwise") for n in REPLAYS)
    assert any(CASES[n]["precision"] == "bf16" and CASES[n]["residual"] for n in REPLAYS)
    moving = [n for n in REPLAYS if CASES[n]["ema_decay"] and CASES[n]["lr_schedule"] and CASES[n]["dropout"] > 0]
    assert moving
    for n in moving:
        c = CASES[n]
        assert all(_slot_writes([_rate(c, i) for i in range(STEPS)], BUILD_LR)), n
        assert all(_slot_writes([_alpha(c, i) for i in range(STEPS)], 1.0)), n
    # the evaluations: the chain and the layer-wise form, once with 9 micro-batches; the EMA of a plain and of a
    # residual model
    assert {CASES[n]["form"].split("-")[0] for n in EVALS} == {"chain", "layerwise"}
    assert {1, 9} <= {CASES[n]["eval_mu"] for n in EVALS}
    assert {CASES[n]["residual"] for n in EVALS if CASES[n]["ema_decay"]} == {False, True}
    assert not any(CASES[n]["shuffle"] for n in EVALS)                 # the evaluations stage the batches themselves
    assert 0 <= EVAL_AFTER < STEPS - 1


# ---------------------------------------------------------------- the checks against an emulated engine
EMU_SIZES = [12, 20, 20, 20, 5]          # residual layers 2 and 3
EMU = dict(name="emulated", sizes=EMU_SIZES, form="emulated", n_mu=17, mb=2, precision="fp32", loss="mse",
           activation="relu", dropout=DROP_P, drop_start=7, stateful=True, residual=True, ema_decay=EMA_DECAYS,
           lr_schedule="linear", shuffle=True)
FAULTS = ("lr-of-previous-step", "mask-of-previous-step", "layer-1-wgrad-from-other-set", "targets-of-other-set",
          "momentum-restarted-in-set-1", "dgrad-from-micro-batch-8-back", "loss-without-micro-batches-16-up",
          "eval-one-step-stale", "count-against-other-set",
          "ema-alpha-of-other-set", "ema-alpha-of-previous-step", "ema-lerp-towards-W0", "ema-bias-not-updated",
          "ema-into-padding", "skip-rounded-like-bf16", "lr-of-other-set", "lr-schedule-one-step-behind",
          "staging-unshuffled", "staging-of-previous-epoch", "ema-perturbs-weights")


class _Emulated:
    """A pp = 1 training engine emulated in fp32 on the CPU, with the buffers ``check_step`` reads: two staging sets
    (NaN in the padding) gathered from a shuffled dataset, act / gate / dz / probs per micro-batch, the loss, and the
    model arena's weights, momentum and EMA, updated in place by the stateful rule; a slot per staging set for the rate
    and the EMA alpha.  ``fault`` makes it commit one of FAULTS."""

    def __init__(self, model, n_mu, mb, data, fault=None):
        self.model, self.n_mu, self.mb, self.data, self.fault = model, n_mu, mb, data, fault
        rows, i, o = n_mu * mb, model.in_dim, model.out_dim
        self.sets = []
        for _ in range(2):
            x, y = torch.zeros(rows, i + 3), torch.zeros(rows, o + 3)
            x[:, i:] = y[:, o:] = float("nan")
            self.sets.append((x, y))
        self.lr_slot, self.alpha_slot = [BUILD_LR, BUILD_LR], [1.0, 1.0]
        self.fill, self.prev_lr, self.a, self.g, self.d, self.p = 0, None, [], [], [], None

    def staging(self, s):
        return self.sets[s]

    def fill_set(self):
        return self.fill

    def uses_chain(self):
        return True

    def _rows(self, t, mu):
        return t[mu * self.mb:(mu + 1) * self.mb]

    def act(self, mu, l):
        return self._rows(self.a[l], mu)

    def gate(self, mu, l):
        return self._rows(self.g[l], mu)

    def dz(self, mu, l):
        return self._rows(self.d[l], mu)

    def probs(self, mu):
        return self._rows(self.p, mu)

    def _gather(self, i):
        """Stage step i's batch into the fill set, as stage_gather does: the rows of its epoch's permutation."""
        f, rows = self.fault, self.n_mu * self.mb
        x_all, t_all = self.data
        epoch, b = i // EPOCH_BATCHES, i % EPOCH_BATCHES
        if f == "staging-of-previous-epoch":
            epoch = max(epoch - 1, 0)
        q = b * rows + torch.arange(rows)
        ids = q if f == "staging-unshuffled" else shuffle_index(len(x_all), SHUFFLE_SEED, epoch, q)
        s_set = self.sets[self.fill]
        s_set[0][:, : x_all.shape[1]] = x_all[ids]
        s_set[1][:, : t_all.shape[1]] = t_all[ids]

    def step(self, i, lr, alpha, dstep, sched):
        from shallowspeed_b200.ops import functional as F

        m, f, n_mu, mb = self.model, self.fault, self.n_mu, self.mb
        self._gather(i)
        s_set, o_set = self.sets[self.fill], self.sets[self.fill ^ 1]
        x, t = s_set[0][:, : m.in_dim].clone(), s_set[1][:, : m.out_dim].clone()
        if f == "targets-of-other-set":
            t = o_set[1][:, : m.out_dim].clone()
        if f == "lr-schedule-one-step-behind":
            lr = sched(max(i - 1, 0))
        lr_used = {"lr-of-previous-step": self.prev_lr, "lr-of-other-set": self.lr_slot[self.fill ^ 1]}.get(f) or lr
        self.lr_slot[self.fill] = lr
        alpha_used = {"ema-alpha-of-other-set": self.alpha_slot[self.fill ^ 1],
                      "ema-alpha-of-previous-step": self.alpha_slot[self.fill]}.get(f, alpha)
        self.alpha_slot[self.fill] = alpha
        scale = torch.tensor(F.dropout_scale(m.dropout), dtype=torch.float32)
        samples = torch.arange(n_mu * mb)
        blocks = [m.arena.block(j)[:, : k + 1].clone() for j, (_, k) in enumerate(m.arena.blocks)]
        a, gates = [x], [None]
        for lin, B in zip(m.linears, blocks):
            z = a[-1] @ B[:, :-1].T + B[:, -1]
            if lin.activation is None:
                a.append(z)
                gates.append(None)
                continue
            keep = F.dropout_mask(m.dropout, m.dropout_seed, lin.dropout[2],
                                  dstep - 1 if f == "mask-of-previous-step" else dstep, samples, lin.out_dims)
            gates.append(torch.where(keep, (z > 0).float() * scale, torch.zeros(())))
            branch = torch.where(keep, z.clamp_min(0.0) * scale, torch.zeros(()))
            if lin.residual:
                skip = bf(a[-1]).float() if f == "skip-rounded-like-bf16" else a[-1]
                branch = skip + branch
            a.append(branch)
        L = len(blocks)
        d = [None] * (L + 1)
        probs, dzs, losses = [], [], []
        for mu in range(n_mu):
            zl, tl = self._rows(a[L], mu), self._rows(t, mu)
            p = F.softmax_ref(zl)
            probs.append(p)
            dzs.append(F.softmax_grad_ref(F.mse_loss_grad_ref(p, tl, n_mu * mb), zl))
            losses.append(F.mse_loss_ref(p, tl, n_mu * mb))
        self.p, d[L] = torch.cat(probs), torch.cat(dzs)
        g = None                                   # g_l = dL/da_l of a residual layer l, fp32 (the chain's registers)
        for l in range(L, 1, -1):
            src = d[l].clone()
            if f == "dgrad-from-micro-batch-8-back":
                src[8 * mb:] = d[l][: (n_mu - 8) * mb]
            pre = src @ blocks[l - 1][:, :-1]
            if m.linears[l - 1].residual:
                pre = pre + g
            g = pre
            d[l - 1] = pre * gates[l - 1]
        d[0] = torch.zeros_like(x)
        self.loss = float(sum(losses[:16] if f == "loss-without-micro-batches-16-up" else losses))
        W0 = m.arena.weights.clone()
        for j, (_, k) in enumerate(m.arena.blocks):
            a_in = o_set[0][:, : x.shape[1]] if f == "layer-1-wgrad-from-other-set" and j == 0 else a[j]
            gr = torch.cat([d[j + 1].T @ a_in, d[j + 1].sum(0)[:, None]], 1)
            W, Vb = m.arena.block(j)[:, : k + 1], m.arena.momentum_block(j)[:, : k + 1]
            v0 = torch.zeros_like(Vb) if f == "momentum-restarted-in-set-1" and self.fill == 1 else Vb
            gp = gr + WD * W
            v = MU * v0 + gp
            W -= lr_used * (gp + MU * v)
            Vb.copy_(v)
        if m.arena.ema is not None:
            n = m.arena.numel
            if f == "ema-perturbs-weights":
                m.arena.block(1).view(torch.int32)[3, 5] += 1               # one ulp
            e0 = m.arena.ema.clone()
            want = ema_lerp_ref(e0, (W0 if f == "ema-lerp-towards-W0" else m.arena.weights)[:n], alpha_used)
            real = _real(m.arena)
            if f == "ema-bias-not-updated":
                for j, (o, k) in enumerate(m.arena.blocks):
                    real[m.arena.offsets[j]:][: o * m.arena.lds[j]].view(o, -1)[:, k] = False
            m.arena.ema.copy_(want if f == "ema-into-padding" else torch.where(real, want, e0))
        self.a, self.g, self.d, self.prev_lr = a, gates, d, lr
        self.fill ^= 1


class _EmulatedEval:
    """The inference engine emulated in fp32: act per layer (the skips added), probs and count_correct of one forward at
    given weights."""

    def __init__(self, model, W, x, t, n_mu, mb, fault=None):
        from shallowspeed_b200.ops import functional as F

        self.mb = mb
        blocks = _blocks(model, W)
        a = [x]
        for lin, B in zip(model.linears, blocks):
            z = a[-1] @ B[:, :-1].float().T + B[:, -1].float()
            if lin.activation is not None:
                z = a[-1] + z.clamp_min(0.0) if lin.residual else z.clamp_min(0.0)
            a.append(z)
        self.a = a
        self.p = torch.cat([F.softmax_ref(a[-1][mu * mb:(mu + 1) * mb]) for mu in range(n_mu)])
        targets = torch.zeros_like(t) if fault == "count-against-other-set" else t
        self.count = int((self.p.argmax(1) == targets.argmax(1)).sum())

    def act(self, mu, l):
        return self.a[l][mu * self.mb:(mu + 1) * self.mb]

    def probs(self, mu):
        return self.p[mu * self.mb:(mu + 1) * self.mb]


def _emulated_run(fault, plain=None):
    """The six emulated steps of EMU: without its EMA, or, given the weights and momentum of that run after every step
    (``plain``), with it and each step through ``check_step``.  Returns the weights and momentum after every step, the
    model and the generator."""
    from shallowspeed_b200.models.mlp import MLP

    ema = plain is not None
    c = dict(EMU, ema_decay=EMU["ema_decay"] if ema else None)
    n_mu, mb, sizes = c["n_mu"], c["mb"], c["sizes"]
    rows = n_mu * mb
    model = MLP(sizes, 0, 1, rows, dropout=c["dropout"], dropout_seed=DROP_SEED, residual=True)
    model.arena.enable_momentum()
    gen = _gen("emulated")
    n = EPOCH_BATCHES * rows + SHUFFLE_SPARE
    x_all = torch.randn(n, sizes[0], generator=gen)
    t_all = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (n,), generator=gen), sizes[-1]).float()
    ids = [shuffle_index(n, SHUFFLE_SEED, i // EPOCH_BATCHES, (i % EPOCH_BATCHES) * rows + torch.arange(rows))
           for i in range(STEPS)]
    xs, ts = [x_all[j] for j in ids], [t_all[j] for j in ids]
    Ws, bs = _init_res_weights(sizes, [lin.residual for lin in model.linears], xs[0], n_mu, gen, c["activation"])
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
        o, k = model.arena.blocks[i]
        model.arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen) * V_SCALE
        model.arena.block(i)[:, k + 1:] = float("nan")
    if ema:
        model.arena.enable_ema()
        model.arena.ema.fill_(EMA_PAD)
        for i, (o, k) in enumerate(model.arena.blocks):
            model.arena.ema_block(i)[:, : k + 1] = model.arena.block(i)[:, : k + 1] + 1e-2 * torch.randn(o, k + 1, generator=gen)
    eng = _Emulated(model, n_mu, mb, (x_all, t_all), fault)
    sched = SCHEDULES[c["lr_schedule"]]
    out = []
    for i in range(STEPS):
        if i:
            for j, lin in enumerate(model.linears):         # the nil features again, as _renil
                if lin.residual:
                    model.arena.weight_view(j)[:, NIL_COL] = 0.0
                    model.arena.weight_view(j)[NIL_ROW(lin.out_dims)] = 0.0
                    model.arena.bias_view(j)[:, NIL_ROW(lin.out_dims)] = 0.0
        W0, V0, fill = model.arena.weights.clone(), model.arena.momentum.clone(), eng.fill_set()
        E0 = model.arena.ema.clone() if ema else None
        dstep = c["drop_start"] + i
        eng.step(i, sched(i), _alpha(c, i) if ema else 1.0, dstep, sched)
        if ema:
            st = dict(i=i, x=xs[i], t=ts[i], x_prev=xs[i - 1] if i else None, t_prev=ts[i - 1] if i else None,
                      lr=sched(i), dstep=dstep, W0=W0, V0=V0, E0=E0, alpha=_alpha(c, i), loss=eng.loss, fill=fill,
                      W_plain=plain[i][0], V_plain=plain[i][1])
            check_step(eng, model, c, st)
        out.append((model.arena.weights.clone(), model.arena.momentum.clone()))
    return out, model, gen


def _check_emulated(fault=None):
    """Six emulated steps of EMU, each through ``check_step`` next to the same run without EMA, then an evaluation
    after step 1 through ``check_eval``."""
    plain, _, _ = _emulated_run(fault)
    snaps, model, gen = _emulated_run(fault, plain)
    n_mu, mb, sizes = EMU["n_mu"], EMU["mb"], EMU["sizes"]
    rows = n_mu * mb
    xv = torch.randn(rows, sizes[0], generator=gen)
    tv = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    j = 1
    veng = _EmulatedEval(model, snaps[j - 1][0] if fault == "eval-one-step-stale" else snaps[j][0], xv, tv, n_mu, mb,
                         fault)
    check_eval(veng, model, snaps[j][0], xv, tv, n_mu, mb, EMU["precision"], EMU["loss"], veng.count)


def test_checks_accept_the_emulated_engine():
    _check_emulated()


@pytest.mark.parametrize("fault", FAULTS)
def test_checks_reject_injected_faults(fault):
    with pytest.raises(AssertionError):
        _check_emulated(fault)
