"""The one-GPU engine (pp = 1, dp = 1) per element against fp64 at EVERY step of a six-step run, in both input-staging
sets, at up to 128 micro-batches.

``PipeEngine`` plans two complete steps, one per staging set, each captured into a graph of its own with its own
device state (the x / y staging buffers, the learning-rate slot, the dropout-step slot, the pinned loss slot), and
``run()`` alternates them while the momentum carries over.  The micro-batch index reaches the row offsets of every
buffer, the chain kernel's ``mu_base``, the dropout rows, the loss slot (stride ``max(n_mu, 16)``), the targets and the
stream map (at most 8 micro-batch streams, so past 8 micro-batches several share one).  Every step of every case below
is checked by ``check_step`` from the engine's own buffers, with the oracles of ``test_gpu_chain.py``,
``test_gpu_gemm.py`` and ``test_gpu_cross_entropy.py``, so errors cannot cascade from step to step:

* staging: set i % 2 holds step i's x and targets bitwise and NaN in its padding, the other set step i - 1's inputs,
  and ``fill_set()`` alternates;
* every layer of every micro-batch (``check_layers``: forward, gates, dropped elements +0, dgrad) with the masks of the
  step's dropout step; the loss head (probabilities, dz_L, and the step's loss against the sum over micro-batches);
* the update at the step's own rate (the per-step rates below; 0.0 leaves W bitwise unchanged and V still advances),
  plain or stateful, deferred / coalesced or accumulated per micro-batch through memory; the momentum per element;
  NaN still in the weights' padding;
* non-vacuity at every step: 5-95 % of every hidden activation positive, every dz non-zero, live units dropped under
  dropout, |z| > 9 reached under a smooth activation.

The device-timed and the pipelined steps of ``bench.py`` never synchronise with the host; for a subset of cases the
same run is replayed through ``Trainer.step_async`` (device-resident inputs) and ``Trainer.step_pipelined`` (pinned host
memory, lagged losses), and once more with the plan walked eagerly instead of replayed from its CUDA graphs; each must
reproduce the checked run's weights, momentum and losses bit for bit (the kernels sum in a fixed order).  The
evaluation engine of ``train.py`` (a second ``NativeWorker`` sharing the first, ordered behind it by
``NativeWorker._enter``) runs between two training steps without a host sync; its forward, probabilities and
``count_correct`` are checked against the weights of the step before it.

The CPU tests check that the grid reaches every branch named above and that the checks reject a set of injected faults
in a three-step fp32 emulation of the engine while they accept the clean emulation.

Worst err / bound over all six steps, measured on an H100 80GB HBM3 (700 W): chain with a cluster fp32 0.57 / tf32 0.95,
chain on one CTA 0.43 / 0.71, chain per micro-batch 0.50 / 0.89, layer-wise 0.50 / 0.97, layer-wise per micro-batch
0.57 / 0.93, split-K fp32 0.59; the interleaved evaluation 0.14.  Every case stays non-degenerate at these rates, the
eager replays are bitwise the graph runs, and the file takes about 30 s there.
"""
import math
import re

import pytest
import torch

from test_gpu_chain import (DROP_P, DROP_SEED, HEAD_RTOL, RTOL, U, _gather, _init_weights, _pitched, _poison,
                            act_fwd_oracle, check_layers, excess, fwd_oracle, head_oracle, rows_update_oracle)
from test_gpu_cross_entropy import ce_head_oracle
from test_gpu_gemm import FP32_ULP, MU, WD, WIDE, _gen, grad_oracle, rtol_for, sgd_oracle

REF = [784, 128, 127, 126, 125, 124, 123, 10]    # the reference model, the benchmark's flagship
ONE_CTA = [784, 32, 24, 10]                        # every layer at most 32 wide: one CTA per micro-batch
SPLITK = WIDE["1000-1500-777"]                     # layer-wise GEMMs with split-K forward and dgrad
BUILD_LR = 0.5
# the rate of each step, all exact in fp32.  Step 3 (set 1) needs no slot write: its set still holds 0.25 from step 1,
# while set 0 went to 0.375 in between.  Step 4 runs at 0.
LRS = (0.25, 0.25, 0.375, 0.25, 0.0, 0.375)
STEPS = len(LRS)
EVAL_AFTER = 2                                     # the interleaved evaluation runs between steps 2 and 3
V_SCALE = 1e-3                                     # the momentum a stateful case starts from

NO_CHAIN, NO_COALESCE = "SSB_NO_CHAIN", "SSB_NO_COALESCE"
FORMS = {                                          # form -> environment that selects it
    "chain-cluster": (), "chain-one-cta": (), "chain-per-mb": (NO_COALESCE,), "layerwise": (NO_CHAIN,),
    "layerwise-per-mb": (NO_CHAIN, NO_COALESCE), "splitk": (),
}


def _case(sizes, form, n_mu, mb, sched="naive", precision="fp32", loss="mse", activation="relu", dropout=0.0,
          drop_start=0, stateful=False, graph=True, replay=False, eval_mu=None):
    """``replay``: also run the unsynchronised replays; ``eval_mu``: also run the interleaved evaluation with this many
    micro-batches (None: not at all)."""
    return dict(sizes=sizes, form=form, n_mu=n_mu, mb=mb, sched=sched, precision=precision, loss=loss,
                activation=activation, dropout=dropout, drop_start=drop_start, stateful=stateful, graph=graph,
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
    # chain kernel, one CTA per micro-batch
    "chain-one-4x32-tf32": _case(ONE_CTA, "chain-one-cta", 4, 32, precision="tf32"),
    "chain-one-17x8-stateful": _case(ONE_CTA, "chain-one-cta", 17, 8, stateful=True),
    # chain kernel, one launch per micro-batch, the weight gradients in one deferred wave
    "chain-per-mb-9x8-naive": _case(REF, "chain-per-mb", 9, 8, replay=True, eval_mu=9),
    "chain-per-mb-9x8-gpipe-gelu-drop": _case(REF, "chain-per-mb", 9, 8, sched="gpipe", **GELU_DROP),
    "chain-per-mb-9x8-pipedream-stateful-tf32": _case(REF, "chain-per-mb", 9, 8, sched="pipedream", stateful=True,
                                                     precision="tf32"),
    "chain-per-mb-17x8-gpipe": _case(REF, "chain-per-mb", 17, 8, sched="gpipe"),
    # layer-wise GEMMs over all micro-batches, SGD fused into the weight-gradient epilogue
    "layerwise-4x32": _case(REF, "layerwise", 4, 32, replay=True, eval_mu=1),
    "layerwise-17x8-gelu-drop-stateful-tf32": _case(REF, "layerwise", 17, 8, stateful=True, precision="tf32",
                                                    **GELU_DROP),
    # layer-wise GEMMs per micro-batch: weight gradients accumulate through memory, then a separate SGD pass
    "layerwise-per-mb-9x8-tf32-ce-eager": _case(REF, "layerwise-per-mb", 9, 8, precision="tf32", loss="cross_entropy",
                                                graph=False),
    "layerwise-per-mb-17x8-stateful": _case(REF, "layerwise-per-mb", 17, 8, sched="gpipe", stateful=True, replay=True),
    # wide layers: split-K forward and dgrad GEMMs
    "splitk-3x32-stateful": _case(SPLITK, "splitk", 3, 32, stateful=True),
}
REPLAYS = [n for n, c in CASES.items() if c["replay"]]
EVALS = [n for n, c in CASES.items() if c["eval_mu"] is not None]
WORST = {}                    # (form, precision) -> (worst err / bound, where)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for (form, precision), (v, what) in sorted(WORST.items()):
        print(f"[steps] worst err/bound {form:>16} {precision}: {v:.3g} ({what})")


def _bits(t):
    return t.detach().float().contiguous().cpu().view(torch.int32)


def _bit_equal(a, b):
    return torch.equal(_bits(a), _bits(b))


def _blocks(model, flat):
    """The [out, in + 1] blocks (W | bias) of a flat weight arena, in fp64 on the CPU."""
    out = []
    for i, (o, k) in enumerate(model.arena.blocks):
        off, ld = model.arena.offsets[i], model.arena.lds[i]
        out.append(flat[off:off + o * ld].view(o, ld)[:, : k + 1].double().cpu())
    return out


def _head(loss):
    return ce_head_oracle if loss == "cross_entropy" else head_oracle


# ================================================================================================== the per-step checks
def check_step(eng, model, c, st):
    """Every check of one step that just ran, from ``eng``'s buffers.  ``st``: the step's index ``i``, inputs ``x`` /
    ``t`` and those of the step before (``x_prev`` / ``t_prev``, None at step 0), ``lr``, dropout step ``dstep``, the
    flat weights ``W0`` and momentum ``V0`` (None: plain rule) before it, the loss the engine reported and the staging
    set ``fill`` it was filled into.  Returns {check: max err / bound}."""
    n_mu, mb, precision, i = c["n_mu"], c["mb"], c["precision"], st["i"]
    rows, L = n_mu * mb, len(model.linears)
    in_dim, out_dim = model.linears[0].in_dims, model.linears[-1].out_dims
    rtol = RTOL[precision]
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

    # ---- every layer of every micro-batch: forward, gates, dropped elements, dgrad
    res = check_layers(eng, model, st["W0"], st["x"], n_mu, mb, precision, st["lr"],
                       lambda mu: mu * mb + torch.arange(mb), step=st["dstep"], check_update=False)
    act = [st["x"].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
    dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
    blocks = _blocks(model, st["W0"])

    # ---- non-vacuity
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

    # ---- the update at this step's rate
    lr, stateful = st["lr"], st["V0"] is not None
    per_mb_wgrad = c["form"] == "layerwise-per-mb"
    W1 = model.arena.weights.detach()
    V1 = model.arena.momentum.detach() if stateful else None
    blocks1 = _blocks(model, W1)
    vblocks0 = _blocks(model, st["V0"]) if stateful else None
    vblocks1 = _blocks(model, V1) if stateful else None
    for l in range(1, L + 1):
        if stateful or per_mb_wgrad:
            if per_mb_wgrad:       # one wgrad GEMM per micro-batch accumulating into G: n_mu - 1 more fp32 roundings
                g, gb = grad_oracle(dz[l], act[l - 1], rtol_for(precision, mb))
                mag, _ = grad_oracle(dz[l].abs(), act[l - 1].abs(), 0.0)
                gb = gb + (n_mu - 1) * FP32_ULP * mag
            else:
                g, gb = grad_oracle(dz[l], act[l - 1], rtol_for(precision, rows))
            mu_, wd, nest = (MU, WD, True) if stateful else (0.0, 0.0, False)
            v0 = vblocks0[l - 1] if stateful else torch.zeros_like(blocks[l - 1])
            Wr, bW, Vr, bV = sgd_oracle(g, gb, blocks[l - 1], v0, lr, mu_, wd, nest)
            res[f"upd{l}"] = excess(blocks1[l - 1], Wr, bW)
            if stateful:
                res[f"mom{l}"] = excess(vblocks1[l - 1], Vr, bV)
        else:
            ref, bound = rows_update_oracle(dz[l], act[l - 1], blocks[l - 1], lr, rtol)
            res[f"upd{l}"] = excess(blocks1[l - 1] - blocks[l - 1], ref, bound)
        k = model.arena.blocks[l - 1][1]
        assert bool(model.arena.block(l - 1)[:, k + 1:].isnan().all()), f"{what}: the padding of layer {l}'s weights changed"
    if lr == 0.0:                      # the parameters only: a NaN in the padding may come back with other bits
        for l in range(L):
            assert _bit_equal(blocks1[l], blocks[l]), f"{what}: lr 0 changed the weights of layer {l + 1}"
            if stateful:
                assert not _bit_equal(vblocks1[l], vblocks0[l]), f"{what}: layer {l + 1}'s momentum stood still at lr 0"

    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, (what, bad)
    key = (c["form"], precision)
    worst = max(res, key=res.get)
    if c["form"] in FORMS and res[worst] > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (res[worst], f"{worst} at {what} of {c['name']}")
    return res


def check_eval(veng, model, W, x, t, n_mu, mb, precision, loss, count):
    """The evaluation engine's forward per layer from its own act[l - 1] at the flat weights ``W``, its probabilities
    per micro-batch, and ``count`` against argmax(probs) == argmax(t) over the rows (first maximum wins)."""
    rtol, L = RTOL[precision], len(model.linears)
    blocks = _blocks(model, W)
    act = [x.double()] + [_gather(lambda mu, l=l: veng.act(mu, l), n_mu) for l in range(1, L + 1)]
    res = {}
    for l, lin in enumerate(model.linears, start=1):
        Wl, b = blocks[l - 1][:, :-1], blocks[l - 1][:, -1]
        if lin.activation is not None:
            (ref, bound), _, _ = act_fwd_oracle(model.activation, act[l - 1], Wl, b, None, 1.0, rtol)
        else:
            ref, bound = fwd_oracle(act[l - 1], Wl, b, False, rtol)
        res[f"eval-fwd{l}"] = excess(act[l], ref, bound)
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
    """Initial weights, momentum and the batches of case ``name``, from a generator of its own."""
    c = CASES[name]
    sizes, rows = c["sizes"], c["n_mu"] * c["mb"]
    gen = _gen("steps", name)
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(STEPS)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
          for _ in range(STEPS)]
    Ws, bs = _init_weights(sizes, xs[0], c["n_mu"], gen, c["activation"], far=c["activation"] != "relu")
    Vs = [torch.randn(o, i + 1, generator=gen) * V_SCALE for i, o in zip(sizes[:-1], sizes[1:])]
    xv = torch.randn(rows, sizes[0], generator=gen)
    tv = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    return dict(xs=xs, ts=ts, Ws=Ws, bs=bs, Vs=Vs, xv=xv, tv=tv)


def _trainer(name, state, monkeypatch, graph=None):
    """A Trainer of case ``name`` in its initial state, NaN in every padding column, on the path the case names
    (``graph``: overrides the case's use of CUDA graphs)."""
    from shallowspeed_b200.parallel.engine import Trainer

    c = CASES[name]
    for k in FORMS[c["form"]]:
        monkeypatch.setenv(k, "1")
    sizes, n_mu, mb = c["sizes"], c["n_mu"], c["mb"]
    rule = dict(momentum=MU, weight_decay=WD, nesterov=True) if c["stateful"] else {}
    tr = Trainer(sizes, global_batch_size=n_mu * mb, n_mubatches=n_mu, lr=BUILD_LR, schedule=c["sched"],
                 precision=c["precision"], loss=c["loss"], activation=c["activation"], dropout=c["dropout"],
                 dropout_seed=DROP_SEED, use_graph=c["graph"] if graph is None else graph, **rule)
    model, eng = tr.model, tr.engine
    for i, (W, b) in enumerate(zip(state["Ws"], state["bs"])):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
        if c["stateful"]:
            model.arena.momentum_block(i)[:, : W.shape[1] + 1] = state["Vs"][i].cuda()
    _assert_path(eng, c)
    rows = n_mu * mb
    _poison(eng, model, sizes, rows, True, gated=c["activation"] != "relu")
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
    mus = {int(m) for m in re.findall(r"mu=(\d+)", text)}
    assert mus == (set(range(c["n_mu"])) if form.endswith("per-mb") else mus & {0}), (mus, text)


def _train_step(tr, c, i, x, t):
    """Step ``i`` as train.py runs it: the optimizer's rate and the model's dropout step set before the worker's step."""
    tr.optimizer.lr = LRS[i]
    tr.model.dropout_step = c["drop_start"] + i
    tr.worker.step_from(tr.schedule, x, t)


_RECORDS = {}


def _checked_run(name, monkeypatch):
    """The case's six steps, each checked by ``check_step`` right after it; returns the weights after every step, the
    final momentum and the loss of every step."""
    c = dict(CASES[name], name=name)
    state = _state(name)
    tr = _trainer(name, state, monkeypatch)
    eng, model = tr.engine, tr.model
    xh = [x.pin_memory() for x in state["xs"]]
    th = [t.pin_memory() for t in state["ts"]]
    rec = dict(W=[], losses=[])
    for i in range(STEPS):
        W0 = model.arena.weights.detach().clone()
        V0 = model.arena.momentum.detach().clone() if c["stateful"] else None
        fill = eng.fill_set()
        _train_step(tr, c, i, xh[i], th[i])
        loss = float(eng.last_loss())
        torch.cuda.synchronize()
        st = dict(i=i, x=state["xs"][i], t=state["ts"][i], x_prev=state["xs"][i - 1] if i else None,
                  t_prev=state["ts"][i - 1] if i else None, lr=LRS[i], dstep=c["drop_start"] + i, W0=W0, V0=V0,
                  loss=loss, fill=fill)
        check_step(eng, model, c, st)
        if c["activation"] != "relu":
            for l in range(1, len(c["sizes"]) - 1):
                pad = _pitched(eng.gate(0, l), c["n_mu"] * c["mb"])[:, c["sizes"][l]:]
                assert bool(pad.isnan().all()), f"step {i} layer {l}: a kernel wrote into the gate's padding"
        rec["W"].append(model.arena.weights.detach().cpu().clone())
        rec["losses"].append(loss)
    rec["V"] = model.arena.momentum.detach().cpu().clone() if c["stateful"] else None
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
    replayed from its graphs (the same kernels in the same order).  Weights, momentum and losses equal the checked
    run's."""
    rec = _record(name, monkeypatch)
    c = CASES[name]
    assert c["graph"]
    state = _state(name)
    for mode in ("async", "pipelined", "eager"):
        tr = _trainer(name, state, monkeypatch, graph=mode != "eager")
        if mode == "eager":
            xh = [x.pin_memory() for x in state["xs"]]
            th = [t.pin_memory() for t in state["ts"]]
            losses = []
            for i in range(STEPS):
                _train_step(tr, c, i, xh[i], th[i])
                losses.append(float(tr.engine.last_loss()))
            want = rec["losses"]
        elif mode == "async":
            xd = [x.cuda() for x in state["xs"]]
            td = [t.cuda() for t in state["ts"]]
            for i in range(STEPS):
                tr.optimizer.lr = LRS[i]
                tr.step_async(xd[i], td[i])
            tr.synchronize()
            losses = [float(tr.loss())]
            want = rec["losses"][-1:]
        else:
            xh = [x.pin_memory() for x in state["xs"]]
            th = [t.pin_memory() for t in state["ts"]]
            lagged = []
            for i in range(STEPS):
                tr.optimizer.lr = LRS[i]
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
        assert [_bits(torch.tensor(v)) for v in losses] == [_bits(torch.tensor(v)) for v in want], (mode, losses, want)
        del tr


@pytest.mark.gpu
@pytest.mark.parametrize("name", EVALS)
def test_evaluation_between_training_steps(name, monkeypatch):
    """train.py's evaluation engine (``NativeWorker(..., share=worker)``, ``InferenceSchedule``) between two training
    steps, nothing synchronised until the end: the training run is bitwise the checked one, and the evaluation reads the
    weights of the step before it."""
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import InferenceSchedule

    rec = _record(name, monkeypatch)
    c = CASES[name]
    state = _state(name)
    tr = _trainer(name, state, monkeypatch)
    rows, n_ev = c["n_mu"] * c["mb"], c["eval_mu"]
    val = Dataset(None, rows, rows // n_ev, device="cuda")
    val.local_batch_size = rows
    val.from_arrays(state["xv"], state["tv"])
    vw = NativeWorker(None, None, tr.model, val, None, use_graph=c["graph"], precision=c["precision"], share=tr.worker)
    sched = InferenceSchedule(n_ev, 1, 0)
    veng = vw.engine_for(sched)                        # built (and synchronised) before the run
    assert veng.uses_chain() == c["form"].startswith("chain")
    _poison(veng, tr.model, c["sizes"], rows, False)
    torch.cuda.synchronize()
    xh = [x.pin_memory() for x in state["xs"]]
    th = [t.pin_memory() for t in state["ts"]]
    for i in range(STEPS):
        _train_step(tr, c, i, xh[i], th[i])
        if i == EVAL_AFTER:
            veng.reset_correct()
            vw.execute(sched, 0)
    tr.worker.synchronize()
    vw.synchronize()
    torch.cuda.synchronize()
    assert _bit_equal(tr.model.arena.weights, rec["W"][-1]), "the training run differs from the uninterrupted one"
    mb = rows // n_ev
    res = check_eval(veng, tr.model, rec["W"][EVAL_AFTER], state["xv"], state["tv"], n_ev, mb, c["precision"],
                     c["loss"], veng.count_correct())
    out0 = vw.output_buffers[0]
    assert out0.data_ptr() == veng.probs(0).data_ptr() and out0.shape == veng.probs(0).shape
    print(f"\n[steps] eval of {name} ({n_ev} micro-batches): " + " ".join(f"{k}={v:.2g}" for k, v in res.items()))


# ================================================================================================== CPU side
def _slot_writes(rates, build_lr):
    """Which steps must write their staging set's learning-rate slot (PipeEngine::run: one slot per set, rewritten
    only when it holds another value)."""
    held, out = [build_lr, build_lr], []
    for i, lr in enumerate(rates):
        out.append(held[i % 2] != lr)
        held[i % 2] = lr
    return out


def test_grid_reaches_every_branch():
    from shallowspeed_b200 import _C

    table = {"chain-cluster": {3, 4, 9, 17, 32, 128}, "chain-one-cta": {4, 17}, "chain-per-mb": {9, 17},
             "layerwise": {4, 17}, "layerwise-per-mb": {9, 17}, "splitk": {3}}
    counts = {f: set() for f in FORMS}
    feats = {k: set() for k in ("stateful", "gelu-drop", "ce", "eager")}
    scheds, tf32 = set(), 0
    for name, c in CASES.items():
        f, n_mu, mb = c["form"], c["n_mu"], c["mb"]
        counts[f].add(n_mu)
        layers = list(zip(c["sizes"][:-1], c["sizes"][1:]))
        eligible = _C.chain_eligible(layers, mb, c["sizes"][-1], True, c["precision"] == "fp32")
        assert eligible == (f != "splitk"), name                       # layer-wise REF runs layer-wise by SSB_NO_CHAIN
        if f in ("chain-cluster", "chain-one-cta"):
            cl = _C.chain_cluster_size(layers, True, True, True, True, False, False)
            ksplit = cl > 1 and -(-c["sizes"][0] // 32) > 4
            assert (cl, ksplit) == ((4, True) if f == "chain-cluster" else (1, False)), name
            assert _C.chain_cluster_budget(mb, cl, c["precision"] == "fp32")[0]
        if f == "splitk":
            assert c["sizes"] == WIDE["1000-1500-777"]
        if f == "chain-per-mb":
            scheds.add((c["sched"], n_mu))
        tf32 += c["precision"] == "tf32"
        if c["stateful"]:
            feats["stateful"].add(f)
        if c["activation"] == "gelu" and c["dropout"] == DROP_P:
            feats["gelu-drop"].add(f)
        if c["loss"] == "cross_entropy":
            feats["ce"].add(f)
        if not c["graph"]:
            feats["eager"].add(f)
        if c["replay"]:
            assert c["drop_start"] == 0, name                          # Trainer draws the masks of step _steps
            assert c["graph"], name                                    # the eager replay is the other plan walk
    assert counts == table, counts
    assert {("naive", 9), ("gpipe", 9), ("pipedream", 9), ("gpipe", 17)} <= scheds
    # more than 8 micro-batches (shared streams) in both per-micro-batch forms, more than 16 (the loss stride) in a
    # coalesced and a per-micro-batch form, and counts that are not powers of two
    assert all(max(counts[f]) > 8 for f in ("chain-per-mb", "layerwise-per-mb"))
    assert max(counts["chain-cluster"]) > 16 and max(counts["chain-per-mb"]) > 16
    assert any(n & (n - 1) for n in counts["chain-cluster"])
    assert abs(tf32 - len(CASES) / 3) <= 2, tf32
    assert feats["stateful"] == set(FORMS)
    assert {"chain-cluster", "chain-per-mb"} <= feats["gelu-drop"] and feats["gelu-drop"] & {"layerwise", "layerwise-per-mb"}
    assert feats["ce"] & {"chain-cluster", "chain-one-cta", "chain-per-mb"} and feats["ce"] & {"layerwise", "layerwise-per-mb"}
    assert feats["eager"] & {"chain-cluster", "chain-one-cta", "chain-per-mb"} and feats["eager"] & {"layerwise", "layerwise-per-mb"}
    assert any(c["drop_start"] > 0 and c["dropout"] > 0 for c in CASES.values())
    # each staging set runs at least two checked steps; an lr-0 step; a step whose set needs no slot write while the
    # other set changed in between
    assert STEPS >= 4
    assert 0.0 in LRS and all(float(torch.tensor(lr, dtype=torch.float32)) == lr for lr in LRS)
    writes = _slot_writes(LRS, BUILD_LR)
    assert any(not writes[i] and LRS[i - 1] != LRS[i] for i in range(2, STEPS)), writes
    # the replays: the bench-shaped reference case, a per-micro-batch and a layer-wise one; the evaluations: the chain
    # and the layer-wise form, once with 9 micro-batches
    assert "chain-ref-4x32" in REPLAYS and CASES["chain-ref-4x32"]["sizes"] == REF
    assert any(CASES[n]["form"].endswith("per-mb") for n in REPLAYS)
    assert any(CASES[n]["form"].startswith("layerwise") for n in REPLAYS)
    assert {CASES[n]["form"].split("-")[0] for n in EVALS} == {"chain", "layerwise"}
    assert {CASES[n]["eval_mu"] for n in EVALS} == {1, 9}
    assert 0 <= EVAL_AFTER < STEPS - 1


# ---------------------------------------------------------------- the checks against an emulated engine
EMU_SIZES = [12, 20, 18, 5]
EMU = dict(name="emulated", sizes=EMU_SIZES, form="emulated", n_mu=17, mb=2, precision="fp32", loss="mse",
           activation="relu", dropout=DROP_P, drop_start=7, stateful=True)
EMU_STEPS = 3
FAULTS = ("lr-of-previous-step", "mask-of-previous-step", "layer-1-wgrad-from-other-set", "targets-of-other-set",
          "momentum-restarted-in-set-1", "dgrad-from-micro-batch-8-back", "loss-without-micro-batches-16-up",
          "eval-one-step-stale", "count-against-other-set")


class _Emulated:
    """A pp = 1 training engine emulated in fp32 on the CPU, with the buffers ``check_step`` reads: two staging sets
    (NaN in the padding), act / dz / probs per micro-batch, the loss, and the model arena's weights and momentum,
    updated in place by the stateful rule.  ``fault`` makes it commit one of FAULTS."""

    def __init__(self, model, n_mu, mb, fault=None):
        self.model, self.n_mu, self.mb, self.fault = model, n_mu, mb, fault
        rows, i, o = n_mu * mb, model.in_dim, model.out_dim
        self.sets = []
        for _ in range(2):
            x, y = torch.zeros(rows, i + 3), torch.zeros(rows, o + 3)
            x[:, i:] = y[:, o:] = float("nan")
            self.sets.append((x, y))
        self.fill, self.prev_lr, self.a, self.d, self.p = 0, None, [], [], None

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

    def dz(self, mu, l):
        return self._rows(self.d[l], mu)

    def probs(self, mu):
        return self._rows(self.p, mu)

    def step(self, x, t, lr, dstep, i):
        from shallowspeed_b200.ops import functional as F

        m, f, n_mu, mb = self.model, self.fault, self.n_mu, self.mb
        s_set, o_set = self.sets[self.fill], self.sets[self.fill ^ 1]
        s_set[0][:, : x.shape[1]] = x
        s_set[1][:, : t.shape[1]] = t
        x, t = s_set[0][:, : x.shape[1]].clone(), s_set[1][:, : t.shape[1]].clone()
        if f == "targets-of-other-set":
            t = o_set[1][:, : t.shape[1]].clone()
        scale = torch.tensor(F.dropout_scale(m.dropout), dtype=torch.float32)
        samples = torch.arange(n_mu * mb)
        blocks = [m.arena.block(j)[:, : k + 1].clone() for j, (_, k) in enumerate(m.arena.blocks)]
        a = [x]
        for lin, B in zip(m.linears, blocks):
            z = a[-1] @ B[:, :-1].T + B[:, -1]
            if lin.activation is not None:
                keep = F.dropout_mask(m.dropout, m.dropout_seed, lin.dropout[2],
                                      dstep - 1 if f == "mask-of-previous-step" else dstep, samples, lin.out_dims)
                z = torch.where(keep, z.clamp_min(0.0) * scale, torch.zeros(()))
            a.append(z)
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
        for l in range(L, 1, -1):
            src = d[l].clone()
            if f == "dgrad-from-micro-batch-8-back":
                src[8 * mb:] = d[l][: (n_mu - 8) * mb]
            d[l - 1] = torch.where(a[l - 1] > 0, (src @ blocks[l - 1][:, :-1]) * scale, torch.zeros(()))
        d[0] = torch.zeros_like(x)
        self.loss = float(sum(losses[:16] if f == "loss-without-micro-batches-16-up" else losses))
        lr_used = self.prev_lr if f == "lr-of-previous-step" and self.prev_lr is not None else lr
        for j, (_, k) in enumerate(m.arena.blocks):
            a_in = o_set[0][:, : x.shape[1]] if f == "layer-1-wgrad-from-other-set" and j == 0 else a[j]
            g = torch.cat([d[j + 1].T @ a_in, d[j + 1].sum(0)[:, None]], 1)
            W, Vb = m.arena.block(j)[:, : k + 1], m.arena.momentum_block(j)[:, : k + 1]
            v0 = torch.zeros_like(Vb) if f == "momentum-restarted-in-set-1" and self.fill == 1 else Vb
            gp = g + WD * W
            v = MU * v0 + gp
            W -= lr_used * (gp + MU * v)
            Vb.copy_(v)
        self.a, self.d, self.prev_lr = a, d, lr
        self.fill ^= 1


class _EmulatedEval:
    """The inference engine emulated in fp32: act per layer, probs and count_correct of one forward at given weights."""

    def __init__(self, model, W, x, t, n_mu, mb, fault=None):
        from shallowspeed_b200.ops import functional as F

        self.mb = mb
        blocks = _blocks(model, W)
        a = [x]
        for lin, B in zip(model.linears, blocks):
            z = a[-1] @ B[:, :-1].float().T + B[:, -1].float()
            a.append(z.clamp_min(0.0) if lin.activation is not None else z)
        self.a = a
        self.p = torch.cat([F.softmax_ref(a[-1][mu * mb:(mu + 1) * mb]) for mu in range(n_mu)])
        targets = torch.zeros_like(t) if fault == "count-against-other-set" else t
        self.count = int((self.p.argmax(1) == targets.argmax(1)).sum())

    def act(self, mu, l):
        return self.a[l][mu * self.mb:(mu + 1) * self.mb]

    def probs(self, mu):
        return self.p[mu * self.mb:(mu + 1) * self.mb]


def _check_emulated(fault=None):
    """Three emulated steps of EMU, each through ``check_step``, then an evaluation after step 1 through
    ``check_eval``."""
    from shallowspeed_b200.models.mlp import MLP

    c = EMU
    n_mu, mb, sizes = c["n_mu"], c["mb"], c["sizes"]
    rows = n_mu * mb
    model = MLP(sizes, 0, 1, rows, dropout=c["dropout"], dropout_seed=DROP_SEED)
    model.arena.enable_momentum()
    gen = _gen("emulated")
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(EMU_STEPS)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
          for _ in range(EMU_STEPS)]
    Ws, bs = _init_weights(sizes, xs[0], n_mu, gen)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
        o, k = model.arena.blocks[i]
        model.arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen) * V_SCALE
        model.arena.block(i)[:, k + 1:] = float("nan")
    eng = _Emulated(model, n_mu, mb, fault)
    snaps = []
    for i in range(EMU_STEPS):
        W0, V0, fill = model.arena.weights.clone(), model.arena.momentum.clone(), eng.fill_set()
        dstep = c["drop_start"] + i
        eng.step(xs[i], ts[i], LRS[i], dstep, i)
        st = dict(i=i, x=xs[i], t=ts[i], x_prev=xs[i - 1] if i else None, t_prev=ts[i - 1] if i else None, lr=LRS[i],
                  dstep=dstep, W0=W0, V0=V0, loss=eng.loss, fill=fill)
        check_step(eng, model, c, st)
        snaps.append(model.arena.weights.clone())
    xv = torch.randn(rows, sizes[0], generator=gen)
    tv = torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
    j = 1
    veng = _EmulatedEval(model, snaps[j - 1] if fault == "eval-one-step-stale" else snaps[j], xv, tv, n_mu, mb, fault)
    check_eval(veng, model, snaps[j], xv, tv, n_mu, mb, c["precision"], c["loss"], veng.count)


def test_checks_accept_the_emulated_engine():
    _check_emulated()


@pytest.mark.parametrize("fault", FAULTS)
def test_checks_reject_injected_faults(fault):
    with pytest.raises(AssertionError):
        _check_emulated(fault)
