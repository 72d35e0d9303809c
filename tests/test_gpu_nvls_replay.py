"""The NVLS data-parallel kernel (``nvls_reduce_kernel`` in ``csrc/kernels/nvls_dp.cu``, ``--comm nvls``) on ONE GPU,
per element against fp64, by running one replica of a dp-way group against a team that lives in memory.

The kernel reaches the team in three places: the load-reduce of a gradient chunk, the store of the new chunk into
every replica and the flag add.  A local team (``NvlsContext.local`` + ``open_local``) runs the same kernel body with
these three as loads, stores and atomics on the members' unicast views.  The real engine (``NativeWorker._build`` with
``comm_mode="nvls"`` and a stand-in communicator of size dp and rank r) runs replica r; the peers are NvlsContexts of
this process.  Before every step the test writes the peers' gradients (partials at the scale of r's own), sets the peers'
weights to the step's weights, raises r's flag_in and flag_out by dp - 1 (the peers' arrivals: with r's own the wait
target ``epoch * dp`` is met) and sets the peers' flag words to a base value.

Checks, per element and per step, from the engine's own act / dz buffers:
* owned chunks (float4 chunk c with c % dp == r): the new weight against ``reduced_oracle`` (r's partial from
  ``grad_oracle`` + the peer partials, summed in fp32 in rank order) and ``sgd_oracle`` at the step's scheduled rate,
  plain or stateful (momentum 0.9, Nesterov, weight decay); every peer's weight equals r's bit for bit;
* other chunks: r's weights and every peer's untouched; the momentum changes exactly on the elements
  ``_C.dp_owner_map`` assigns to r under ``DP_PROTO_NVLS``; the EMA is ``ema_lerp_ref(E0, W1, alpha)`` bit for bit on
  owned chunks and untouched elsewhere;
* guards: the momentum and EMA arenas are views into larger buffers poisoned with a NaN past ``numel``, and the team's
  W and G between ``numel`` and ``numel_pad`` hold sentinels; none may change (the owners once ran to ``numel_pad``);
* protocol: r's flags end at ``epoch * dp``, each peer's two flag words grew by exactly one, the epoch advanced by one,
  ``cta_done`` is re-armed to 0, and ``layer_protocols()`` reports NVLS on every layer.

With NVLink multicast on the device, one case runs the production multicast kernel through a one-device team (the kernel
still runs as replica r of dp): ld_reduce returns the local gradients, so the oracle is r's partial alone.

Not covered here, and left to ``test_gpu_multi.py`` and the other multi-GPU files: concurrent replicas, the switch's own
reduction order and atomicity, and the file-descriptor exchange of ``make_nvls_context``.
"""
import gc
import os

import pytest
import torch

import test_gpu_dp_replay as DP
from test_gpu_chain import FP32_ULP, _gather, _init_weights, _poison, excess
from test_gpu_dp_replay import LR, MU, NAN, WD, _StandInComm, _device_view, _gen, check_momentum_ownership, reduced_oracle
from test_gpu_gemm import grad_oracle, rtol_for, sgd_oracle

REF, WIDE, BIG = DP.REF, DP.WIDE, DP.BIG
ODD = [784, 128, 10]            # arena of 102,752 floats: numel % 64 == 32, so numel_pad - numel = 32
STEPS = 3                       # both staging sets, the momentum and the EMA carry over
EMA_DECAY = 0.3                 # alpha 1 on the first step, 0.7 after it
GUARD = 256                     # poisoned floats past the momentum / EMA arenas
POISON = 0x7FE5A5A5             # a quiet NaN with a payload no arithmetic produces
W_TAIL, G_TAIL = 3.0, 1024.0    # sentinels of the team's W / G in [numel, numel_pad)
FLAG_BASE = 1000                # peer p's flag words before a step: FLAG_BASE + p
WORST = {}


def _C():
    from shallowspeed_b200 import _C as mod

    return mod


def _schedule():
    from shallowspeed_b200.lr_schedule import LRSchedule

    return LRSchedule(LR, "cosine", total_steps=STEPS + 1, warmup_steps=1, warmup_start_factor=0.5)


# ================================================================================================== mirrors
def numel_pad(numel):
    """NvlsContext's allocation length of W and of G: the arena rounded up to 64 floats."""
    return -(-numel // 64) * 64


def chunk_owner(numel, dp):
    """Per float of the arena, the replica whose owner loop reduces and updates it: chunk c = i // 4 goes to c % dp."""
    return (torch.arange(numel) // 4) % dp


def kernel_chunks(numel, dp, rank, threads):
    """The chunks replica ``rank``'s owner loop visits with ``threads`` threads in its grid: thread t runs i = t,
    t + threads, .. while c = i * dp + rank < numel / 4 (nvls_dp.cu)."""
    n4, out = numel // 4, []
    for t in range(min(threads, n4)):
        i = t
        while i * dp + rank < n4:
            out.append(i * dp + rank)
            i += threads
    return torch.tensor(sorted(out), dtype=torch.long)


def wait_target(dp, epoch):
    """What both waits of a launch of epoch ``epoch`` poll for: one arrival per replica and step."""
    return epoch * dp


def flag_prefill(dp, epoch):
    """r's flag_in and flag_out before the launch of epoch ``epoch``: its value after the previous launch plus the dp - 1
    peers' arrivals of this step.  r's own arrival then meets the wait."""
    return wait_target(dp, epoch - 1) + dp - 1


def _note(case, res):
    worst = max(res, key=res.get)
    WORST[case] = res[worst]
    print(f"\n[nvls-replay] {case}: max err/bound {res[worst]:.3g} ({worst})")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, (case, bad)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for case, v in WORST.items():
        print(f"[nvls-replay] worst err/bound {v:.3g}  {case}")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _poison_word():
    return torch.tensor([POISON], dtype=torch.int32).view(torch.float32)[0]


# ================================================================================================== the check
def nvls_check(e, res, s):
    """One step of replica ``e["rank"]`` against everything known before it.  ``e`` holds flat CPU tensors:
    W0 (numel_pad: every member's weights before), W1 / G0 / G1 / flag_in / flag_out per member in memory (a dict
    rank -> value), V0 / V1 / E0 / E1 over numel + GUARD (None without momentum / EMA), the per-layer blocks of r's own
    partial (own, own_b) and the peers' (P), the arena geometry, lr, alpha, epoch, epoch_after and cta_done."""
    C = _C()
    dp, rank, numel, pad = e["dp"], e["rank"], e["numel"], e["pad"]
    peers = sorted(p for p in e["W1"] if p != rank)
    # ---- protocol state
    assert e["epoch_after"] == e["epoch"], "the epoch did not advance by one"
    assert e["cta_done"] == 0, "cta_done was not re-armed"
    target = wait_target(dp, e["epoch"])
    assert e["flag_in"][rank] == target and e["flag_out"][rank] == target, \
        f"r's flags {e['flag_in'][rank]} / {e['flag_out'][rank]}, expected {target}"
    for p in peers:
        assert e["flag_in"][p] == FLAG_BASE + p + 1 and e["flag_out"][p] == FLAG_BASE + p + 1, \
            f"the flag words of {p} did not grow by exactly one"
    # ---- ownership: chunks, whole arena
    owned = torch.zeros(pad, dtype=torch.bool)
    owned[:numel] = chunk_owner(numel, dp) == rank
    W0, Wr = e["W0"], e["W1"][rank]
    assert torch.equal(_bits(Wr[~owned]), _bits(W0[~owned])), "r wrote a chunk it does not own (or past numel)"
    for p in peers:
        assert torch.equal(_bits(e["W1"][p][owned]), _bits(Wr[owned])), f"the weights of {p} differ from r's on its chunks"
        assert torch.equal(_bits(e["W1"][p][~owned]), _bits(W0[~owned])), f"r wrote a chunk of {p} it does not own"
    for m in e["G1"]:
        assert torch.equal(_bits(e["G1"][m][numel:]), _bits(e["G0"][m][numel:])), f"G of {m} changed past numel"
        if m != rank:
            assert torch.equal(_bits(e["G1"][m]), _bits(e["G0"][m])), f"reduce_sgd changed the gradients of {m}"
    # ---- per element: the owned update and momentum
    stateful = e["V0"] is not None
    for i, (o, k) in enumerate(e["blocks"]):
        off, ld = e["offsets"][i], e["lds"][i]

        def blk(flat):
            return flat[off: off + o * ld].view(o, ld)[:, : k + 1]

        own_el = C.dp_owner_map(C.DP_PROTO_NVLS, k, o, ld, off, dp).long() == rank
        assert torch.equal(own_el, blk(owned)), f"layer {i + 1}: dp_owner_map differs from the chunk owners"
        V0 = blk(e["V0"]).double() if stateful else None
        V1 = blk(e["V1"]) if stateful else None
        DP.check_owned_update(blk(Wr), e["own"][i], e["own_b"][i], [e["P"][p][i] for p in sorted(e["P"])],
                              blk(W0).double(), V0, V1, e["lr"], stateful, own_el, res, s + "%s" + str(i + 1))
        if stateful:
            check_momentum_ownership(V0.float(), V1, own_el, f"{s} layer {i + 1}")
    # ---- guards past the arena, the EMA
    for name in ("V", "E"):
        if e[name + "0"] is not None:
            a, b = e[name + "0"], e[name + "1"]
            assert torch.equal(_bits(b[numel:]), _bits(a[numel:])), f"{name}: written past the arena's {numel} floats"
    if e["E0"] is not None:
        from shallowspeed_b200.ops.functional import ema_lerp_ref

        E0, E1, o = e["E0"][:numel], e["E1"][:numel], owned[:numel]
        want = ema_lerp_ref(E0, Wr[:numel], e["alpha"])
        assert torch.equal(_bits(E1[o]), _bits(want[o])), "an owned EMA entry differs from lerp(E0, W1, alpha)"
        assert torch.equal(_bits(E1[~o]), _bits(E0[~o])), "the EMA moved on a chunk r does not own"


# ================================================================================================== the replica
class _Member:
    """Device tensors over one NvlsContext's buffers."""

    def __init__(self, ctx):
        b = ctx.buffers()
        self.W, self.G = _device_view(b["W"], "<f4"), _device_view(b["G"], "<f4")
        self.flag_in, self.flag_out = _device_view(b["flag_in"], "<i4"), _device_view(b["flag_out"], "<i4")
        self.epoch, self.cta_done = _device_view(b["epoch"], "<i4"), _device_view(b["cta_done"], "<i4")


def local_nvls_context(ctxs):
    """A ``make_nvls_context`` whose team is NvlsContexts of this process (``NvlsContext.local`` + ``open_local``);
    every member lands in ``ctxs``, rank order."""
    def make_nvls_context(comm, model, lr):
        arena = model.arena
        ctxs[:] = [_C().NvlsContext.local(comm.size, p, int(arena.weights.numel())) for p in range(comm.size)]
        ctx = ctxs[comm.rank]
        ctx.open_local(ctxs)
        arena.rebind(ctx.weights(), ctx.grads(), copy=True)
        torch.cuda.synchronize()
        return ctx

    return make_nvls_context


def one_device_nvls_context(ctxs):
    """A ``make_nvls_context`` that binds a multicast object of ONE device: the production kernel as replica r of dp,
    whose team is itself."""
    def make_nvls_context(comm, model, lr):
        arena = model.arena
        ctx = _C().NvlsContext(comm.size, comm.rank, int(arena.weights.numel()), float(lr), devices=1)
        fd = ctx.export_fd()
        ctx.add_device()
        ctx.bind_and_map()
        os.close(fd)
        ctxs[:] = [ctx]
        arena.rebind(ctx.weights(), ctx.grads(), copy=True)
        torch.cuda.synchronize()
        return ctx

    return make_nvls_context


def _guarded(t):
    """``t`` moved into a buffer GUARD floats longer, poisoned past it: (the view the engine gets, the whole buffer)."""
    big = torch.full((t.numel() + GUARD,), _poison_word().item(), dtype=torch.float32, device=t.device)
    big.view(torch.int32)[t.numel():] = POISON
    big[: t.numel()] = t
    return big[: t.numel()], big


def _run(case, sizes, dp, rank, precision="fp32", form="plain", n_mu=4, mb_rows=32, env=None, multicast=False,
         monkeypatch=None):
    """Build replica ``rank`` of ``dp`` through NativeWorker with ``comm_mode="nvls"``, run STEPS steps against the
    team and check each with ``nvls_check``.  form: "plain", "rule" (momentum, Nesterov, weight decay), "ema" (plain
    rule + EMA), "ema-rule"."""
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E
    from shallowspeed_b200.pipe import NaiveParallelSchedule

    C = _C()
    env = env or {}
    for key, v in env.items():
        monkeypatch.setenv(key, v)
    L, rows = len(sizes) - 1, mb_rows * n_mu
    stateful, ema = form in ("rule", "ema-rule"), form.startswith("ema")
    model = MLP(sizes, 0, 1, rows * dp).to("cuda")
    rule = dict(momentum=MU, weight_decay=WD, nesterov=True) if stateful else {}
    opt = SGD(model.parameters(), LR, arena=model.arena, ema_decay=EMA_DECAY if ema else None, **rule)
    ctxs = []
    monkeypatch.setattr(E, "make_nvls_context", (one_device_nvls_context if multicast else local_nvls_context)(ctxs))

    class _Shape:
        mubatch_size = mb_rows

    w = E.NativeWorker(_StandInComm(dp, rank), None, model, _Shape(), opt, comm_mode="nvls", precision=precision)
    arena = model.arena
    numel, pad = arena.numel, numel_pad(arena.numel)
    assert ctxs[0].numel_pad() == pad and ctxs[0].arena_numel() == numel
    gen = _gen(case)
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(STEPS)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
          for _ in range(STEPS)]
    Ws, bs = _init_weights(sizes, xs[0], n_mu, gen)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        arena.weight_view(i).copy_(W)
        arena.bias_view(i).copy_(b[None, :])
        if stateful:
            o, k = arena.blocks[i]
            arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen).cuda() * 1e-3
    # the engine takes the momentum / EMA arenas as views into poisoned, longer buffers
    Vbig = Ebig = None
    if stateful:
        arena.momentum, Vbig = _guarded(arena.momentum)
    if ema:
        arena.ema, Ebig = _guarded(arena.ema)

    sched = NaiveParallelSchedule(n_mu, 1, 0)
    eng = w.engine_for(sched)
    # ---- the path this case is meant to exercise
    plan = eng.plan_text(0)
    assert plan.count(" nvls_reduce_sgd ") == 1 and "dp_ll" not in plan and "fused_wgrad_dp" not in plan, plan
    assert list(eng.layer_protocols()) == [C.DP_PROTO_NVLS] * L
    coalesced = "SSB_NO_COALESCE" not in env
    assert eng.coalesced() == coalesced
    if sizes is REF:
        assert eng.uses_chain()
    elif sizes is WIDE:
        assert not eng.uses_chain()
    assert (f"momentum={MU:g}" in eng.describe()) == stateful, eng.describe()
    _poison(eng, model, sizes, rows, True)

    team = {p: _Member(c) for p, c in (enumerate(ctxs) if not multicast else [(rank, ctxs[0])])}
    me = team[rank]
    lrs = _schedule()
    blocks, offsets, lds = list(arena.blocks), [int(x) for x in arena.offsets], [int(x) for x in arena.lds]
    res = {}
    for step in range(STEPS):
        s = f"s{step + 1}."
        epoch = int(me.epoch[0].item()) + 1
        opt.lr = lrs.schedule(step)
        alpha = opt.ema_alpha if ema else None
        assert step == 0 or opt.lr != lrs.schedule(step - 1)
        W0b = [arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(blocks)]
        scale = DP._grad_scale(sizes, W0b, xs[step], ts[step], n_mu, model.batch_size)
        P = {p: [(torch.randn(o, k + 1, generator=gen, dtype=torch.float64) * sc).float() for (o, k), sc in
                 zip(blocks, scale)] for p in team if p != rank}
        torch.cuda.synchronize()
        me.W[numel:] = W_TAIL
        me.G[numel:] = G_TAIL
        W0 = me.W.cpu()
        G0 = {}
        for p in team:
            if p == rank:
                continue
            G = torch.zeros(pad)
            for i, (o, k) in enumerate(blocks):
                G[offsets[i]: offsets[i] + o * lds[i]].view(o, lds[i])[:, : k + 1] = P[p][i]
            G[numel:] = G_TAIL
            team[p].G.copy_(G.cuda())
            team[p].W.copy_(me.W)
            team[p].flag_in.fill_(FLAG_BASE + p)
            team[p].flag_out.fill_(FLAG_BASE + p)
            G0[p] = G
        for f in (me.flag_in, me.flag_out):
            assert int(f[0].item()) == wait_target(dp, epoch - 1)
            f += dp - 1
            assert int(f[0].item()) == flag_prefill(dp, epoch)
        V0 = Vbig.cpu() if stateful else None
        E0 = Ebig.cpu() if ema else None
        torch.cuda.synchronize()

        w.step_from(sched, xs[step].pin_memory(), ts[step].pin_memory())
        eng.synchronize()
        torch.cuda.synchronize()

        act = [xs[step].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L)]
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"step {step + 1}: dz[{l}] is all zero"
        G0[rank] = torch.cat([me.G[:numel].cpu(), torch.full((pad - numel,), G_TAIL)])
        own, own_b = [], []
        for i, (o, k) in enumerate(blocks):
            if precision == "bf16":
                from test_gpu_bf16 import grad_oracle_bf16 as oracle, rtol_bf16 as rtol_of
            else:
                oracle, rtol_of = grad_oracle, (lambda kk, p=precision: rtol_for(p, kk))
            if coalesced:
                g, gb = oracle(dz[i + 1], act[i], rtol_of(rows))
            else:   # one wgrad GEMM per micro-batch accumulating into G: n_mu - 1 more fp32 roundings
                g, gb = oracle(dz[i + 1], act[i], rtol_of(mb_rows))
                mag, _ = oracle(dz[i + 1].abs(), act[i].abs(), 0.0)
                gb = gb + (n_mu - 1) * FP32_ULP * mag
            res[s + f"grad{i + 1}"] = excess(arena.block(i, grads=True)[:, : k + 1].cpu(), g, gb)
            own.append(g)
            own_b.append(gb)
        e = dict(dp=dp, rank=rank, numel=numel, pad=pad, blocks=blocks, offsets=offsets, lds=lds, lr=opt.lr,
                 alpha=alpha, epoch=epoch, epoch_after=int(me.epoch[0].item()), cta_done=int(me.cta_done[0].item()),
                 W0=W0, W1={p: m.W.cpu() for p, m in team.items()}, G0=G0, G1={p: m.G.cpu() for p, m in team.items()},
                 flag_in={p: int(m.flag_in[0].item()) for p, m in team.items()},
                 flag_out={p: int(m.flag_out[0].item()) for p, m in team.items()},
                 V0=V0, V1=Vbig.cpu() if stateful else None, E0=E0, E1=Ebig.cpu() if ema else None,
                 own=own, own_b=own_b, P=P)
        nvls_check(e, res, s)
    _note(case, res)
    eng.synchronize()
    del eng, w
    gc.collect()
    torch.cuda.synchronize()


# ================================================================================================== GPU grid
# name: (sizes, dp, rank, precision, form, n_mu, env).  REF runs the chain kernel, WIDE the layer-wise GEMMs; ODD and
# BIG have numel % 64 == 32 (the overrun case); BIG at dp 8 gives each thread several grid-stride iterations.
NC = {"SSB_NO_COALESCE": "1"}
CASES = {
    "ref-dp2-r1-fp32-plain": (REF, 2, 1, "fp32", "plain", 4, {}),
    "ref-dp2-r0-tf32-rule": (REF, 2, 0, "tf32", "rule", 4, {}),
    "ref-dp4-r3-bf16-plain": (REF, 4, 3, "bf16", "plain", 4, {}),
    "ref-dp4-r1-fp32-ema": (REF, 4, 1, "fp32", "ema", 4, {}),
    "ref-dp8-r7-fp32-ema-rule": (REF, 8, 7, "fp32", "ema-rule", 4, {}),
    "ref-dp8-r2-tf32-rule-n1": (REF, 8, 2, "tf32", "rule", 1, {}),
    "ref-dp4-r2-fp32-rule-no-coalesce": (REF, 4, 2, "fp32", "rule", 4, NC),
    "odd-dp2-r1-fp32-rule": (ODD, 2, 1, "fp32", "rule", 4, {}),
    "odd-dp4-r3-bf16-ema-rule": (ODD, 4, 3, "bf16", "ema-rule", 4, {}),
    "odd-dp8-r7-tf32-ema-n1-no-coalesce": (ODD, 8, 7, "tf32", "ema", 1, NC),
    "wide-dp2-r0-fp32-rule": (WIDE, 2, 0, "fp32", "rule", 4, {}),
    "wide-dp4-r3-bf16-ema-rule-no-coalesce": (WIDE, 4, 3, "bf16", "ema-rule", 4, NC),
    "big-dp8-r7-fp32-ema-rule": (BIG, 8, 7, "fp32", "ema-rule", 2, {}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_nvls_replay(name, monkeypatch):
    sizes, dp, rank, precision, form, n_mu, env = CASES[name]
    _run(name, sizes, dp, rank, precision, form, n_mu=n_mu, env=env, monkeypatch=monkeypatch)


@pytest.mark.gpu
def test_nvls_multicast_one_device_team(monkeypatch):
    """The production multicast kernel (STATEFUL + EMA) through a multicast object of this one device."""
    C = _C()
    if not C.NvlsContext.supported():
        pytest.skip("this device / driver does not support NVLink multicast (CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED)")
    try:
        probe = C.NvlsContext(2, 1, 1024, 0.0, devices=1)
        os.close(probe.export_fd())
    except RuntimeError as err:
        pytest.skip(f"NVLink multicast is reported, but the driver refuses a multicast object of one device: {err}")
    del probe
    _run("multicast-one-device ref-dp2-r1-ema-rule", REF, 2, 1, "fp32", "ema-rule", multicast=True,
         monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("dp,rank", [(2, 0), (4, 1), (8, 7)])
def test_standalone_collectives_on_a_local_team(dp, rank):
    """``all_reduce_grads()`` and ``reduce_sgd(lr)``: on r's chunks, G of every member becomes the in-place sum of the
    members' G in rank order, bit for bit (W: W - lr * sum within one rounding of either order); nothing else changes,
    nothing past numel."""
    C = _C()
    numel = 102752 + 32 * rank                      # numel % 64 == 32 at rank 0, 0 at the others
    pad = numel_pad(numel)
    team = [C.NvlsContext.local(dp, p, numel) for p in range(dp)]
    team[rank].open_local(team)
    mem = [_Member(c) for c in team]
    gen = _gen("standalone", dp, rank)
    owned = torch.zeros(pad, dtype=torch.bool)
    owned[:numel] = chunk_owner(numel, dp) == rank
    lr_t = torch.tensor([0.375], device="cuda")
    for epoch, op in ((1, "all_reduce_grads"), (2, "reduce_sgd"), (3, "all_reduce_grads")):
        G = [torch.randn(pad, generator=gen) for _ in range(dp)]
        W = torch.randn(pad, generator=gen)
        for p, m in enumerate(mem):
            m.G.copy_(G[p].cuda())
            m.W.copy_(W.cuda())
            if p != rank:
                m.flag_in.fill_(FLAG_BASE + p)
                m.flag_out.fill_(FLAG_BASE + p)
        mem[rank].flag_in.add_(dp - 1)
        mem[rank].flag_out.add_(dp - 1)
        torch.cuda.synchronize()
        if op == "reduce_sgd":
            team[rank].reduce_sgd(lr_t)
        else:
            team[rank].all_reduce_grads()
        torch.cuda.synchronize()
        tot = G[0].clone()
        for g in G[1:]:
            tot += g                                  # fp32, rank order: the replay's sum
        for p, m in enumerate(mem):
            Gp, Wp = m.G.cpu(), m.W.cpu()
            if op == "all_reduce_grads":
                assert torch.equal(_bits(Gp[owned]), _bits(tot[owned])), f"{op}: G of {p} on r's chunks"
                assert torch.equal(_bits(Gp[~owned]), _bits(G[p][~owned])), f"{op}: G of {p} off r's chunks"
                assert torch.equal(_bits(Wp), _bits(W)), f"{op}: W of {p} changed"
            else:
                want = W.double() - 0.375 * tot.double()
                bound = 2.0**-23 * (W.double().abs() + 0.375 * tot.double().abs())
                assert excess(Wp[owned], want[owned], bound[owned]) <= 1.0, f"{op}: W of {p} on r's chunks"
                assert torch.equal(_bits(Wp[~owned]), _bits(W[~owned])), f"{op}: W of {p} off r's chunks"
                assert torch.equal(_bits(Gp), _bits(G[p])), f"{op}: G of {p} changed"
            if p != rank:
                assert int(m.flag_in[0].item()) == int(m.flag_out[0].item()) == FLAG_BASE + p + 1
        assert int(mem[rank].flag_in[0].item()) == int(mem[rank].flag_out[0].item()) == wait_target(dp, epoch)
        assert int(mem[rank].epoch[0].item()) == epoch and int(mem[rank].cta_done[0].item()) == 0


# ================================================================================================== CPU side
def _arena_geometry(sizes):
    """(blocks [(out, in)], offsets, lds, numel) of ParamArena for ``sizes``, without a device."""
    from shallowspeed_b200.models.layers import ParamArena

    arena = ParamArena([(o, i) for i, o in zip(sizes[:-1], sizes[1:])], device="cpu")
    return list(arena.blocks), [int(x) for x in arena.offsets], [int(x) for x in arena.lds], arena.numel


@pytest.mark.parametrize("sizes", [REF, ODD, WIDE, BIG, [520, 1024, 130], [130, 10]],
                         ids=["ref", "odd", "wide", "big", "wide-pp4-s2", "wide-pp4-s3"])
def test_owner_mirror_matches_dp_owner_map_and_the_kernel_loop(sizes):
    """The chunk owners against ``_C.dp_owner_map(DP_PROTO_NVLS)`` on every layer, and the chunks the owner loops of
    all replicas visit (at a grid of a few threads, so that each runs several grid-stride iterations): each chunk below
    numel / 4 exactly once, at its owner, none past it."""
    C = _C()
    blocks, offsets, lds, numel = _arena_geometry(sizes)
    assert numel % 32 == 0 and numel_pad(numel) - numel in (0, 32)
    for dp in (2, 4, 8):
        own = chunk_owner(numel, dp)
        for i, (o, k) in enumerate(blocks):
            got = C.dp_owner_map(C.DP_PROTO_NVLS, k, o, lds[i], offsets[i], dp).long()
            want = own[offsets[i]: offsets[i] + o * lds[i]].view(o, lds[i])[:, : k + 1]
            assert torch.equal(got, want), (sizes, dp, i)
        if numel <= 200000:
            seen = torch.cat([kernel_chunks(numel, dp, r, 7 * 256) for r in range(dp)])
            assert torch.equal(seen.sort().values, torch.arange(numel // 4))
            for r in range(dp):
                assert bool((kernel_chunks(numel, dp, r, 3 * 256) % dp == r).all())


def test_odd_arenas_are_in_the_grid():
    """The overrun case is reached: arenas whose padded length exceeds numel, at every dp of the grid."""
    assert _arena_geometry(ODD)[3] % 64 == 32 and _arena_geometry(BIG)[3] % 64 == 32
    assert _arena_geometry([520, 1024, 130])[3] % 64 == 32 and _arena_geometry([130, 10])[3] % 64 == 32
    odd = {CASES[n][1] for n in CASES if CASES[n][0] in (ODD, BIG)}
    assert odd == {2, 4, 8}


@pytest.mark.parametrize("dp", [2, 4, 8])
def test_flag_prefill_meets_each_wait_with_the_own_arrival(dp):
    """Before the launch of epoch e r's flags hold e * dp - 1 (the previous target plus the peers' arrivals); its own
    arrival meets the target exactly, and the value it leaves is what the next prefill starts from."""
    after = 0
    for epoch in range(1, 6):
        pre = flag_prefill(dp, epoch)
        assert pre == after + dp - 1 and pre < wait_target(dp, epoch) == pre + 1
        after = pre + 1
        assert after == epoch * dp


def _emulated(seed=0, stateful=True, ema=True):
    """A correct replica r = 2 of dp = 4 on a small model whose arena has numel % 64 == 32 ([30, 20, 12]), emulated in
    fp32 on the CPU, in the form ``nvls_check`` reads; faults are injected into it.  ``Wall``: the update on every
    chunk below numel, for faults that apply it where r does not own."""
    sizes, dp, rank, epoch = [30, 20, 12], 4, 2, 5
    blocks, offsets, lds, numel = _arena_geometry(sizes)
    pad = numel_pad(numel)
    assert pad - numel == 32
    g = torch.Generator().manual_seed(seed)
    lr, alpha = 0.25, 0.7
    own = [torch.randn(o, k + 1, generator=g, dtype=torch.float64) * 1e-2 for o, k in blocks]
    own_b = [2.0**-16 * a.abs() + 1e-30 for a in own]
    P = {p: [torch.randn(o, k + 1, generator=g) * 1e-2 for o, k in blocks] for p in range(dp) if p != rank}
    W0 = torch.full((pad,), NAN)
    W0[numel:] = W_TAIL
    Gs = {p: torch.zeros(pad) for p in range(dp)}
    for i, (o, k) in enumerate(blocks):
        sl = slice(offsets[i], offsets[i] + o * lds[i])
        W0[sl].view(o, lds[i])[:, : k + 1] = torch.randn(o, k + 1, generator=g)
        Gs[rank][sl].view(o, lds[i])[:, : k + 1] = own[i].float()
        for p in P:
            Gs[p][sl].view(o, lds[i])[:, : k + 1] = P[p][i]
    for p in Gs:
        Gs[p][numel:] = G_TAIL
    poison = _poison_word()
    V0 = torch.cat([torch.randn(numel, generator=g) * 1e-3, torch.full((GUARD,), float(poison))]) if stateful else None
    if V0 is not None:
        V0.view(torch.int32)[numel:] = POISON
    E0 = torch.cat([torch.randn(numel, generator=g), torch.zeros(GUARD)]) if ema else None
    if E0 is not None:
        E0.view(torch.int32)[numel:] = POISON
    tot = Gs[0].clone()
    for p in range(1, dp):
        tot = tot + Gs[p]
    owned = torch.zeros(pad, dtype=torch.bool)
    owned[:numel] = chunk_owner(numel, dp) == rank
    W1, V1 = W0.clone(), V0.clone() if stateful else None
    if stateful:
        gp = tot[:numel] + WD * W0[:numel]
        v = MU * V0[:numel] + gp
        wn = W0[:numel] - lr * (gp + MU * v)
        V1[:numel] = torch.where(owned[:numel], v, V0[:numel])
    else:
        wn = W0[:numel] - lr * tot[:numel]
    W1[:numel] = torch.where(owned[:numel], wn, W0[:numel])
    E1 = None
    if ema:
        from shallowspeed_b200.ops.functional import ema_lerp_ref

        E1 = E0.clone()
        E1[:numel] = torch.where(owned[:numel], ema_lerp_ref(E0[:numel], W1[:numel], alpha), E0[:numel])
    return dict(dp=dp, rank=rank, numel=numel, pad=pad, blocks=blocks, offsets=offsets, lds=lds, lr=lr, alpha=alpha,
                epoch=epoch, epoch_after=epoch, cta_done=0, W0=W0, W1={p: W1.clone() for p in range(dp)},
                G0={p: G.clone() for p, G in Gs.items()}, G1={p: G.clone() for p, G in Gs.items()},
                flag_in={p: wait_target(dp, epoch) if p == rank else FLAG_BASE + p + 1 for p in range(dp)},
                flag_out={p: wait_target(dp, epoch) if p == rank else FLAG_BASE + p + 1 for p in range(dp)},
                V0=V0, V1=V1, E0=E0, E1=E1, own=own, own_b=own_b, P=P, owned=owned,
                Wall=torch.cat([wn, W0[numel:]]))


def test_checks_accept_the_emulated_replica():
    for stateful in (False, True):
        for ema in (False, True):
            nvls_check(_emulated(stateful=stateful, ema=ema), {}, "s1.")
            res = {}
            nvls_check(_emulated(stateful=stateful, ema=ema), res, "s1.")
            assert res and max(res.values()) <= 1.0, res


def _first(mask, k=0):
    return int(mask.nonzero()[k])


def _wrong_stride(e):            # the owner loop strides by dp + 1: r updates chunks of others, misses some of its own
    n4, dp, r = e["numel"] // 4, e["dp"], e["rank"]
    wrong = torch.zeros(e["pad"], dtype=torch.bool)
    for c in range(r, n4, dp + 1):
        wrong[4 * c: 4 * c + 4] = True
    for p in e["W1"]:
        e["W1"][p] = torch.where(wrong, e["Wall"], e["W0"])


def _store_missing_from_a_peer(e):
    p = (e["rank"] + 1) % e["dp"]
    c = _first(e["owned"])
    e["W1"][p][c: c + 4] = e["W0"][c: c + 4]


def _applied_twice(e):
    rank, owned = e["rank"], e["owned"]
    i = _first(owned & ~torch.isnan(e["W0"]))
    d = e["W1"][rank][i] - e["W0"][i]
    for p in e["W1"]:
        e["W1"][p][i] = e["W1"][p][i] + d


def _ema_on_a_foreign_chunk(e):
    i = _first(~e["owned"][: e["numel"]] & ~torch.isnan(e["W0"][: e["numel"]]))
    e["E1"][i] = e["E1"][i] * 0.5 + e["W1"][e["rank"]][i] * 0.5


def _overrun(e):                 # the owners of the chunks in [numel, numel_pad) read and write V / E past the arena
    n, pad, dp, r = e["numel"], e["pad"], e["dp"], e["rank"]
    for c in range(n // 4, pad // 4):
        if c % dp == r:
            e["V1"][4 * c: 4 * c + 4] = NAN
            e["E1"][4 * c: 4 * c + 4] = NAN
            for p in e["W1"]:
                e["W1"][p][4 * c: 4 * c + 4] = W_TAIL - e["lr"] * e["dp"] * G_TAIL


def _overrun_guard_only(e):      # the same, seen in the momentum guard alone
    c = next(c for c in range(e["numel"] // 4, e["pad"] // 4) if c % e["dp"] == e["rank"])
    e["V1"][4 * c] = float("nan")


def _epoch_not_bumped(e):
    e["epoch_after"] = e["epoch"] - 1


def _flag_added_twice_to_a_peer(e):
    p = (e["rank"] + 1) % e["dp"]
    e["flag_out"][p] += 1


def _cta_done_not_rearmed(e):
    e["cta_done"] = 3


@pytest.mark.parametrize("fault,reason", [
    (_wrong_stride, "r wrote a chunk it does not own"), (_store_missing_from_a_peer, "differ from r's on its chunks"),
    (_ema_on_a_foreign_chunk, "the EMA moved on a chunk r does not own"),
    (_overrun, "r wrote a chunk it does not own (or past numel)"), (_overrun_guard_only, "V: written past the arena"),
    (_epoch_not_bumped, "the epoch did not advance"), (_flag_added_twice_to_a_peer, "did not grow by exactly one"),
    (_cta_done_not_rearmed, "cta_done was not re-armed")],
    ids=["wrong-owner-stride", "store-missing-from-a-peer", "ema-on-a-foreign-chunk",
         "overrun", "overrun-momentum-guard", "epoch-not-bumped", "flag-added-twice", "cta-done-not-rearmed"])
def test_checks_reject_injected_faults(fault, reason):
    """Each fault is rejected, and for the reason it stands for (the first check it breaks)."""
    e = _emulated()
    fault(e)
    with pytest.raises(AssertionError) as info:
        nvls_check(e, {}, "s1.")
    assert reason in str(info.value), str(info.value)


def test_update_applied_twice_is_caught_by_the_oracle():
    """An update applied twice keeps every bit-equality check (it lands in every member) and fails the per-element
    bound alone (without an EMA, which would also move away from lerp(E0, W1))."""
    e = _emulated(ema=False)
    _applied_twice(e)
    res = {}
    nvls_check(e, res, "s1.")
    assert max(res.values()) > 1.0 and max(res, key=res.get).startswith("s1.upd"), res
