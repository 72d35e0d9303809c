"""The fused data-parallel kernels (``dp_ll_wgrad_kernel`` in ``csrc/kernels/dp_ll.cu``, ``fused_wgrad_dp_kernel`` and
``dp_reduce_sgd_kernel`` in ``csrc/kernels/fused_dp.cu``) on ONE GPU, per element against fp64, by running one replica
of a dp-way group and replaying its peers from memory.

Every peer-to-peer message of these protocols is data at a known address stamped with the step's epoch: LL lines
{value, epoch, value, epoch} in the landing zones llA / llC, partial tiles in the staging buffer, and the arrive / done
flags.  Before a step the test writes every message the dp - 1 peers would have sent to replica r into r's buffers.  The
real engine (``NativeWorker._build`` with a stand-in communicator of size dp and rank r) then runs rank r against peer
contexts that are plain allocations of this process (``DpContext.open_local_peers``).  After the step the test reads
back every message r sent into its peers' memory.  Every wait the kernels perform is satisfied before the launch, so
nothing depends on a second process.  At dp = 1 the flag protocol needs no replay: the replica is every tile's owner.

Decoys.  Every line and staging slot r must not read holds the current epoch and a NaN payload: the other parity half,
the own-source lines, rows past a layer's end, line 16 of tiles without a bias column, and staging slots nobody sends to
r.  Every arrive / done flag r does not set itself holds the epoch.  An addressing or parity fault then shows up as NaN
in a checked output instead of a bounded spin that ends in a trap.  The message model below derives every address from
the kernels' own formulas (``dp_ll.cu`` phases A / B / C, as ``test_dp_ll_geometry.py`` writes them down, and
``fused_dp.cu::stage_slot``); the CPU tests check that the lines and flags the peers send are exactly the ones r polls.

Oracle, per layer from the engine's own act / dz buffers (as ``test_gpu_chain.py``):
* r's own partial: ``grad_oracle`` of ``test_gpu_gemm.py``, ``[dz.T @ act | colsum(dz)]`` and its bound.  With
  per-micro-batch launches G accumulates through memory: one more fp32 rounding of the magnitude per added micro-batch.
* the reduced gradient of an element r owns is ``own partial + sum of the injected peer partials``, added by the
  kernel in fp32 in rank order 0, 1, .., dp - 1.  Each of the dp - 1 additions rounds a running sum whose magnitude is
  at most the sum of |partial| (|g| + bound covers the fp32 value of the own partial), so the bound of the sum grows by
  ``(dp - 1) * 2^-24 * sum |partial|``.
* the update: ``sgd_oracle`` of ``test_gpu_gemm.py``, plain or stateful (momentum 0.9, Nesterov, weight decay 5e-4).
Elements owned by a peer: under LL, bit-equal to the injected phase-C line (the copy path); under the two-shot flag
protocol, untouched by r; under one-shot, updated by r like its own.  The momentum must change exactly on the elements
``_C.dp_owner_map`` assigns to r (the map ``NativeWorker.optimizer_state`` assembles checkpoints with) and nowhere else.

The DP half of the replay is ``dp_setup`` / ``dp_prefill`` / ``dp_check``; ``test_gpu_pp_replay.py`` calls the same
functions to run a pipeline stage as one replica of a dp x pp layout, where the kernels read the stage's receive slots.

Not covered here, and left to ``test_gpu_multi.py``: concurrent peers, the single-copy atomicity of LL lines over
NVLink, and bit-identity across real replicas.
"""
import gc
import math
import zlib

import pytest
import torch

from test_gpu_chain import ATOL, FP32_ULP, RTOL, _gather, _init_weights, _poison, dgrad_oracle, excess, fwd_oracle, head_oracle
from test_gpu_gemm import U, grad_oracle, rtol_for, sgd_oracle

REF = [784, 128, 127, 126, 125, 124, 123, 10]     # the reference model: every layer narrow, in = 127 / 123 ragged
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]  # layer-wise GEMMs, two-shot for the > 2 MB layers
BIG = [4096, 4096, 10]                              # 2048 two-shot tiles against 120 CTAs: several tiles per CTA
LR, MU, WD = 0.5, 0.9, 5e-4
STEPS = 3                                           # the epoch parity alternates, the momentum carries over
NAN = float("nan")
MAX_CTAS = 120                                      # kFusedDpMaxCtas (pipe_engine.cpp)
WORST = {}


def _C():
    from shallowspeed_b200 import _C as mod

    return mod


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ================================================================================================== geometry mirrors
def flag_geometry(sizes, dp, two_shot=False, one_shot=False, wide_tiles=False):
    """Per layer (first layer first), the staging geometry DpContext builds (dp_context.cpp, dp_layer_geometry in
    fused_dp.cu): layers of <= 2 MB of gradient run one-shot with 32-wide tiles unless ``wide_tiles``; ``two_shot`` /
    ``one_shot`` force a protocol on every layer (SSB_DP_TWO_SHOT / SSB_DP_ONE_SHOT, the latter winning)."""
    out, stage_off, slot_base, tile_base = [], 0, 0, 0
    for i, o in zip(sizes[:-1], sizes[1:]):
        one = (i * o * 4 <= (2 << 20) and not two_shot) or one_shot
        bn = 64 if i >= 64 else (i + 31) // 32 * 32
        if one and not wide_tiles:
            bn = 32
        tm, tn = -(-o // 128), -(-i // bn)
        slots = tm * tn if one else -(-(tm * tn) // dp)
        out.append(dict(**{"in": i}, out=o, block_n=bn, n_tiles_m=tm, n_tiles_n=tn, slots=slots,
                        slot_floats=128 * bn + 128, stage_offset=stage_off, slot_flag_base=slot_base,
                        tile_flag_base=tile_base, one_shot=int(one)))
        stage_off += slots * (128 * bn + 128)
        slot_base += slots
        tile_base += tm * tn
    parity = -(-max(stage_off, 64) // 64) * 64
    for g in out:
        g.update(stage_parity_stride=parity, stage_src_stride=2 * parity, slots_per_src=max(slot_base, 1))
    return out


def ll_tiles(sizes):
    """[(layer, in, out, mt, nt)] in landing-zone order: dp_ll_plan numbers the deepest layer's tiles first, then row
    tiles, then 32-wide column tiles."""
    out = []
    for li in reversed(range(len(sizes) - 1)):
        i, o = sizes[li], sizes[li + 1]
        out += [(li, i, o, mt, nt) for mt in range(-(-o // 128)) for nt in range(-(-i // 32))]
    return out


# ================================================================================================== LL message model
def _tile_lines(o, mt, nt):
    """(row in tile, line) of every line of one tile: valid rows only; 17 lines per row with the bias column (nt 0)."""
    rows, lpr = min(128, o - 128 * mt), 17 if nt == 0 else 16
    return torch.arange(rows).repeat_interleave(lpr), torch.arange(lpr).repeat(rows)


def _fields(li, i, mt, nt, row, j, idx):
    return dict(idx=idx, layer=torch.full_like(j, li), m=128 * mt + row, k=torch.full_like(j, i),
                n=torch.where(j < 16, 32 * nt + 2 * j, torch.full_like(j, i)), bias=j == 16)


def _cat(parts):
    return {key: {f: torch.cat([p[f] for p in lst]) for f in lst[0]} for key, lst in parts.items()}


def ll_messages(tiles, dp, src, parity):
    """Every LL line replica ``src`` stores in one step, as {(zone, dst): fields}.  idx = line in dst's zone; (layer, m,
    n) = the element of the line's first value (n = in on the bias line); k = the layer's in.
    Phase A (llA of the row's owner): (((parity * dp + src) * n_tiles + tile) * rpo + row - owner * rpo) * 17 + line.
    Phase B (llC of every other replica, the rows src owns): ((parity * n_tiles + tile) * 128 + row) * 17 + line."""
    rpo, n_tiles, parts = 128 // dp, len(tiles), {}
    for t, (li, i, o, mt, nt) in enumerate(tiles):
        row, j = _tile_lines(o, mt, nt)
        owner = row // rpo
        for d in range(dp):
            if d == src:
                continue
            s = owner == d
            idx = (((parity * dp + src) * n_tiles + t) * rpo + row[s] - d * rpo) * 17 + j[s]
            parts.setdefault(("A", d), []).append(_fields(li, i, mt, nt, row[s], j[s], idx))
            s = owner == src
            idx = ((parity * n_tiles + t) * 128 + row[s]) * 17 + j[s]
            parts.setdefault(("C", d), []).append(_fields(li, i, mt, nt, row[s], j[s], idx))
    return _cat(parts)


def ll_polls(tiles, dp, rank, parity):
    """The lines replica ``rank`` polls in its own zones: phase B, its rows from every other source; phase C, every
    valid row it does not own."""
    rpo, n_tiles, a, c = 128 // dp, len(tiles), [], []
    for t, (_li, _i, o, mt, nt) in enumerate(tiles):
        row, j = _tile_lines(o, mt, nt)
        mine = row // rpo == rank
        for sr in range(dp):
            if sr != rank:
                a.append((((parity * dp + sr) * n_tiles + t) * rpo + row[mine] - rank * rpo) * 17 + j[mine])
        c.append(((parity * n_tiles + t) * 128 + row[~mine]) * 17 + j[~mine])
    return {"A": torch.cat(a), "C": torch.cat(c)}


def ll_prefill_lines(tiles, dp, rank, parity):
    """What the peers of ``rank`` send it in one step: {zone: (src, fields)}."""
    out = {"A": [], "C": []}
    for p in range(dp):
        if p == rank:
            continue
        msgs = ll_messages(tiles, dp, p, parity)
        for z in ("A", "C"):
            out[z].append((p, msgs[(z, rank)]))
    return out


def line_values(f, values):
    """(a, b, a_valid, b_valid) of the lines ``f`` from per-layer [out, in + 1] ``values``: (m, n) and (m, n + 1) on a
    pair line, (m, in) and 0 on the bias line; NaN where a column lies past in."""
    a = torch.full(f["idx"].shape, NAN, dtype=values[0].dtype)
    b = torch.full_like(a, NAN)
    for li in f["layer"].unique().tolist():
        s = f["layer"] == li
        V, m, n, k, bias = values[li], f["m"][s], f["n"][s], f["k"][s], f["bias"][s]
        va = bias | (n < k)
        vb = ~bias & (n + 1 < k)
        a[s] = torch.where(va, V[m, torch.where(va, n, 0)], torch.full_like(a[s], NAN))
        b[s] = torch.where(vb, V[m, torch.where(vb, n + 1, 0)], torch.where(bias, 0.0, NAN))
    a_valid = f["bias"] | (f["n"] < f["k"])
    b_valid = f["bias"] | (f["n"] + 1 < f["k"])
    return a, b, a_valid, b_valid


def write_lines(zone, f, values, epoch):
    """Store {a, epoch, b, epoch} at the lines ``f`` of ``zone`` (int32 [lines, 4])."""
    a, b, _, _ = line_values(f, [v.float() for v in values])
    zone[f["idx"], 0] = a.view(torch.int32)
    zone[f["idx"], 1] = epoch
    zone[f["idx"], 2] = b.view(torch.int32)
    zone[f["idx"], 3] = epoch


def decoy_zone(lines, epoch):
    z = torch.empty(lines, 4, dtype=torch.int32)
    z[:, 0] = z[:, 2] = torch.tensor(NAN).view(torch.int32)
    z[:, 1] = z[:, 3] = epoch
    return z


def check_lines(zone, f, ref, bound, epoch, what):
    """The lines ``f`` of ``zone``: both epoch words equal ``epoch``; the values against per-layer ``ref`` (``bound``
    None: bit for bit), the second value of a bias line exactly 0.  Returns the worst err / bound."""
    L = zone[f["idx"]]
    assert bool((L[:, 1] == epoch).all() and (L[:, 3] == epoch).all()), f"{what}: a line without this step's epoch"
    a, b = L[:, 0].contiguous().view(torch.float32), L[:, 2].contiguous().view(torch.float32)
    ra, rb, va, vb = line_values(f, ref)
    if bound is None:
        same = (a.view(torch.int32) == ra.float().view(torch.int32)) | ~va
        same &= (b.view(torch.int32) == rb.float().view(torch.int32)) | ~vb
        assert bool(same.all()), f"{what}: {int((~same).sum())} lines differ from the expected weights"
        return 0.0
    assert bool((b[f["bias"]] == 0).all()), f"{what}: the second value of a bias line is not 0"
    ba, bb, _, _ = line_values(f, bound)
    pair = vb & ~f["bias"]
    return max(excess(a[va], ra[va], ba[va]), excess(b[pair], rb[pair], bb[pair]))


def check_only(zone, f, epoch, what):
    """No line of ``zone`` outside ``f`` carries ``epoch``: nothing was written anywhere else."""
    hit = (zone[:, 1] == epoch) | (zone[:, 3] == epoch)
    want = torch.zeros_like(hit)
    want[f["idx"]] = True
    assert torch.equal(hit, want), f"{what}: {int((hit != want).sum())} lines written where no message belongs"


# ================================================================================================== flag message model
def flag_messages(geom, dp, src, parity):
    """Every partial tile replica ``src`` pushes in one step: dicts (layer, t, mt, nt, dst, base, arrive).  base =
    float offset of the slot in dst's staging buffer (fused_dp.cu::stage_slot): src * stage_src_stride + stage_offset
    + slot * slot_floats (+ parity * stage_parity_stride one-shot); slot = t one-shot, t / dp two-shot; owner t % dp.
    arrive = src * slots_per_src + slot_flag_base + slot in dst's arrive flags."""
    out = []
    for li, g in enumerate(geom):
        for t in range(g["n_tiles_m"] * g["n_tiles_n"]):
            slot = t if g["one_shot"] else t // dp
            for d in (range(dp) if g["one_shot"] else [t % dp]):
                base = (src * g["stage_src_stride"] + g["stage_offset"] + slot * g["slot_floats"]
                        + (parity * g["stage_parity_stride"] if g["one_shot"] else 0))
                out.append(dict(layer=li, t=t, mt=t // g["n_tiles_n"], nt=t % g["n_tiles_n"], dst=d, base=base,
                                arrive=src * g["slots_per_src"] + g["slot_flag_base"] + slot))
    return out


def flag_polls(geom, dp, rank):
    """Flags replica ``rank`` polls: arrive (every source, including itself) for the tiles it reduces, done for the
    two-shot tiles another replica owns."""
    arrive, done = set(), set()
    for g in geom:
        for t in range(g["n_tiles_m"] * g["n_tiles_n"]):
            if g["one_shot"] or t % dp == rank:
                slot = t if g["one_shot"] else t // dp
                arrive |= {s * g["slots_per_src"] + g["slot_flag_base"] + slot for s in range(dp)}
            elif not g["one_shot"]:
                done.add(g["tile_flag_base"] + t)
    return arrive, done


def flag_done_writes(geom, dp, rank):
    """done flags replica ``rank`` sets (in every replica, itself included): its two-shot tiles."""
    return {g["tile_flag_base"] + t for g in geom if not g["one_shot"]
            for t in range(g["n_tiles_m"] * g["n_tiles_n"]) if t % dp == rank}


def flag_prefill(geom, dp, rank, parity):
    """(arrive flags, done flags, slot messages) the peers of ``rank`` send it in one step."""
    msgs = [(p, m) for p in range(dp) if p != rank for m in flag_messages(geom, dp, p, parity) if m["dst"] == rank]
    done = set().union(*[flag_done_writes(geom, dp, p) for p in range(dp) if p != rank])
    return {m["arrive"] for _, m in msgs}, done, msgs


def _idx(flags):
    return torch.tensor(sorted(flags), dtype=torch.long)


def _slot(values, g, mt, nt, dtype=torch.float32):
    """[128, block_n] tile and [128] bias of the [out, in + 1] block ``values``, NaN past the layer's end."""
    bn, i, o = g["block_n"], g["in"], g["out"]
    tile = torch.full((128, bn), NAN, dtype=dtype)
    r1, c0 = min(128, o - 128 * mt), nt * bn
    c1 = min(bn, i - c0)
    tile[:r1, :c1] = values[128 * mt: 128 * mt + r1, c0: c0 + c1]
    bias = torch.full((128,), NAN, dtype=dtype)
    if nt == 0:
        bias[:r1] = values[128 * mt: 128 * mt + r1, i]
    return tile, bias


# ================================================================================================== the oracle
def reduced_oracle(g, gb, peers):
    """own partial (g, bound) + the peer partials, summed in fp32 in rank order: (ref, bound), fp64."""
    ref, mag = g.clone(), g.abs() + gb
    for p in peers:
        ref += p.double()
        mag += p.double().abs()
    return ref, gb + len(peers) * U * mag


def check_momentum_ownership(V0, V1, owned, what):
    """V of the [out, in + 1] block changed on the owned elements and on no other.  ``mu * v + g`` can round back to
    v on a few owned elements (measured: 1 of the 1024 x 1001 of a tf32 layer); the oracle checks those per element, so here at most
    1e-4 of the owned elements may keep their bits."""
    changed = V0.view(torch.int32) != V1.view(torch.int32)
    stray, kept = int((changed & ~owned).sum()), int((owned & ~changed).sum())
    assert stray == 0 and kept <= 1e-4 * int(owned.sum()), \
        f"{what}: momentum changed on {stray} elements another replica owns, unchanged on {kept} it owns"


def _grad_scale(sizes, Ws, x, t, n_mu, batch):
    """Per layer, the mean |weight gradient| of a plain fp64 backward pass: the scale of the injected peer partials."""
    L, acts = len(sizes) - 1, [x.double()]
    for l in range(L):
        acts.append(fwd_oracle(acts[-1], Ws[l][:, :-1], Ws[l][:, -1], l < L - 1, 0.0)[0])
    mb = x.shape[0] // n_mu
    dz = torch.cat([head_oracle(acts[L][mu * mb:(mu + 1) * mb], t[mu * mb:(mu + 1) * mb], batch, 0.0)[1][0]
                    for mu in range(n_mu)])
    out = [None] * L
    for l in range(L, 0, -1):
        out[l - 1] = float(torch.cat([dz.T @ acts[l - 1], dz.sum(0)[:, None]], 1).abs().mean())
        if l > 1:
            dz = dgrad_oracle(dz, Ws[l - 1][:, :-1], acts[l - 1], 0.0)[0]
    return out


def _note(case, res):
    worst = max(res, key=res.get)
    WORST[case] = res[worst]
    print(f"\n[dp-replay] {case}: max err/bound {res[worst]:.3g} ({worst})")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, (case, bad)


@pytest.fixture(scope="module", autouse=True)
def _worst_table():
    yield
    for case, v in WORST.items():
        print(f"[dp-replay] worst err/bound {v:.3g}  {case}")


# ================================================================================================== the replica
def _device_view(ptr_bytes, typestr):
    ptr, nbytes = ptr_bytes

    class _Buf:
        __cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": typestr, "data": (ptr, False), "version": 3,
                                    "strides": None}

    return torch.as_tensor(_Buf(), device="cuda")


class _Buffers:
    """Device tensors over one DpContext's buffers."""

    def __init__(self, ctx):
        b = ctx.buffers()
        self.W, self.stage = _device_view(b["W"], "<f4"), _device_view(b["stage"], "<f4")
        self.arrive, self.done = _device_view(b["arrive"], "<i4"), _device_view(b["done"], "<i4")
        self.epoch = _device_view(b["epoch"], "<i4")
        self.llA = _device_view(b["llA"], "<i4").view(-1, 4) if b["llA"][1] else None
        self.llC = _device_view(b["llC"], "<i4").view(-1, 4) if b["llC"][1] else None


class _StandInComm:
    """A DP communicator of size dp and rank r that never communicates: the peers are replayed from memory."""

    def __init__(self, size, rank):
        self.size, self.rank = size, rank

    def Get_size(self):
        return self.size

    def Get_rank(self):
        return self.rank


def _build_replica(sizes, dp, rank, mb_rows, n_mu, precision, stateful, monkeypatch):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E

    rows = mb_rows * n_mu
    model = MLP(sizes, 0, 1, rows * dp).to("cuda")
    rule = dict(momentum=MU, weight_decay=WD, nesterov=True) if stateful else {}
    opt = SGD(model.parameters(), LR, arena=model.arena, **rule)
    ctxs = []
    make_dp_context = local_dp_context(ctxs)
    monkeypatch.setattr(E, "make_dp_context", make_dp_context)

    class _Shape:
        mubatch_size = mb_rows

    comm = _StandInComm(dp, rank)
    w = E.NativeWorker(comm, None, model, _Shape(), opt, comm_mode="fused", precision=precision)
    if dp == 1:
        # NativeWorker gives a lone replica no DP transport (it needs none); install the fused one to run the flag
        # protocol with the replica as the owner of every tile
        w.dp_mode = "fused"
        w._dp_ctx = make_dp_context(comm, model, w.lr)
    return w, model, ctxs


def local_dp_context(ctxs):
    """A ``make_dp_context`` whose peers are DpContexts of this process (``open_local_peers``) instead of CUDA IPC
    mappings; every context of the group lands in ``ctxs``, rank order."""
    def make_dp_context(comm, model, lr):
        arena = model.arena
        layers = [(lin.in_dims, lin.out_dims, int(arena.offsets[lin.block_index]), int(arena.lds[lin.block_index]))
                  for lin in model.linears]
        ctxs[:] = [_C().DpContext(comm.size, p, int(arena.weights.numel()), layers, float(lr)) for p in range(comm.size)]
        ctx = ctxs[comm.rank]
        ctx.open_local_peers(ctxs)
        arena.rebind(ctx.weights(), arena.grads, copy=True)
        torch.cuda.synchronize()
        return ctx

    return make_dp_context


def dp_setup(ctxs, rank, protocol, sizes, env, arena, protos):
    """What ``dp_prefill`` / ``dp_check`` need about replica ``rank`` of the group ``ctxs``: device views of every
    context's buffers, the LL tiles (``protocol`` "ll") or the flag geometry of the layers ``sizes``, and per layer the
    owner map of the protocol it ran (``protos``) and the elements ``rank`` owns."""
    C = _C()
    dp = len(ctxs)
    d = dict(dp=dp, rank=rank, ll=protocol == "ll", bufs=[_Buffers(c) for c in ctxs], protos=protos)
    d["me"] = d["bufs"][rank]
    if d["ll"]:
        d["tiles"] = ll_tiles(sizes)
    else:
        d["geom"] = flag_geometry(sizes, dp, two_shot="SSB_DP_TWO_SHOT" in env, one_shot="SSB_DP_ONE_SHOT" in env,
                                  wide_tiles="SSB_DP_WIDE_TILES" in env)
    d["owners"] = [C.dp_owner_map(int(protos[i]), k, o, int(arena.lds[i]), int(arena.offsets[i]), dp).long()
                   for i, (o, k) in enumerate(arena.blocks)]
    d["owned"] = [(ow == rank) | (ow < 0) for ow in d["owners"]]
    return d


def dp_peer_data(d, gen, blocks, scale, W0, lr):
    """What the peers contribute to one step: their partials ``P`` ([out, in + 1] per layer, of the magnitude
    ``scale``) and, under LL, the new weights ``Wc`` they send for their rows (phase C), an update's distance from the
    current ones."""
    P = {p: [(torch.randn(o, k + 1, generator=gen, dtype=torch.float64) * sc).float() for (o, k), sc in zip(blocks, scale)]
         for p in range(d["dp"]) if p != d["rank"]}
    Wc = {p: [(W0[i] - lr * torch.randn(o, k + 1, generator=gen, dtype=torch.float64) * scale[i]).float()
              for i, (o, k) in enumerate(blocks)] for p in P} if d["ll"] else {}
    return P, Wc


def dp_prefill(d, P, Wc, epoch):
    """Before a step of DP epoch ``epoch``: the peers' messages into my buffers (LL lines in llA / llC, or partial tiles
    in the staging buffer and arrive / done flags), decoys everywhere else, my outbound targets in the peers cleared."""
    dp, rank, me, bufs, parity = d["dp"], d["rank"], d["me"], d["bufs"], epoch & 1
    if d["ll"]:
        tiles = d["tiles"]
        lines = me.llA.shape[0]
        pre = ll_prefill_lines(tiles, dp, rank, parity)
        zones = {}
        for z, vals in (("A", P), ("C", Wc)):
            zone = decoy_zone(lines, epoch)
            for p, f in pre[z]:
                write_lines(zone, f, vals[p], epoch)
            zones[z] = zone
        polls = ll_polls(tiles, dp, rank, parity)
        for z in ("A", "C"):
            sent = torch.cat([f["idx"] for _, f in pre[z]]).sort().values
            assert torch.equal(sent, polls[z].sort().values), f"{z}: the prefill misses a polled line"
            assert bool((zones[z][polls[z], 1] == epoch).all() and (zones[z][polls[z], 3] == epoch).all())
        me.llA.copy_(zones["A"].cuda())
        me.llC.copy_(zones["C"].cuda())
        for p in P:
            bufs[p].llA.zero_()
            bufs[p].llC.zero_()
    else:
        geom = d["geom"]
        arrive_pre, done_pre, msgs = flag_prefill(geom, dp, rank, parity)
        polled_arrive, polled_done = flag_polls(geom, dp, rank)
        sps = geom[0]["slots_per_src"] if geom else 1      # a stage without layers keeps one arrive flag per source
        own_src = set(range(rank * sps, (rank + 1) * sps))
        assert arrive_pre == polled_arrive - own_src and done_pre == polled_done
        stage = torch.full_like(me.stage, NAN, device="cpu")
        for p, m in msgs:
            g = geom[m["layer"]]
            tile, bias = _slot(P[p][m["layer"]], g, m["mt"], m["nt"])
            stage[m["base"]: m["base"] + 128 * g["block_n"]] = tile.reshape(-1)
            stage[m["base"] + 128 * g["block_n"]: m["base"] + g["slot_floats"]] = bias
        arrive = torch.full(me.arrive.shape, epoch, dtype=torch.int32)
        arrive[_idx(own_src)] = 0
        done = torch.full(me.done.shape, epoch, dtype=torch.int32)
        done[_idx(flag_done_writes(geom, dp, rank))] = 0
        assert bool((arrive[_idx(arrive_pre)] == epoch).all()) and bool((done[_idx(done_pre)] == epoch).all())
        me.stage.copy_(stage.cuda())
        me.arrive.copy_(arrive.cuda())
        me.done.copy_(done.cuda())
        for p in P:
            bufs[p].stage.fill_(NAN)
            bufs[p].arrive.zero_()
            bufs[p].done.zero_()
    for p in P:
        bufs[p].W.fill_(NAN)


def check_owned_update(W1, own, own_b, peers, W0, V0, V1, lr, stateful, owned, res, key):
    """The owned elements of one layer's [out, in + 1] block after the step against ``reduced_oracle`` +
    ``sgd_oracle``: the weights' err / bound into ``res[key % "upd"]``, the momentum's (``stateful``) into
    ``res[key % "mom"]``."""
    tot, tb = reduced_oracle(own, own_b, peers)
    v0 = V0 if stateful else torch.zeros_like(W0)
    Wr, bW, Vr, bV = sgd_oracle(tot, tb, W0, v0, lr, MU if stateful else 0.0, WD if stateful else 0.0, stateful)
    res[key % "upd"] = excess(W1[owned], Wr[owned], bW[owned])
    if stateful:
        res[key % "mom"] = excess(V1[owned], Vr[owned], bV[owned])


def dp_check(d, res, step, arena, own, own_b, P, Wc, W0, V0, lr, stateful, epoch):
    """After a step of DP epoch ``epoch``, from my own partials ``own`` / ``own_b`` (the oracle of the engine's own act /
    dz): every owned update and momentum entry, every copied or untouched peer element, every outbound LL line or
    staging tile and arrive / done flag, the weights published to the peers, and the momentum ownership."""
    C = _C()
    dp, rank, bufs, protos, parity = d["dp"], d["rank"], d["bufs"], d["protos"], epoch & 1
    owners, owned = d["owners"], d["owned"]
    s = f"s{step + 1}."
    assert int(d["me"].epoch[0].item()) == epoch, "the DP epoch did not advance by one"
    # ---- 1. owned elements (and 2. for one-shot): per element against fp64
    W1 = [arena.block(i)[:, : k + 1].cpu() for i, (_, k) in enumerate(arena.blocks)]
    for i, (o, k) in enumerate(arena.blocks):
        pad = arena.block(i)[:, k + 1:]
        assert bool(torch.isnan(pad).all()), f"step {step + 1}: the padding of layer {i + 1}'s weights changed"
        V1 = arena.momentum_block(i)[:, : k + 1].cpu() if stateful else None
        check_owned_update(W1[i], own[i], own_b[i], [P[p][i] for p in P], W0[i], V0[i] if stateful else None, V1, lr,
                           stateful, owned[i], res, s + "%s" + str(i + 1))
        if stateful:
            check_momentum_ownership(V0[i].float(), V1, owned[i], f"step {step + 1} layer {i + 1}")
        # ---- 2. elements owned by peers
        for p in P:
            pm = owners[i] == p
            if d["ll"]:
                assert torch.equal(W1[i][pm].view(torch.int32), Wc[p][i][pm].view(torch.int32)), \
                    f"step {step + 1} layer {i + 1}: rows of rank {p} differ from its phase-C lines"
            else:
                assert torch.equal(W1[i][pm].view(torch.int32), W0[i][pm].float().view(torch.int32)), \
                    f"step {step + 1} layer {i + 1}: replica {rank} wrote a tile rank {p} owns"

    # ---- 3. outbound messages, read from the peers' buffers
    if d["ll"]:
        mine = ll_messages(d["tiles"], dp, rank, parity)
        for p in P:
            zA, zC = bufs[p].llA.cpu(), bufs[p].llC.cpu()
            res[s + "lineA"] = max(res.get(s + "lineA", 0.0),
                                   check_lines(zA, mine[("A", p)], own, own_b, epoch, f"phase A to {p}"))
            check_lines(zC, mine[("C", p)], W1, None, epoch, f"phase C to {p}")
            check_only(zA, mine[("A", p)], epoch, f"llA of {p}")
            check_only(zC, mine[("C", p)], epoch, f"llC of {p}")
        for p in P:
            assert bool(torch.isnan(bufs[p].W).all()), f"the LL kernel wrote into the weights of {p}"
        return
    geom = d["geom"]
    sent = [m for m in flag_messages(geom, dp, rank, parity)]
    pub = flag_done_writes(geom, dp, rank)
    for p in range(dp):
        stage_p, arrive_p, done_p = bufs[p].stage.cpu(), bufs[p].arrive.cpu(), bufs[p].done.cpu()
        to_p = [m for m in sent if m["dst"] == p]
        want = torch.zeros_like(arrive_p, dtype=torch.bool)
        want[_idx(m["arrive"] for m in to_p)] = True
        got = arrive_p == epoch
        if p == rank:
            assert bool(got[want].all()), "an own-source arrive flag was not set"
            assert bool((done_p[_idx(pub)] == epoch).all()), "a done flag of an owned tile was not set"
            continue
        assert torch.equal(got, want) and bool((arrive_p[~want] == 0).all()), f"arrive flags of {p}"
        dwant = torch.zeros_like(done_p, dtype=torch.bool)
        dwant[_idx(pub)] = True
        assert torch.equal(done_p == epoch, dwant) and bool((done_p[~dwant] == 0).all()), f"done flags of {p}"
        written = torch.zeros_like(stage_p, dtype=torch.bool)
        for m in to_p:
            g = geom[m["layer"]]
            bn = g["block_n"]
            tile = stage_p[m["base"]: m["base"] + 128 * bn].view(128, bn)
            bias = stage_p[m["base"] + 128 * bn: m["base"] + g["slot_floats"]]
            rt, rb = _slot(own[m["layer"]], g, m["mt"], m["nt"], torch.float64)
            bt, bb = _slot(own_b[m["layer"]], g, m["mt"], m["nt"], torch.float64)
            v = ~torch.isnan(rt)
            res[s + "push"] = max(res.get(s + "push", 0.0), excess(tile[v], rt[v], bt[v]))
            written[m["base"]: m["base"] + 128 * bn] = True
            if m["nt"] == 0:
                v = ~torch.isnan(rb)
                res[s + "push"] = max(res[s + "push"], excess(bias[v], rb[v], bb[v]))
                written[m["base"] + 128 * bn: m["base"] + g["slot_floats"]] = True
        assert bool(torch.isfinite(stage_p[written]).all()), f"a pushed slot of {p} holds a non-finite value"
        assert bool(torch.isnan(stage_p[~written]).all()), f"the staging buffer of {p} was written outside the slots"
        # published weights: the two-shot tiles I own, bit for bit; nothing else
        Wp = bufs[p].W.cpu()
        touched = torch.zeros_like(Wp, dtype=torch.bool)
        for i, (o, k) in enumerate(arena.blocks):
            off, ld = int(arena.offsets[i]), int(arena.lds[i])
            blk, tb = Wp[off: off + o * ld].view(o, ld), touched[off: off + o * ld].view(o, ld)
            if protos[i] == C.DP_PROTO_TWO_SHOT:
                pm = owners[i] == rank
                tb[:, : k + 1] = pm
                assert torch.equal(blk[:, : k + 1][pm].view(torch.int32), W1[i][pm].view(torch.int32)), \
                    f"layer {i + 1}: the weights published to {p} differ from mine"
        assert bool(torch.isnan(Wp[~touched]).all()), f"weights of {p} written outside my published tiles"


def _run(case, sizes, dp, rank, protocol, env=None, mb_rows=32, n_mu=2, precision="fp32", stateful=False,
         monkeypatch=None, steps=STEPS):
    """Build replica ``rank`` of ``dp`` through NativeWorker, run ``steps`` steps with its peers replayed and check
    every owned update, every copied or untouched peer element, every outbound message and the momentum ownership."""
    from shallowspeed_b200.pipe import NaiveParallelSchedule

    C = _C()
    env = env or {}
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    L, rows = len(sizes) - 1, mb_rows * n_mu
    w, model, ctxs = _build_replica(sizes, dp, rank, mb_rows, n_mu, precision, stateful, monkeypatch)
    sched = NaiveParallelSchedule(n_mu, 1, 0)
    eng = w.engine_for(sched)
    arena = model.arena
    gen = _gen(case)
    xs = [torch.randn(rows, sizes[0], generator=gen) for _ in range(steps)]
    ts = [torch.nn.functional.one_hot(torch.randint(0, sizes[-1], (rows,), generator=gen), sizes[-1]).float()
          for _ in range(steps)]
    Ws, bs = _init_weights(sizes, xs[0], n_mu, gen)
    for i, (W, b) in enumerate(zip(Ws, bs)):
        arena.weight_view(i).copy_(W)
        arena.bias_view(i).copy_(b[None, :])
        if stateful:
            o, k = arena.blocks[i]
            arena.momentum_block(i)[:, : k + 1] = torch.randn(o, k + 1, generator=gen).cuda() * 1e-3

    # ---- the path this case is meant to exercise
    plan, protos = eng.plan_text(0), list(eng.layer_protocols())
    assert (f"momentum={MU:g}" in eng.describe()) == stateful, eng.describe()
    coalesced = "SSB_NO_COALESCE" not in env
    assert eng.coalesced() == coalesced
    d = dp_setup(ctxs, rank, protocol, sizes, env, arena, protos)
    if protocol == "ll":
        assert ctxs[rank].ll_tiles() == len(d["tiles"]) and eng.uses_chain()
        assert "dp_ll" in plan and "fused_wgrad_dp" not in plan and "dp_reduce_sgd" not in plan, plan
        assert ("bump_step" in plan) == (env.get("SSB_DP_GATE", "1") != "0"), plan
        assert protos == [C.DP_PROTO_LL] * L
    else:
        assert ctxs[rank].ll_tiles() == 0 and "dp_ll" not in plan, plan
        kernel = "fused_wgrad_dp" if coalesced else "dp_reduce_sgd"
        assert plan.count(f" {kernel} ") == L and ("fused_wgrad_dp" in plan) == coalesced, plan
        geom = d["geom"]
        got = ctxs[rank].layer_geometry()
        for g, h in zip(geom, got):
            assert all(g[key] == h[key] for key in g), (g, h)
        assert protos == [C.DP_PROTO_ALL if g["one_shot"] else C.DP_PROTO_TWO_SHOT for g in geom]
        want = protocol.split("+")
        assert ("one-shot" in want) == any(g["one_shot"] for g in geom), geom
        assert ("two-shot" in want) == any(not g["one_shot"] for g in geom), geom
        if "multi-tile" in want:
            assert max(g["n_tiles_m"] * g["n_tiles_n"] for g in geom) > MAX_CTAS
    _poison(eng, model, sizes, rows, True)

    res = {}
    for step in range(steps):
        epoch = int(d["me"].epoch[0].item()) + 1
        W0 = [arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(arena.blocks)]
        V0 = [arena.momentum_block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(arena.blocks)] if stateful else None
        scale = _grad_scale(sizes, W0, xs[step], ts[step], n_mu, model.batch_size)
        P, Wc = dp_peer_data(d, gen, arena.blocks, scale, W0, LR)
        torch.cuda.synchronize()
        dp_prefill(d, P, Wc, epoch)
        torch.cuda.synchronize()

        w.step_from(sched, xs[step].pin_memory(), ts[step].pin_memory())
        eng.synchronize()
        torch.cuda.synchronize()

        act = [xs[step].double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L)]
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"step {step + 1}: dz[{l}] is all zero"
        own, own_b = [], []
        for i, (o, k) in enumerate(arena.blocks):
            if coalesced:
                g, gb = grad_oracle(dz[i + 1], act[i], rtol_for(precision, rows))
            else:   # one wgrad GEMM per micro-batch accumulating into G: n_mu - 1 more fp32 roundings
                g, gb = grad_oracle(dz[i + 1], act[i], rtol_for(precision, mb_rows))
                mag, _ = grad_oracle(dz[i + 1].abs(), act[i].abs(), 0.0)
                gb = gb + (n_mu - 1) * FP32_ULP * mag
            own.append(g)
            own_b.append(gb)
        dp_check(d, res, step, arena, own, own_b, P, Wc, W0, V0, LR, stateful, epoch)
    _note(case, res)
    eng.synchronize()
    del eng, w
    gc.collect()
    torch.cuda.synchronize()


# ================================================================================================== GPU grid
# dp = 1, flag protocol: every owner is the replica itself
DP1 = {
    "ref-one-shot": (REF, "one-shot", {}, "fp32", False),
    "ref-one-shot-tf32": (REF, "one-shot", {}, "tf32", False),
    "ref-one-shot-stateful": (REF, "one-shot", {}, "fp32", True),
    "ref-wide-tiles": (REF, "one-shot", {"SSB_DP_WIDE_TILES": "1"}, "fp32", False),
    "ref-two-shot": (REF, "two-shot", {"SSB_DP_TWO_SHOT": "1"}, "fp32", False),
    "ref-no-bulk": (REF, "one-shot", {"SSB_DP_BULK": "0"}, "fp32", False),
    "ref-reduce-sgd": (REF, "one-shot", {"SSB_NO_COALESCE": "1"}, "fp32", False),
    "ref-reduce-sgd-two-shot-stateful": (REF, "two-shot", {"SSB_NO_COALESCE": "1", "SSB_DP_TWO_SHOT": "1"}, "fp32", True),
    "wide": (WIDE, "one-shot+two-shot", {}, "fp32", False),
    "wide-tf32-stateful": (WIDE, "one-shot+two-shot", {}, "tf32", True),
    "wide-two-shot-no-bulk": (WIDE, "two-shot", {"SSB_DP_TWO_SHOT": "1", "SSB_DP_BULK": "0"}, "fp32", False),
    "wide-reduce-sgd": (WIDE, "one-shot+two-shot", {"SSB_NO_COALESCE": "1"}, "fp32", False),
    "big-multi-tile": (BIG, "one-shot+two-shot+multi-tile", {}, "fp32", False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DP1))
def test_dp1_flag_protocol(name, monkeypatch):
    sizes, proto, env, precision, stateful = DP1[name]
    _run(f"dp1 {name}", sizes, 1, 0, proto, env=env, precision=precision, stateful=stateful, monkeypatch=monkeypatch)


# LL replay: rows per owner 64 / 32 / 16, kLB 9 / 5 / 3
LL_RANKS = [(2, 0), (2, 1), (4, 0), (4, 2), (4, 3), (8, 0), (8, 3), (8, 7)]
LL_CASES = [(dp, r, gate, "fp32", False) for dp, r in LL_RANKS for gate in ("1", "0")]
LL_CASES += [(4, 1, "1", "tf32", False), (8, 5, "1", "fp32", True), (2, 1, "0", "fp32", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("dp,rank,gate,precision,stateful", LL_CASES)
def test_ll_replay(dp, rank, gate, precision, stateful, monkeypatch):
    _run(f"ll dp{dp} r{rank} gate{gate} {precision}{' stateful' if stateful else ''}", REF, dp, rank, "ll",
         env={"SSB_DP_GATE": gate}, mb_rows=128 // dp // 4, n_mu=4, precision=precision, stateful=stateful,
         monkeypatch=monkeypatch)


# flag-protocol replay at dp 2 / 4
# (the wide model at dp 4 once: its staging buffers make it the slowest case)
FLAG_CASES = [(sizes, dp, r, shot, st) for sizes in ("ref", "wide") for dp in (2, 4) for r in (0, 1)
              for shot in ("one-shot", "two-shot") for st in (False, True)
              if (not st or (dp, r) in ((2, 1), (4, 0))) and (sizes == "ref" or dp == 2)]
FLAG_CASES.append(("wide", 4, 1, "two-shot", False))


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,dp,rank,shot,stateful", FLAG_CASES)
def test_flag_replay(sizes, dp, rank, shot, stateful, monkeypatch):
    env = {"SSB_DP_LL": "0", "SSB_DP_ONE_SHOT" if shot == "one-shot" else "SSB_DP_TWO_SHOT": "1"}
    _run(f"flags {sizes} dp{dp} r{rank} {shot}{' stateful' if stateful else ''}", {"ref": REF, "wide": WIDE}[sizes], dp,
         rank, shot, env=env, stateful=stateful, monkeypatch=monkeypatch)


# ================================================================================================== CPU side
def _grid_ll():
    return sorted({(dp, r) for dp, r, *_ in LL_CASES})


def _grid_flags():
    """(sizes, dp, rank, geometry switches) of every flag-protocol case of the GPU grid."""
    out = [({"ref": REF, "wide": WIDE}[sz], dp, r, dict(one_shot=shot == "one-shot", two_shot=shot == "two-shot"))
           for sz, dp, r, shot, _st in FLAG_CASES]
    for sizes, _proto, env, _p, _s in DP1.values():
        out.append((sizes, 1, 0, dict(two_shot="SSB_DP_TWO_SHOT" in env, wide_tiles="SSB_DP_WIDE_TILES" in env)))
    return out


@pytest.mark.parametrize("dp,rank", _grid_ll())
def test_ll_prefill_covers_exactly_the_polled_lines(dp, rank):
    check_ll_prefill(REF, dp, rank)


def check_ll_prefill(sizes, dp, rank):
    """For both parities: the lines the peers send to ``rank`` are exactly the ones it polls, each once; none of them
    is a line it writes itself, and they stay inside the landing zone DpContext allocates."""
    tiles = ll_tiles(sizes)
    zone = _C().dp_ll_zone_lines(dp, len(tiles))
    for parity in (0, 1):
        pre = ll_prefill_lines(tiles, dp, rank, parity)
        polls = ll_polls(tiles, dp, rank, parity)
        mine = ll_messages(tiles, dp, rank, parity)
        assert all(d != rank for _z, d in mine)                         # nothing of mine lands in my own zones
        for z in ("A", "C"):
            sent = torch.cat([f["idx"] for _, f in pre[z]])
            assert sent.unique().numel() == sent.numel(), "two peers write one line"
            assert torch.equal(sent.sort().values, polls[z].sort().values)
            # (a replica whose rows lie past every layer's end, rank 1 of dp 2 on 48-wide layers, polls no phase-A line)
            assert sent.numel() == 0 or (int(sent.min()) >= parity * zone // 2 and int(sent.max()) < (parity + 1) * zone // 2)
        # every valid row of every tile is either mine (phase B) or arrives in phase C, exactly once
        rows = sum(min(128, o - 128 * mt) * (17 if nt == 0 else 16) for _l, _i, o, mt, nt in tiles)
        n_mine = sum(f["idx"].numel() for key, f in mine.items() if key[0] == "C") // (dp - 1)
        assert polls["C"].numel() + n_mine == rows


@pytest.mark.parametrize("case", range(len(_grid_flags())))
def test_flag_prefill_covers_exactly_the_polled_flags(case):
    sizes, dp, rank, switches = _grid_flags()[case]
    check_flag_prefill(sizes, dp, rank, switches)


def check_flag_prefill(sizes, dp, rank, switches):
    """The arrive / done flags the peers set for ``rank`` are exactly the ones it polls but does not set itself, the
    slots they guard do not overlap, and they stay inside the buffers DpContext allocates."""
    geom = flag_geometry(sizes, dp, **switches)
    for parity in (0, 1):
        arrive, done, msgs = flag_prefill(geom, dp, rank, parity)
        polled_arrive, polled_done = flag_polls(geom, dp, rank)
        sps = geom[0]["slots_per_src"] if geom else 1
        own_src = set(range(rank * sps, (rank + 1) * sps))
        mine = flag_messages(geom, dp, rank, parity)
        assert {m["arrive"] for m in mine if m["dst"] == rank} == polled_arrive & own_src
        assert arrive == polled_arrive - own_src and done == polled_done
        assert not (done & flag_done_writes(geom, dp, rank))
        spans = sorted((m["base"], m["base"] + geom[m["layer"]]["slot_floats"]) for _, m in msgs)
        assert all(a1 <= b0 for (_, a1), (b0, _) in zip(spans, spans[1:])), "two slots overlap"
        assert all(0 <= a and b <= dp * geom[0]["stage_src_stride"] for a, b in spans)
        assert all(0 <= f < dp * sps for f in arrive) and all(0 <= f < sum(g["n_tiles_m"] * g["n_tiles_n"] for g in geom)
                                                              for f in done)


def _emulated_ll_replica(seed=0):
    """A correct replica r = 1 of dp = 4 on a small model, emulated in fp32 on the CPU: returns everything the GPU test
    compares, so that faults can be injected into it."""
    sizes, dp, rank, epoch = [70, 40, 130, 10], 4, 1, 7
    parity, g = epoch & 1, torch.Generator().manual_seed(seed)
    tiles = ll_tiles(sizes)
    blocks = [(o, i) for i, o in zip(sizes[:-1], sizes[1:])]
    rpo = 128 // dp
    own = [torch.randn(o, k + 1, generator=g, dtype=torch.float64) * 1e-2 for o, k in blocks]
    own_b = [RTOL["fp32"] * a.abs() + ATOL for a in own]
    P = {p: [(torch.randn(o, k + 1, generator=g) * 1e-2) for o, k in blocks] for p in range(dp) if p != rank}
    W0 = [torch.randn(o, k + 1, generator=g, dtype=torch.float64) for o, k in blocks]
    V0 = [torch.randn(o, k + 1, generator=g, dtype=torch.float64) * 1e-3 for o, k in blocks]
    Wc = {p: [(w + 1e-3 * torch.randn(w.shape, generator=g, dtype=torch.float64)).float() for w in W0] for p in P}
    owner = [(torch.arange(o)[:, None] % 128 // rpo).expand(o, k + 1) for o, k in blocks]
    W1, V1 = [], []
    for i, (o, k) in enumerate(blocks):
        tot = own[i].float()
        for p in sorted(P):
            tot = tot + P[p][i]
        v = MU * V0[i].float() + tot + WD * W0[i].float()
        w_new = W0[i].float() - LR * (tot + WD * W0[i].float() + MU * v)
        mine = owner[i] == rank
        w1 = W0[i].float().clone()
        w1[mine] = w_new[mine]
        for p in P:
            w1[owner[i] == p] = Wc[p][i][owner[i] == p]
        W1.append(w1)
        V1.append(torch.where(mine, v, V0[i].float()))
    out_lines = {}
    for (z, d), f in ll_messages(tiles, dp, rank, parity).items():
        zone = out_lines.setdefault(d, {"A": torch.zeros(_C().dp_ll_zone_lines(dp, len(tiles)), 4, dtype=torch.int32),
                                        "C": torch.zeros(_C().dp_ll_zone_lines(dp, len(tiles)), 4, dtype=torch.int32)})
        write_lines(zone[z], f, [a.float() for a in own] if z == "A" else W1, epoch)
    return dict(sizes=sizes, dp=dp, rank=rank, epoch=epoch, parity=parity, tiles=tiles, blocks=blocks, own=own,
                own_b=own_b, P=P, W0=W0, V0=V0, Wc=Wc, owner=owner, W1=W1, V1=V1, out=out_lines)


def _check_emulated(e):
    """The GPU test's checks, applied to an emulated replica."""
    mine = ll_messages(e["tiles"], e["dp"], e["rank"], e["parity"])
    res = {}
    for i, (o, k) in enumerate(e["blocks"]):
        tot, tb = reduced_oracle(e["own"][i], e["own_b"][i], [e["P"][p][i] for p in e["P"]])
        Wr, bW, Vr, bV = sgd_oracle(tot, tb, e["W0"][i], e["V0"][i], LR, MU, WD, True)
        m = e["owner"][i] == e["rank"]
        res[f"upd{i}"] = excess(e["W1"][i][m], Wr[m], bW[m])
        res[f"mom{i}"] = excess(e["V1"][i][m], Vr[m], bV[m])
        check_momentum_ownership(e["V0"][i].float(), e["V1"][i], m, f"layer {i}")
        for p in e["P"]:
            pm = e["owner"][i] == p
            assert torch.equal(e["W1"][i][pm].view(torch.int32), e["Wc"][p][i][pm].view(torch.int32)), "phase-C copy"
    for p in e["P"]:
        zA, zC = e["out"][p]["A"], e["out"][p]["C"]
        res[f"lineA{p}"] = check_lines(zA, mine[("A", p)], e["own"], e["own_b"], e["epoch"], f"phase A to {p}")
        check_lines(zC, mine[("C", p)], e["W1"], None, e["epoch"], f"phase C to {p}")
        check_only(zA, mine[("A", p)], e["epoch"], f"llA of {p}")
        check_only(zC, mine[("C", p)], e["epoch"], f"llC of {p}")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad


def test_checks_reject_injected_faults():
    """The oracle and the message checks accept an emulated correct replica and reject each plausible kernel fault."""
    e = _emulated_ll_replica()
    _check_emulated(e)
    mine = ll_messages(e["tiles"], e["dp"], e["rank"], e["parity"])
    own_rows = [e["owner"][i] == e["rank"] for i in range(len(e["blocks"]))]

    def faulty(mutate):
        f = _emulated_ll_replica()
        mutate(f)
        with pytest.raises(AssertionError):
            _check_emulated(f)

    p0 = sorted(e["P"])[0]

    def dropped(f):                      # a peer partial dropped from the owner's sum
        m = own_rows[0]
        f["W1"][0][m] = (f["W1"][0][m].double() - LR * (1 + MU) * f["P"][p0][0][m].double()).float()

    def twice(f):                        # a peer partial counted twice
        m = own_rows[1]
        f["W1"][1][m] = (f["W1"][1][m].double() + LR * (1 + MU) * f["P"][p0][1][m].double()).float()

    def wrong_parity(f):                 # phase-A lines sent to the other parity half
        other = ll_messages(f["tiles"], f["dp"], f["rank"], 1 - f["parity"])
        zone = torch.zeros_like(f["out"][p0]["A"])
        write_lines(zone, other[("A", p0)], [a.float() for a in f["own"]], f["epoch"])
        f["out"][p0]["A"] = zone

    def bias_row_off_by_one(f):          # the bias gradient of row m + 1 sent as row m's
        shifted = [torch.cat([a[:, :-1], torch.roll(a[:, -1:], -1, 0)], 1).float() for a in f["own"]]
        zone = torch.zeros_like(f["out"][p0]["A"])
        write_lines(zone, mine[("A", p0)], shifted, f["epoch"])
        f["out"][p0]["A"] = zone

    def momentum_on_peer_row(f):         # a momentum entry written on a row another replica owns
        r = int((f["owner"][2][:, 0] != f["rank"]).nonzero()[0])
        f["V1"][2][r, 3] += 1e-3

    def phase_c_wrong_row(f):            # a phase-C line copied into the next row
        pm = f["owner"][1] == p0
        r = int(pm[:, 0].nonzero()[0])
        f["W1"][1][r, :] = f["Wc"][p0][1][r + 1, :]

    def epoch_word(f):                   # one epoch word of one line wrong
        f["out"][p0]["C"][mine[("C", p0)]["idx"][5], 3] = f["epoch"] - 1

    for mutate in (dropped, twice, wrong_parity, bias_row_off_by_one, momentum_on_peer_row, phase_c_wrong_row,
                   epoch_word):
        faulty(mutate)


def test_geometry_mirror_matches_the_host_formulas():
    """The Python mirror of DpContext's geometry against the rules it restates: tile counts, slot counts, one-shot
    decisions and the owner map of the two-shot protocol."""
    C = _C()
    for sizes in (REF, WIDE, BIG):
        for dp in (1, 2, 4):
            geom = flag_geometry(sizes, dp)
            for g in geom:
                tiles = g["n_tiles_m"] * g["n_tiles_n"]
                assert g["one_shot"] == int(g["in"] * g["out"] * 4 <= 2 << 20)
                assert g["slots"] == (tiles if g["one_shot"] else -(-tiles // dp))
            for g in flag_geometry(sizes, dp, two_shot=True):
                tiles = g["n_tiles_m"] * g["n_tiles_n"]
                if dp > 1 and g["out"] <= 300:
                    ow = C.dp_owner_map(C.DP_PROTO_TWO_SHOT, g["in"], g["out"], g["in"] + 1, 0, dp).long()
                    for t in range(tiles):
                        mt, nt = divmod(t, g["n_tiles_n"])
                        c0, c1 = nt * g["block_n"], min((nt + 1) * g["block_n"], g["in"])
                        assert bool((ow[128 * mt: 128 * mt + 128, c0:c1] == t % dp).all())
                        if nt == 0:                                 # the bias rides with tile column 0
                            assert bool((ow[128 * mt: 128 * mt + 128, g["in"]] == t % dp).all())
    assert sum(C.dp_ll_tiles(i, o) for i, o in zip(REF[:-1], REF[1:])) == len(ll_tiles(REF)) == 49
    big = flag_geometry(BIG, 1)
    assert big[0]["n_tiles_m"] * big[0]["n_tiles_n"] == 2048 and not big[0]["one_shot"]
