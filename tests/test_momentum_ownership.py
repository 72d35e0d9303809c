"""Ownership of the sharded SGD momentum (CPU, host-side rule only): under every data-parallel protocol the owned sets
of the replicas partition each layer's parameter elements (weights and bias column) exactly once, and the protocols
that keep full copies give every replica everything."""
import pytest
import torch

from shallowspeed_b200.layers import MLP

SIZE_SETS = {"reference": [784, 128, 127, 126, 125, 124, 123, 10], "wide": [784, 1024, 1000, 1024, 520, 1024, 130, 10]}


def _C():
    from shallowspeed_b200 import _C

    return _C


def _param_mask(arena):
    m = torch.zeros(arena.numel, dtype=torch.bool)
    for i, (o, k) in enumerate(arena.blocks):
        m[arena.offsets[i]:arena.offsets[i] + o * arena.lds[i]].view(o, arena.lds[i])[:, : k + 1] = True
    return m


def _expected_owner(proto, C, k, o, ld, off, dp):
    """Independent statement of the rule (tile rows / tiles / float4 chunks) for one [out, in + 1] block."""
    m = torch.arange(o).view(o, 1).expand(o, k + 1)
    n = torch.arange(k + 1).view(1, k + 1).expand(o, k + 1)
    if proto == C.DP_PROTO_LL:
        return (m % 128) // (128 // dp)
    if proto == C.DP_PROTO_TWO_SHOT:
        block_n, _tm, tn, _s, _sf = C.dp_layer_geometry(k, o, dp, False)
        nt = torch.where(n >= k, torch.zeros_like(n), n // block_n)
        return ((m // 128) * tn + nt) % dp
    return ((off + m * ld + n) // 4) % dp


@pytest.mark.parametrize("sizes", list(SIZE_SETS), ids=list(SIZE_SETS))
@pytest.mark.parametrize("dp", [2, 4, 8])
@pytest.mark.parametrize("proto", ["LL", "TWO_SHOT", "NVLS"])
def test_owned_sets_partition_every_parameter(sizes, dp, proto):
    from shallowspeed_b200.parallel.engine import owned_elements

    C = _C()
    p = getattr(C, f"DP_PROTO_{proto}")
    model = MLP(SIZE_SETS[sizes], 0, 1, 128)
    arena = model.arena
    params = _param_mask(arena)
    masks = [owned_elements(arena, model.linears, [p] * len(model.linears), dp, r) for r in range(dp)]
    count = torch.stack(masks).sum(0)
    assert bool((count[params] == 1).all())                 # every parameter element exactly once
    assert int(count[~params].sum()) == 0                   # padding belongs to nobody
    assert all(int(mk.sum()) > 0 for mk in masks)           # every replica owns a share
    for lin in model.linears:
        i = lin.block_index
        o, k = arena.blocks[i]
        got = C.dp_owner_map(p, k, o, arena.lds[i], arena.offsets[i], dp).long()
        assert torch.equal(got, _expected_owner(p, C, k, o, arena.lds[i], arena.offsets[i], dp))


@pytest.mark.parametrize("dp", [1, 2, 8])
def test_replicated_protocols_give_every_rank_everything(dp):
    from shallowspeed_b200.parallel.engine import owned_elements

    C = _C()
    model = MLP(SIZE_SETS["reference"], 0, 1, 128)
    params = _param_mask(model.arena)
    for r in range(dp):
        mk = owned_elements(model.arena, model.linears, [C.DP_PROTO_ALL] * len(model.linears), dp, r)
        assert torch.equal(mk, params)
    # the canonical assembly takes shared entries (and padding) from rank 0 only: still exactly one contributor each
    canon = [owned_elements(model.arena, model.linears, [C.DP_PROTO_LL] * 3 + [C.DP_PROTO_ALL] * 4, max(dp, 2), r,
                            shared_to_rank0=True) for r in range(max(dp, 2))]
    assert bool((torch.stack(canon).sum(0) == 1).all())
