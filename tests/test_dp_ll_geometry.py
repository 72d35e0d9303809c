"""Host-side geometry of the LL two-shot data-parallel kernel (csrc/kernels/dp_ll.cu), checked without a GPU.

The kernel addresses two landing zones per replica with closed-form indices:

    llA[owner]: (((parity * dp + src) * n_tiles + tile) * rows_per_owner + row_in_slice) * 17 + line     (reduce-scatter hop)
    llC[rank] :  ((parity * n_tiles + tile) * 128 + row) * 17 + line                                       (all-gather hop)

This model re-derives them in Python for every (parity, src, tile, row, line) a step can touch and asserts that no two
writers ever hit the same line, that every line a reader polls is written by exactly one peer, and that everything stays
inside the allocation the DpContext makes (``dp_ll_zone_lines``)."""
import itertools

import pytest

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]


def _C():
    from shallowspeed_b200 import _C as mod

    return mod


def _tiles(sizes):
    C = _C()
    out = []
    for i, o in zip(sizes[:-1], sizes[1:]):
        out.append(C.dp_ll_tiles(i, o))
    return out


def test_tile_counts_of_the_reference_model():
    t = _tiles(SIZES)
    assert t == [25, 4, 4, 4, 4, 4, 4]          # in / 32 tiles per layer (out <= 128: one row of tiles)
    assert sum(t) == 49                          # + 4 chain CTAs: co-resident on 132 SMs


@pytest.mark.parametrize("dp", [2, 4, 8])
def test_landing_zone_indices_are_unique_and_in_bounds(dp):
    n_tiles = sum(_tiles(SIZES))
    zone = _C().dp_ll_zone_lines(dp, n_tiles)
    rpo = 128 // dp
    assert zone == 2 * n_tiles * 128 * 17
    for parity in (0, 1):
        # ---- reduce-scatter hop: writer = (src rank, tile, row, line) -> line index in llA[owner(row)]
        seen = {owner: set() for owner in range(dp)}
        for src, tile, row, line in itertools.product(range(dp), range(0, n_tiles, 7), range(128), (0, 7, 16)):
            owner = row // rpo
            if owner == src:
                continue                          # own rows stay in shared memory
            idx = (((parity * dp + src) * n_tiles + tile) * rpo + (row - owner * rpo)) * 17 + line
            assert 0 <= idx < zone
            assert idx not in seen[owner], "two writers for one LL line"
            seen[owner].add(idx)
        # reader side: owner r polls, for each of its rows, the lines of every OTHER source - all of them were written
        for r in range(dp):
            for src, tile, row_in_slice, line in itertools.product(range(dp), range(0, n_tiles, 7), range(rpo), (0, 7, 16)):
                if src == r:
                    continue
                idx = (((parity * dp + src) * n_tiles + tile) * rpo + row_in_slice) * 17 + line
                assert idx in seen[r]
        # ---- all-gather hop: the owner of a row writes it into llC of every other replica
        for rank in range(dp):
            got = set()
            for tile, row, line in itertools.product(range(0, n_tiles, 7), range(128), (0, 7, 16)):
                if row // rpo == rank:
                    continue
                idx = ((parity * n_tiles + tile) * 128 + row) * 17 + line
                assert 0 <= idx < zone and idx not in got
                got.add(idx)


def test_parity_halves_do_not_overlap():
    n_tiles = sum(_tiles(SIZES))
    for dp in (2, 4, 8):
        rpo = 128 // dp
        last_even = (((0 * dp + dp - 1) * n_tiles + n_tiles - 1) * rpo + rpo - 1) * 17 + 16
        first_odd = (((1 * dp + 0) * n_tiles + 0) * rpo + 0) * 17 + 0
        assert last_even < first_odd
