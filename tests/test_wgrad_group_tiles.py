"""Host-side tiling of the grouped weight-gradient launch (pure C++ arithmetic, no GPU needed): every element of a
layer's [out, in] block belongs to exactly one tile, exactly one tile per feature tile owns the bias column, and the
shared memory plan lets several CTAs share an SM."""
import numpy as np
import pytest

from shallowspeed_b200 import _C

REF = [(784, 128), (128, 127), (127, 126), (126, 125), (125, 124), (124, 123), (123, 10)]
SMEM_PER_SM = 228 * 1024


@pytest.mark.parametrize("rows", [1, 8, 24, 100, 128, 512, 1024])
def test_tiles_cover_every_weight_once_and_one_tile_per_feature_tile_owns_the_bias(rows):
    for out in (1, 10, 31, 32, 33, 97, 127, 128):
        for inp in (1, 7, 31, 32, 33, 64, 65, 123, 784, 4096):
            tiles, stages, smem = _C.wgrad_group_tiles(out, inp, rows)
            hits = np.zeros((out, inp), dtype=np.int32)
            owners = {}
            for m0, n0, r, c, owns_bias in tiles:
                assert r == 32 and c in (32, 64) and m0 % r == 0 and n0 % c == 0
                assert m0 < out and n0 < inp                   # no tile lies wholly outside the block
                hits[m0:m0 + r, n0:n0 + c] += 1
                if owns_bias:
                    assert n0 + c >= inp                       # its tile store is the one that can reach the bias slot
                    owners[m0] = owners.get(m0, 0) + 1
            assert (hits == 1).all(), (out, inp, rows)
            assert owners == {m0: 1 for m0 in range(0, out, 32)}, (out, inp, rows)
            num_kb = -(-rows // 32)
            assert 1 <= stages <= min(num_kb, 6)
            assert 3 * (smem + 1024) <= SMEM_PER_SM, (out, inp, rows, smem)    # three CTAs per SM fit in shared memory


def test_reference_model_runs_184_ctas():
    # four micro-batches of 32 rows: K = 128, four k-blocks in every CTA
    counts = [len(_C.wgrad_group_tiles(out, inp, 128)[0]) for inp, out in REF]
    assert counts == [4 * 25, 16, 16, 16, 16, 16, 4]
    assert sum(counts) == 184                                  # more than the 132 SMs of an H100: two or more per SM
    assert _C.wgrad_group_tiles(10, 123, 128)[0][-1] == (0, 96, 32, 32, True)   # layer 7: one 32-row feature tile


def test_only_chain_eligible_gemms_are_grouped():
    with pytest.raises(ValueError, match="out <= 128"):
        _C.wgrad_group_tiles(129, 64, 128)
    with pytest.raises(ValueError):
        _C.wgrad_group_tiles(0, 64, 128)
