"""Host-side planning of the split-K GEMM variant (pure C++ logic, no GPU needed).  An EMPTY k-split would leave a CTA
whose accumulator never completes (its epilogue would sit in a bounded spin until the trap), so the planner's
"no empty split" guarantee is checked exhaustively here."""
import pytest

from shallowspeed_b200 import _C


@pytest.mark.parametrize("sms", [132, 148])
def test_planner_never_leaves_a_split_empty_and_keeps_two_ctas_per_sm_in_smem(sms):
    seen_split = 0
    for m in (10, 127, 128, 1000, 2048, 4096, 8192, 16384):
        for rows in (4, 8, 32, 33, 128, 256):
            for k in (10, 123, 784, 1000, 2048, 4096, 8192, 8200):
                splits, per, grid_z, stages, smem, err = _C.splitk_plan(m, rows, k, sms, 0)
                num_kb = (k + 31) // 32
                assert err == ""
                assert splits >= 1
                if splits == 1:
                    continue
                seen_split += 1
                assert grid_z == splits
                assert (splits - 1) * per < num_kb <= splits * per          # every split owns >= 1 k-block
                assert per >= 8                                              # enough work to fill the pipeline
                bn = 64 if rows >= 64 else (rows + 15) // 16 * 16
                tiles = ((m + 127) // 128) * ((rows + bn - 1) // bn)
                assert tiles * 2 <= sms and tiles * splits <= 2 * sms + tiles
                assert 2 <= stages <= 6 and smem <= 113 * 1024               # two CTAs per SM fit
    assert seen_split > 20


def test_forcing_an_illegal_split_count_is_rejected_not_silently_accepted():
    # 25 k-blocks into 8 splits -> ceil = 4 per split -> only 7 non-empty splits
    splits, per, grid_z, stages, smem, err = _C.splitk_plan(128, 32, 784, 148, 8)
    assert "empty split" in err
    splits, per, grid_z, stages, smem, err = _C.splitk_plan(128, 32, 784, 148, 5)      # 5 x 5 = 25: legal
    assert err == "" and grid_z == 5 and per == 5


# --------------------------------------------------------------------------------------------- chain kernel budget
def test_chain_budget_fits_the_sm_and_keeps_a_double_buffered_ring():
    for split in (False, True):
        for mb in (1, 4, 16, 32, 33, 64, 96, 128):
            ok, kps, stages, smem = _C.chain_budget(mb, split)
            assert ok                               # 3xTF32 derives its lo parts in registers: no twin buffers
            assert kps in (1, 2, 4) and 2 <= stages <= 8
            assert smem <= 227 * 1024               # opt-in dynamic shared memory limit of an sm_90a CTA
    assert _C.chain_budget(32, False)[:3] == (True, 4, 2)      # the flagship config: K=128 per stage, double-buffered
    assert _C.chain_budget(32, True)[:3] == (True, 4, 2)
    assert not _C.chain_budget(129, False)[0]


def test_chain_eligibility_rules():
    ref = [(784, 128), (128, 127), (127, 126), (126, 125), (125, 124), (124, 123), (123, 10)]
    assert _C.chain_eligible(ref, 32, 10, True, False) and _C.chain_eligible(ref, 32, 10, True, True)
    assert _C.chain_eligible(ref, 128, 10, True, False)
    assert _C.chain_eligible(ref, 128, 10, True, True)                # fp32 (3xTF32) needs no extra shared memory
    assert not _C.chain_eligible([(784, 256), (256, 10)], 32, 10, True, False)     # wider than one M tile
    assert not _C.chain_eligible([(784, 128), (128, 64)], 32, 64, True, False)     # loss head handles <= 32 classes
    assert _C.chain_eligible([(784, 128), (128, 64)], 32, 64, False, False)        # ... but a middle stage may be 64 wide
    assert not _C.chain_eligible([(8192, 128)] * 17, 32, 128, False, False)        # more layers than the plan holds


# --------------------------------------------------------------------------------------------- fused DP geometry
@pytest.mark.parametrize("dp", [2, 4, 8])
def test_dp_geometry_covers_every_tile_exactly_once(dp):
    for (i, o) in [(784, 128), (128, 127), (123, 10), (8192, 8192), (1000, 520), (5, 3)]:
        for one_shot in (True, False):
            block_n, tm, tn, slots, slot_floats = _C.dp_layer_geometry(i, o, dp, one_shot)
            assert block_n % 32 == 0 and 32 <= block_n <= 128
            assert tm * 128 >= o > (tm - 1) * 128 and tn * block_n >= i > (tn - 1) * block_n
            tiles = tm * tn
            assert slot_floats == 128 * block_n + 128                  # tile + the bias-gradient column
            if one_shot:
                assert slots == tiles                                   # everybody holds every tile
            else:
                # tile t is owned by replica t % dp and uses slot t // dp there
                per_owner = {}
                for t in range(tiles):
                    per_owner.setdefault(t % dp, set()).add(t // dp)
                assert all(max(v) < slots and len(v) == sum(1 for t in range(tiles) if t % dp == r) for r, v in per_owner.items())
