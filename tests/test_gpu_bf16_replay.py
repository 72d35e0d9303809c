"""The one-GPU replays of test_gpu_dp_replay (a data-parallel replica, its peers replayed from memory) and
test_gpu_pp_replay (a pipeline stage, its neighbours' boundary tiles and flags replayed) with ``precision="bf16"``.

The replays run unchanged; for the duration of a case their GEMM oracles are swapped for the bf16 ones of test_gpu_bf16:
every product from the operands rounded to bf16, within RTOL_BF16 = 2^-16 of sum |a'||b'| (plus test_gpu_gemm's K > 4096
term), the bias gradient the fp32 column sum of the unrounded dZ.  So every owned update, every copied or untouched peer
element and every outbound tile or line is checked per element against the bf16 oracle, in the dp x pp stages as well
(an LL and a flag-protocol stage, whose DP checks run on the partials of the swapped oracle)."""
import pytest

import test_gpu_dp_replay as DP
import test_gpu_pp_replay as PP
from test_gpu_bf16 import RTOL_BF16, bf, grad_oracle_bf16, rtol_bf16
from test_gpu_chain import dgrad_oracle, fwd_oracle

pytestmark = pytest.mark.gpu


def _rtol_for(precision, k, splits=1):
    assert precision == "bf16", precision
    return rtol_bf16(k, splits)


def _bf16_oracles(monkeypatch, *modules):
    for module in modules:
        monkeypatch.setattr(module, "grad_oracle", grad_oracle_bf16)
        monkeypatch.setattr(module, "rtol_for", _rtol_for)


@pytest.mark.parametrize("dp,rank,gate", [(2, 1, "1"), (4, 2, "0"), (8, 7, "1")])
def test_ll_replay(dp, rank, gate, monkeypatch):
    _bf16_oracles(monkeypatch, DP)
    DP._run(f"ll dp{dp} r{rank} gate{gate} bf16", DP.REF, dp, rank, "ll", env={"SSB_DP_GATE": gate},
            mb_rows=128 // dp // 4, n_mu=4, precision="bf16", monkeypatch=monkeypatch)


@pytest.mark.parametrize("sizes,dp,rank,shot", [("ref", 2, 1, "one-shot"), ("ref", 4, 0, "two-shot"),
                                                ("wide", 2, 0, "two-shot")])
def test_flag_replay(sizes, dp, rank, shot, monkeypatch):
    _bf16_oracles(monkeypatch, DP)
    env = {"SSB_DP_LL": "0", "SSB_DP_ONE_SHOT" if shot == "one-shot" else "SSB_DP_TWO_SHOT": "1"}
    DP._run(f"flags {sizes} dp{dp} r{rank} {shot} bf16", {"ref": DP.REF, "wide": DP.WIDE}[sizes], dp, rank, shot,
            env=env, precision="bf16", monkeypatch=monkeypatch)


def test_dp1_flag_protocol_stateful(monkeypatch):
    _bf16_oracles(monkeypatch, DP)
    DP._run("dp1 ref-one-shot-stateful bf16", DP.REF, 1, 0, "one-shot", precision="bf16", stateful=True,
            monkeypatch=monkeypatch)


# folded boundaries (the chain kernel stores into the neighbour's slot) and the unfolded transport, first and last stage
PP_CASES = {
    "ref-pp2-s0-gpipe-mb24": PP._case(PP.REF, 2, 0, "gpipe", mb=24, precision="bf16"),
    "ref-pp2-s1-1f1b-mb24": PP._case(PP.REF, 2, 1, "1f1b", mb=24, precision="bf16"),
    "ref-pp2-s0-unfolded": PP._case(PP.REF, 2, 0, "1f1b", env=PP.UNFOLD, push="small", precision="bf16"),
    "ref-pp4-s2-unfolded-mb128": PP._case(PP.REF, 4, 2, "gpipe", mb=128, n_mu=2, env=PP.UNFOLD, push="multi",
                                          precision="bf16"),
    # dp x pp: the LL wave over act_in, and the flag protocol behind per-micro-batch weight gradients
    "ref-pp2-s1-dp2-r0-1f1b": PP._case(PP.REF, 2, 1, "1f1b", dp=2, rank=0, precision="bf16"),
    "ref-pp4-s1-dp4-r2-flags-two-shot-stateful": PP._case(PP.REF, 4, 1, "gpipe", env={"SSB_DP_LL": "0", "SSB_DP_TWO_SHOT": "1"},
                                                          stateful=True, dp=4, rank=2, precision="bf16"),
}


@pytest.mark.parametrize("name", list(PP_CASES))
def test_pp_stage_replay(name, monkeypatch):
    _bf16_oracles(monkeypatch, PP, DP)        # DP: the partials dp_check compares the outbound messages with
    # the stage's forward and dgrad products from the rounded operands; the replay looks its rtol up by precision
    monkeypatch.setattr(PP, "RTOL", {"bf16": RTOL_BF16})
    monkeypatch.setattr(PP, "fwd_oracle", lambda x, W, b, relu, rtol: fwd_oracle(bf(x), bf(W), b, relu, rtol))
    monkeypatch.setattr(PP, "dgrad_oracle", lambda dz, W, mask, rtol: dgrad_oracle(bf(dz), bf(W), mask, rtol))
    monkeypatch.setitem(PP.CASES, name + "-bf16", PP_CASES[name])
    PP._run(name + "-bf16", monkeypatch)
