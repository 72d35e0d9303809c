"""The plan self-check itself, on hand-written plans (the real plans are checked on the GPU in test_gpu_zz_aux.py)."""
import pytest

from shallowspeed_b200.parallel.plan_check import PlanError, check_plan, parse_plan

GOOD = """
0 record_event stream=0 event=0
1 mlp_chain stream=0 mu=0
2 record_event stream=0 event=1
3 wait_event stream=5 event=1
4 gemm stream=5 layer=7
5 record_event stream=5 event=2
6 wait_event stream=6 event=1
7 gemm stream=6 layer=6
8 record_event stream=6 event=3
9 wait_event stream=0 event=2
10 wait_event stream=0 event=3
11 sgd stream=0
12 loss_d2h stream=0
"""


def test_parses_fields_and_accepts_a_fork_join_plan():
    ops = parse_plan(GOOD)
    assert ops[4].name == "gemm" and ops[4].stream == 5 and ops[4].layer == 7 and ops[1].mu == 0
    s = check_plan(GOOD)
    assert s == {"ops": 13, "kernels_and_copies": 5, "streams": 3, "events": 4, "cross_stream_edges": 4}


def test_comm_group_payload_is_ignored_by_the_parser():
    txt = GOOD + "13 pp_send_recv stream=0 [send->1:4096 recv<-1:4096 ]\n"
    assert parse_plan(txt)[-1].name == "pp_send_recv"
    check_plan(txt)


@pytest.mark.parametrize("mutate,msg", [
    (lambda t: t.replace("3 wait_event stream=5 event=1", "3 wait_event stream=5 event=9"), "before anything records"),
    (lambda t: t.replace("8 record_event stream=6 event=3", "8 record_event stream=6 event=2"), "recorded twice"),
    (lambda t: t.replace("10 wait_event stream=0 event=3\n", ""), "not waited for by the main stream"),
    (lambda t: t.replace("6 wait_event stream=6 event=1\n", ""), "without being forked"),
    (lambda t: t.replace("8 record_event stream=6 event=3\n", "").replace("10 wait_event stream=0 event=3\n", ""), "never joined"),
    (lambda t: t.replace("9 wait_event stream=0 event=2", "9 wait_event stream=5 event=2"), "its own event"),
])
def test_rejects_malformed_plans(mutate, msg):
    with pytest.raises(PlanError, match=msg):
        check_plan(mutate(GOOD))
