"""Parity checks against the original ShallowSpeed implementation: instruction streams of every schedule it implements,
the model partitioner, and its PipeDream stub.  What the original produced is stored in
tests/golden/reference_pipeline.json.gz (see tests/golden/README.md), so the checks run without it."""
import gzip
import json
import os

import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pipeline.json.gz")


@pytest.fixture(scope="module")
def ref():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def _stream(sched):
    return [[[type(i).__name__, getattr(i, "mubatch_id", None)] for i in tick] for tick in sched.steps()]


def _decode(ref, s):
    """'|'-separated ticks of ' '-separated instructions, each a legend code with ':<mubatch_id>' where it has one"""
    if not s:
        return []
    return [[[ref["legend"][i.split(":")[0]], int(i.split(":")[1]) if ":" in i else None] for i in tick.split(" ") if i]
            for tick in s.split("|")]


@pytest.mark.parametrize("M", [1, 2, 4, 7])
@pytest.mark.parametrize("S", [1, 2, 4, 8])
def test_instruction_streams_equal_the_reference(ref, M, S):
    from shallowspeed_b200 import pipe

    for ours in (pipe.NaiveParallelSchedule, pipe.GPipeSchedule, pipe.InferenceSchedule):
        for stage in range(S):
            theirs = _decode(ref, ref["streams"][f"{ours.__name__}/{M}/{S}/{stage}"])
            assert _stream(ours(M, S, stage)) == theirs, (ours.__name__, M, S, stage)


def test_reference_pipedream_is_a_stub_ours_is_not(ref):
    from shallowspeed_b200 import pipe
    from shallowspeed_b200.parallel.validate import validate

    assert ref["pipedream_is_stub"]               # the original's PipeDreamSchedule raises NotImplementedError
    validate(pipe.PipeDreamSchedule, 8, 4)


@pytest.mark.parametrize("pp", [1, 2, 4, 8])
def test_partitioner_matches_reference(ref, pp):
    from shallowspeed_b200.layers import MLP

    sizes = [784, 128, 127, 126, 125, 124, 123, 10]
    for stage in range(pp):
        r = ref["partitions"][f"{pp}/{stage}"]
        o = MLP(sizes, stage, pp, 128)
        assert (o.in_dim, o.out_dim) == (r["in_dim"], r["out_dim"])
        assert [type(l).__name__ for l in o.layers] == [l["type"] for l in r["layers"]]
        for lo, lr in zip(o.layers, r["layers"]):
            if type(lo).__name__ == "Linear":
                assert (lo.activation is not None) == lr["has_activation"]
                assert list(lo._params["W"].data.shape) == lr["W"]
                assert list(lo._params["b"].data.shape) == lr["b"]
