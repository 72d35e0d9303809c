#!/usr/bin/env python
"""Regenerate tests/golden/ from the original ShallowSpeed installed in oracle/_ref (oracle/build_reference.py).

    python oracle/make_golden.py

Writes reference_pipeline.json.gz (instruction streams, PipeDream stub, MLP partition) and reference_mlp_numerics.npz
(init / forward / gradient sample of the default MLP); tests/golden/README.md describes both formats."""
import contextlib
import gzip
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
LEGEND = {"Z": "ZeroGrad", "LI": "LoadMuBatchInput", "LT": "LoadMuBatchTarget", "F": "Forward", "BA": "BackwardGradAcc",
          "BR": "BackwardGradAllReduce", "SA": "SendActivations", "RA": "RecvActivations", "SG": "SendInputGrad",
          "RG": "RecvOutputGrad", "O": "OptimizerStep"}


def load_reference():
    sys.path.insert(0, os.path.join(ROOT, "baseline", "mpi_shim"))
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import shallowspeed.layers as rlayers
    import shallowspeed.pipe as rpipe

    return rpipe, rlayers


def pipeline(rpipe, rlayers):
    code = {v: k for k, v in LEGEND.items()}

    def enc(sched):
        return "|".join(" ".join(code[type(i).__name__] + ("" if getattr(i, "mubatch_id", None) is None else f":{i.mubatch_id}")
                                 for i in tick) for tick in sched.steps())

    out = {"legend": LEGEND, "streams": {}, "pipedream_is_stub": False, "partitions": {}}
    for M in [1, 2, 4, 7]:
        for S in [1, 2, 4, 8]:
            for cls in ("NaiveParallelSchedule", "GPipeSchedule", "InferenceSchedule"):
                for stage in range(S):
                    out["streams"][f"{cls}/{M}/{S}/{stage}"] = enc(getattr(rpipe, cls)(M, S, stage))
    try:
        rpipe.PipeDreamSchedule()
    except NotImplementedError:
        out["pipedream_is_stub"] = True
    for pp in [1, 2, 4, 8]:
        for stage in range(pp):
            with contextlib.redirect_stdout(io.StringIO()):
                r = rlayers.MLP(SIZES, stage, pp, 128)
            layers = []
            for l in r.layers:
                d = {"type": type(l).__name__}
                if d["type"] == "Linear":
                    d["has_activation"] = l.activation is not None
                    d["W"] = list(l._params["W"].data.shape)
                    d["b"] = list(l._params["b"].data.shape)
                layers.append(d)
            out["partitions"][f"{pp}/{stage}"] = {"in_dim": r.in_dim, "out_dim": r.out_dim, "layers": layers}
    with gzip.GzipFile(os.path.join(OUT, "reference_pipeline.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps(out, sort_keys=True, separators=(",", ":")).encode())


def numerics(rlayers):
    with contextlib.redirect_stdout(io.StringIO()):
        ref = rlayers.MLP(SIZES, 0, 1, 128)
    rs = np.random.RandomState(0)
    x = rs.randn(32, 784).astype(np.float32)
    t = np.eye(10, dtype=np.float32)[rs.randint(0, 10, 32)]
    params = list(ref.parameters())
    init = [p.data.astype(np.float32).copy() for p in params]
    y = ref.forward(x, 0)
    ref.backward(t, 0)
    pick = np.random.RandomState(1234)
    shapes = np.full((len(params), 2), -1, np.int32)
    idx, iv, gv, cnt = [], [], [], []
    for i, p in enumerate(params):
        shapes[i, :p.data.ndim] = p.data.shape
        k = np.sort(pick.choice(p.data.size, size=min(p.data.size, 64), replace=False))
        cnt.append(len(k))
        idx.append(k)
        iv.append(init[i].reshape(-1)[k])
        gv.append(np.asarray(p.grad, np.float32).reshape(-1)[k])
    np.savez_compressed(os.path.join(OUT, "reference_mlp_numerics.npz"), output=np.asarray(y, np.float32), shapes=shapes,
                        counts=np.array(cnt, np.int32), idx=np.concatenate(idx).astype(np.int32),
                        init=np.concatenate(iv).astype(np.float32), grad=np.concatenate(gv).astype(np.float32))


if __name__ == "__main__":
    rpipe, rlayers = load_reference()
    pipeline(rpipe, rlayers)
    numerics(rlayers)
    print("golden data written to", OUT)
