"""CLI-level smoke tests on the CPU: train.py (sequential and a spawned DP x PP grid through the
portable VM), checkpoint/resume, and the JSON contract of bench.py's reference arm."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, timeout=600):
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_train_sequential_cpu(tmp_path):
    log = tmp_path / "m.jsonl"
    r = _run(["train.py", "--device", "cpu", "--steps", "6", "--no-eval", "--synthetic", "--log-json", str(log),
              "--save", str(tmp_path / "ck")])
    assert r.returncode == 0, r.stderr[-2000:]
    recs = [json.loads(l) for l in open(log)]
    assert any(rec.get("event") == "epoch" and rec["steps"] == 6 for rec in recs)
    assert (tmp_path / "ck" / "stage0of1.pt").exists()


def test_resume_continues_the_same_run(tmp_path):
    """6 steps in one go == 4 steps, checkpoint, resume to step 6: same global step, same position in the data, same
    weights (the CPU path is bit-deterministic); a resume under a different learning rate is refused."""
    import torch

    base = ["train.py", "--device", "cpu", "--no-eval", "--synthetic"]
    r = _run(base + ["--steps", "6", "--save", str(tmp_path / "full")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(base + ["--steps", "4", "--save", str(tmp_path / "part")])
    assert r.returncode == 0, r.stderr[-2000:]
    r = _run(base + ["--steps", "6", "--resume", str(tmp_path / "part"), "--save", str(tmp_path / "resumed")])
    assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(tmp_path / "full" / "stage0of1.pt")
    b = torch.load(tmp_path / "resumed" / "stage0of1.pt")
    assert a["step"] == b["step"] == 6 and a["hparams"] == b["hparams"]
    assert torch.equal(a["weights"], b["weights"])
    r = _run(base + ["--steps", "6", "--resume", str(tmp_path / "part"), "--lr", "0.5"])
    assert r.returncode != 0 and "checkpoint was written with lr" in (r.stderr + r.stdout)


def test_train_accepts_reference_flags_and_pipedream():
    # same three flags as the reference CLI; 'pipedream' (a stub there) works here
    r = _run(["train.py", "--device", "cpu", "--spawn", "--dp", "2", "--pp", "2", "--schedule", "pipedream", "--steps", "3",
              "--no-eval", "--synthetic"])
    assert r.returncode == 0, r.stderr[-2000:]


def test_train_rejects_bad_grids():
    r = _run(["train.py", "--device", "cpu", "--dp", "3", "--steps", "1", "--no-eval", "--synthetic"])
    assert r.returncode != 0            # 128 % 3 != 0 / world size mismatch


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "shallowspeed", "pipe.py")),
                    reason="reference not installed in oracle/_ref (oracle/build_reference.py, run by build())")
def test_bench_reference_arm_json_contract():
    r = _run(["bench.py", "--impl", "reference", "--steps", "5", "--warmup", "3"])
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "dtype", "data", "config", "e2e", "gpu_launches"):
        assert key in d, key
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 5 and d["value"] > 0
    assert d["config"]["global_batch"] == 128 and d["config"]["n_mubatches"] == 4


def test_blocking_ddp_contrast_script(tmp_path):
    """scripts/ddp_blocking_mnist.py (reference: scripts/DDP_PyTorch_MNIST.py): 1 process, then 2 gloo ranks with a
    blocking all-reduce per parameter; hashes agree across ranks and the divergence from the 1-process model is reported."""
    script = os.path.join(ROOT, "scripts", "ddp_blocking_mnist.py")
    env = dict(os.environ, OMP_NUM_THREADS="1")
    common = ["--epochs", "1", "--samples", "1280", "--device", "cpu"]
    r = subprocess.run([sys.executable, script] + common, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert (tmp_path / "data" / "models" / "model_p1.pkl").exists()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29671", script] + common, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("L1 divergence")]
    assert line and float(line[0].rsplit(" ", 1)[1]) < 1.0      # same global batches, summation order differs


def test_parsers_know_the_runtime_knobs():
    sys.path.insert(0, ROOT)
    try:
        import bench
        import train
    finally:
        sys.path.remove(ROOT)
    a = train.build_parser().parse_args(["--dp", "2", "--pp", "2", "--schedule", "pipedream-flush", "--comm", "nvls",
                                         "--pp-transport", "peer", "--watchdog-s", "30", "--precision", "tf32"])
    assert (a.comm, a.pp_transport, a.watchdog_s, a.precision, a.schedule) == ("nvls", "peer", 30.0, "tf32", "pipedream-flush")
    d = train.build_parser().parse_args([])
    assert (d.dp, d.pp, d.schedule, d.comm, d.pp_transport, d.watchdog_s, d.precision) == (1, 1, "naive", "fused", None, None, "fp32")
    old = sys.argv
    try:
        sys.argv = ["bench.py"]
        b = bench.parse()
    finally:
        sys.argv = old
    assert b.gpus == 1 and b.impl in ("ours", None, "") or b.impl == "ours"
    assert b.precision == "fp32" and b.comm == "fused" and b.pp_transport is None and not b.no_alt


def test_importing_the_package_leaves_the_environment_alone():
    """Every default lives in the code that reads it: importing the package (and the native engine's front end) sets
    no environment variable, so a process and the workers it spawns build the same plans whatever imported what."""
    code = ("import json, os, sys; sys.path.insert(0, sys.argv[1]); import torch; before = dict(os.environ); "
            "import shallowspeed_b200, shallowspeed_b200.parallel.engine; print(json.dumps([before, dict(os.environ)]))")
    env = {k: v for k, v in os.environ.items() if not k.startswith("SSB_")}
    r = subprocess.run([sys.executable, "-c", code, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    before, after = json.loads(r.stdout.strip().splitlines()[-1])
    assert after == before, sorted(set(after.items()) ^ set(before.items()))


def test_bench_dump_outputs_stays_within_its_budget(tmp_path):
    """--dump-outputs writes a small arena in full and a large one as a fixed, seeded sample with its positions, always
    within the byte budget (64 MB by default; a tiny budget here so the arena is 'large')."""
    import importlib.util
    import types

    import numpy as np
    import torch

    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    assert bench.DUMP_LIMIT_BYTES == 64 << 20
    w = torch.arange(200_000, dtype=torch.float32)
    trainer = types.SimpleNamespace(model=types.SimpleNamespace(arena=types.SimpleNamespace(weights=w)),
                                    pp_comm=types.SimpleNamespace(Get_rank=lambda: 0), is_last=True)
    grid = types.SimpleNamespace(replica=0, pp=1)

    full = tmp_path / "full"
    bench.dump_outputs(str(full), trainer, 0.5, grid)
    assert sorted(p.name for p in full.iterdir()) == ["loss.npy", "weights_stage0.npy"]
    assert np.array_equal(np.load(full / "weights_stage0.npy"), w.numpy()) and np.load(full / "loss.npy")[0] == 0.5

    limit = 64 << 10
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), trainer, 0.5, grid, limit_bytes=limit)
        assert sum(p.stat().st_size for p in (tmp_path / d).iterdir()) <= limit
    idx, vals = np.load(tmp_path / "a" / "weights_stage0_idx.npy"), np.load(tmp_path / "a" / "weights_stage0.npy")
    assert len(idx) > 1000 and np.array_equal(vals, w.numpy()[idx])
    assert np.array_equal(idx, np.load(tmp_path / "b" / "weights_stage0_idx.npy"))   # same positions on every run

