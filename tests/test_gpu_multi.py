"""Multi-GPU tests (one process per GPU, NCCL + the fused peer-memory DP kernels).
Each case spawns `world` ranks with torch.multiprocessing and compares against the CPU
oracle run in the parent."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]


def _nvls_supported():
    if not torch.cuda.is_available():
        return False
    from shallowspeed_b200 import _C

    return bool(_C.NvlsContext.supported())


WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]     # > 128 wide: per-layer GEMM kernels, two-shot DP for the 4 MB layers
GBS, N_MU, LR, STEPS = 128, 4, 0.05, 4


def _worker(rank, world, dp, pp, sched_name, comm_mode, port, out_dir, coalesce, two_shot=False, sizes=None, extra_env=None, steps=STEPS,
            pp_transport=None):
    sizes = sizes or SIZES
    os.environ.update(extra_env or {})
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    if not coalesce:
        os.environ["SSB_NO_COALESCE"] = "1"
    if two_shot:
        os.environ["SSB_DP_TWO_SHOT"] = "1"
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS
    from shallowspeed_b200.utils import assert_sync, get_model_hash

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(dp, pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    model = MLP(sizes, grid.stage, pp, GBS).to(f"cuda:{rank}")
    opt = SGD(model.parameters(), LR, arena=model.arena)
    x, y = synthetic_mnist(n=GBS * STEPS)
    ds = Dataset(None, GBS, GBS // dp // N_MU, device=f"cuda:{rank}")
    ds.local_batch_size = GBS // dp
    ds.from_arrays(x[grid.replica::dp], y[grid.replica::dp])
    w = NativeWorker(dp_comm, pp_comm, model, ds, opt, grid=grid, comm_mode=comm_mode, pp_transport=pp_transport)
    sched = SCHEDULE_NAME_TO_CLS[sched_name](N_MU, pp, grid.stage)
    losses = []
    for b in range(steps):
        w.execute(sched, b)
        losses.append(w.batch_loss())
    w.sync_to_model()
    assert_sync(dp_comm, get_model_hash(model))          # replicas bit-identical
    if grid.replica == 0:
        torch.save({"params": [p.data.cpu().clone() for p in model.parameters()], "losses": losses},
                   os.path.join(out_dir, f"stage{grid.stage}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _cpu_oracle(sizes=None, steps=STEPS):
    sizes = sizes or SIZES
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.pipe import NaiveParallelSchedule, Worker

    x, y = synthetic_mnist(n=GBS * STEPS)
    model = MLP(sizes, 0, 1, GBS)
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(x, y)
    w = Worker(None, None, model, ds, SGD(model.parameters(), LR, arena=model.arena))
    for b in range(steps):
        w.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    return [p.data.clone() for p in model.parameters()], MLP(sizes, 0, 1, GBS)


def _run(dp, pp, sched, comm_mode, tmp_path, coalesce=True, two_shot=False, sizes=None, extra_env=None, steps=STEPS, tight=False,
         pp_transport=None):
    import torch.multiprocessing as mp

    world = dp * pp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29800 + (os.getpid() + dp * 7 + pp * 13 + len(sched)) % 150
    mp.spawn(_worker, args=(world, dp, pp, sched, comm_mode, port, str(tmp_path), coalesce, two_shot, sizes, extra_env, steps,
                            pp_transport), nprocs=world,
             join=True)
    got = [p for s in range(pp) for p in torch.load(tmp_path / f"stage{s}.pt")["params"]]
    ref, init = _cpu_oracle(sizes, steps)
    for i, (p0, a, b) in enumerate(zip(init.parameters(), got, ref)):
        upd_err = float(((a - p0.data) - (b - p0.data)).norm() / ((b - p0.data).norm() + 1e-12))
        if tight:   # ONE step: no ReLU sign flips yet - fp32-level agreement (bias 1e-4, weight at the fp32 storage-rounding floor)
            assert upd_err < (1e-4 if i % 2 == 1 else 3e-3), (i, upd_err)
        else:       # 4 steps: bounded by ReLU sign flips between two fp32 implementations (see test_gpu_engine)
            assert upd_err < 3e-2, upd_err


@pytest.mark.parametrize("comm_mode", ["fused", "nccl"])
def test_dp2(comm_mode, tmp_path):
    _run(2, 1, "naive", comm_mode, tmp_path)


@pytest.mark.parametrize("dp,pp,sched,comm_mode", [(2, 1, "naive", "fused"), (2, 1, "naive", "nvls"), (1, 2, "gpipe", "fused"),
                                                   (1, 2, "pipedream", "fused"), (2, 2, "gpipe", "fused"), (8, 1, "naive", "fused")])
def test_single_step_matches_the_cpu_oracle_tightly(dp, pp, sched, comm_mode, tmp_path):
    """The tight multi-GPU numerics check: one optimizer step, per-parameter update error against the fp32 CPU oracle
    at 1e-4 (biases) / 3e-3 (weights), the same bounds as the single-GPU test_engine_fp32_single_step_is_fp32_accurate."""
    if comm_mode == "nvls" and not _nvls_supported():
        pytest.skip("NVLink multicast not supported on this device / driver")
    _run(dp, pp, sched, comm_mode, tmp_path, steps=1, tight=True)


def test_dp2_fused_two_shot_protocol(tmp_path):
    """owner-reduces / publishes-weights variant (used for big layers), forced on the small model"""
    _run(2, 1, "naive", "fused", tmp_path, two_shot=True)


@pytest.mark.parametrize("two_shot", [False, True])
def test_dp2_fused_per_microbatch_path(two_shot, tmp_path):
    _run(2, 1, "gpipe", "fused", tmp_path, coalesce=False, two_shot=two_shot)


@pytest.mark.parametrize("sched", ["naive", "gpipe", "pipedream"])
def test_pp2(sched, tmp_path):
    _run(1, 2, sched, "fused", tmp_path)


def test_dp2_pp2_gpipe_fused(tmp_path):
    _run(2, 2, "gpipe", "fused", tmp_path)


def test_dp4_fused(tmp_path):
    _run(4, 1, "naive", "fused", tmp_path)


def test_pp4_1f1b(tmp_path):
    _run(1, 4, "pipedream", "fused", tmp_path)


def test_dp8_fused(tmp_path):
    _run(8, 1, "naive", "fused", tmp_path)


def test_dp2_pp4_gpipe(tmp_path):
    _run(2, 4, "gpipe", "fused", tmp_path)


def test_wide_model_dp2_fused(tmp_path):
    """layers wider than 128: per-layer tensor-core GEMM kernels (no chain), multi-tile fused wgrad+DP kernels,
    two-shot single-owner protocol on the 4 MB layers"""
    _run(2, 1, "naive", "fused", tmp_path, sizes=WIDE)


def test_wide_model_dp2_pp2_1f1b(tmp_path):
    _run(2, 2, "pipedream", "fused", tmp_path, sizes=WIDE)


# ---------------------------------------------------------------------------------------------------------
# NVLS path (--comm nvls): the switch reduces the gradient arena and multicasts the updated weights.
# ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("dp,pp,sched,coalesce", [(2, 1, "naive", True), (2, 1, "gpipe", False), (2, 2, "pipedream", True)])
def test_nvls_reduce_sgd_matches_oracle(dp, pp, sched, coalesce, tmp_path):
    if not _nvls_supported():
        pytest.skip("NVLink multicast not supported on this device / driver")
    _run(dp, pp, sched, "nvls", tmp_path, coalesce=coalesce)


# ---------------------------------------------------------------------------------------------------------
# Peer-memory pipeline transport (--pp-transport peer, the default): one-sided pushes + epoch flags instead of
# NCCL send/recv.
# ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("dp,pp,sched", [(1, 2, "naive"), (1, 2, "gpipe"), (1, 2, "pipedream"), (1, 4, "gpipe"), (2, 2, "pipedream")])
def test_pp_peer_transport_matches_oracle(dp, pp, sched, tmp_path):
    _run(dp, pp, sched, "fused", tmp_path, pp_transport="peer")


# ---------------------------------------------------------------------------------------------------------
# Train <-> validation alternation on ONE pipeline communicator (advisor finding, round 1): the validation worker's
# engine and the training worker's engine share the native ncclComm but own separate streams and graphs; without an
# explicit edge between them stage 0 could enqueue training sends while its validation sends were still pending.
# ---------------------------------------------------------------------------------------------------------
ROUNDS, VAL_BATCHES, TRAIN_STEPS = 3, 3, 3


def _alternation_worker(rank, world, pp, sched_name, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS, InferenceSchedule

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(1, pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    model = MLP(SIZES, grid.stage, pp, GBS).to(f"cuda:{rank}")
    opt = SGD(model.parameters(), LR, arena=model.arena)
    x, y = synthetic_mnist(n=GBS * ROUNDS * TRAIN_STEPS)
    ds = Dataset(None, GBS, GBS // N_MU, device=f"cuda:{rank}")
    ds.local_batch_size = GBS
    ds.from_arrays(x, y)
    vds = Dataset(None, GBS, GBS, device=f"cuda:{rank}")
    vds.local_batch_size = GBS
    vds.from_arrays(x[: GBS * VAL_BATCHES], y[: GBS * VAL_BATCHES])
    w = NativeWorker(dp_comm, pp_comm, model, ds, opt, grid=grid)
    vw = NativeWorker(None, pp_comm, model, vds, None, grid=grid, comm_mode="nccl", share=w)
    sched = SCHEDULE_NAME_TO_CLS[sched_name](N_MU, pp, grid.stage)
    probs = []
    step = 0
    for _r in range(ROUNDS):
        # NO host synchronisation between the two phases on the non-last stages: exactly the situation train.py creates
        for b in range(VAL_BATCHES):
            vw.execute(InferenceSchedule(1, pp, grid.stage), b)
            if grid.stage == pp - 1:
                probs.append(vw.output_buffers[0].cpu().clone())
        for _s in range(TRAIN_STEPS):
            w.execute(sched, step)
            step += 1
    w.sync_to_model()
    torch.save({"params": [p.data.cpu().clone() for p in model.parameters()], "probs": probs}, os.path.join(out_dir, f"stage{grid.stage}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("pp,sched", [(2, "gpipe"), (2, "pipedream")])
def test_train_eval_alternation_on_one_pipeline_comm(pp, sched, tmp_path):
    import torch.multiprocessing as mp

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.pipe import InferenceSchedule, NaiveParallelSchedule, Worker

    if torch.cuda.device_count() < pp:
        pytest.skip(f"needs {pp} GPUs")
    port = 29950 + (os.getpid() + len(sched)) % 40
    mp.spawn(_alternation_worker, args=(pp, pp, sched, port, str(tmp_path)), nprocs=pp, join=True)
    got = [torch.load(tmp_path / f"stage{s}.pt") for s in range(pp)]
    # CPU oracle: the same alternation, sequentially
    x, y = synthetic_mnist(n=GBS * ROUNDS * TRAIN_STEPS)
    model = MLP(SIZES, 0, 1, GBS)
    init = [p.data.clone() for p in model.parameters()]
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(x, y)
    vds = Dataset(None, GBS, GBS)
    vds.local_batch_size = GBS
    vds.from_arrays(x[: GBS * VAL_BATCHES], y[: GBS * VAL_BATCHES])
    w = Worker(None, None, model, ds, SGD(model.parameters(), LR, arena=model.arena))
    vw = Worker(None, None, model, vds, None)
    ref_probs, step = [], 0
    for _r in range(ROUNDS):
        model.eval()
        for b in range(VAL_BATCHES):
            vw.execute(InferenceSchedule(1, 1, 0), b)
            ref_probs.append(vw.output_buffers[0].clone())
        model.train()
        for _s in range(TRAIN_STEPS):
            w.execute(NaiveParallelSchedule(N_MU, 1, 0), step)
            step += 1
    probs = got[pp - 1]["probs"]
    assert len(probs) == len(ref_probs)
    for a, b in zip(probs, ref_probs):
        assert float((a - b).abs().max()) < 2e-3
    params = [p for s in range(pp) for p in got[s]["params"]]
    for p0, a, b in zip(init, params, [p.data for p in model.parameters()]):
        upd_err = float(((a - p0) - (b - p0)).norm() / ((b - p0).norm() + 1e-12))
        assert upd_err < 3e-2, upd_err


# ---------------------------------------------------------------------------------------------------------
# LL two-shot fused DP kernel (csrc/kernels/dp_ll.cu; default for narrow layers) against the flag-protocol kernels it
# replaces (SSB_DP_LL=0): same MMAs, same fixed-rank-order sum, same update expression => bit-identical weights.
# Also with the gate off (SSB_DP_GATE=0: the kernel is ordered behind the chain kernel by a graph edge).
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dp", [2, 4, 8])
def test_dp_ll_kernel_is_bitwise_identical_to_flag_protocol(dp, tmp_path):
    if torch.cuda.device_count() < dp:
        pytest.skip(f"needs {dp} GPUs")
    outs = {}
    for name, env in (("flags", {"SSB_DP_LL": "0"}), ("ll_gated", {"SSB_DP_LL": "1", "SSB_DP_GATE": "1"}),
                      ("ll_edge", {"SSB_DP_LL": "1", "SSB_DP_GATE": "0"})):
        d = tmp_path / name
        d.mkdir()
        _run(dp, 1, "naive", "fused", d, extra_env=env)          # also checks the oracle tolerance and replica equality
        outs[name] = torch.load(d / "stage0.pt")
    for name in ("ll_gated", "ll_edge"):
        assert outs[name]["losses"] == outs["flags"]["losses"], name
        for a, b in zip(outs[name]["params"], outs["flags"]["params"]):
            assert torch.equal(a, b), name
