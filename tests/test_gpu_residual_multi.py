"""Residual models (GELU with dropout, and ReLU) on several H100s: data parallel (dp = 2, 4, 8) under the fused in-kernel
reduction, NCCL and NVLS, and pipelines (pp = 2, 4) under GPipe and 1F1B over the peer-memory transport and NCCL, each
against the one-GPU engine at the same global batch.  The stage boundaries between hidden layers have a residual layer on
both sides: the producer stage keeps the gradient it receives as its last layer's skip gradient.  Layouts reorder fp32
sums, so the runs are compared with a tolerance: each parameter's update over the run agrees to 1e-4 of its norm, every
step's loss to 1e-5 relative; DP replicas are bit-identical (``assert_sync``).  Skipped when the layout needs more GPUs
than there are."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

REF = [784, 96, 96, 96, 96, 96, 96, 10]
LR, GBS, N_MU, STEPS = 0.05, 128, 4, 3
P, SEED = 0.2, 12345


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _rank_main(rank, world, dp, pp, port, comm, transport, out_dir, act, sched_name):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule, PipeDreamSchedule
    from shallowspeed_b200.utils import assert_sync, get_model_hash

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(dp, pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    model = MLP(REF, grid.stage, pp, GBS, dropout=P if act == "gelu" else 0.0, dropout_seed=SEED, activation=act,
                residual=True).to("cuda")
    opt = SGD(model.parameters(), LR, arena=model.arena)
    x, y = synthetic_mnist(n=GBS * STEPS)
    ds = Dataset(None, GBS, GBS // dp // N_MU, device="cuda")
    ds.local_batch_size = GBS // dp
    ds.from_arrays(x[grid.replica::dp], y[grid.replica::dp])
    w = NativeWorker(dp_comm if dp > 1 else None, pp_comm if pp > 1 else None, model, ds, opt, grid=grid,
                     comm_mode=comm, pp_transport=transport)
    sched = (PipeDreamSchedule if sched_name == "1f1b" else GPipeSchedule)(N_MU, pp, grid.stage)
    losses = []
    for b in range(STEPS):
        model.dropout_step = b
        w.execute(sched, b)
        losses.append(w.batch_loss())
    eng = w.engine_for(sched)
    w.sync_to_model()
    assert_sync(dp_comm, get_model_hash(model))
    torch.save({"w": model.arena.weights[: model.arena.numel].cpu(), "losses": losses,
                "describe": eng.describe(), "chain": bool(eng.uses_chain())},
               os.path.join(out_dir, f"s{grid.stage}r{grid.replica}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp, dp, pp, act, comm="fused", transport=None, sched="gpipe"):
    import torch.multiprocessing as mp

    world = dp * pp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29400 + (os.getpid() + world * 11 + len(os.listdir(tmp))) % 300
    out = tmp / f"run{len(os.listdir(tmp))}"
    out.mkdir()
    mp.spawn(_rank_main, args=(world, dp, pp, port, comm, transport, str(out), act, sched), nprocs=world, join=True)
    return [[torch.load(out / f"s{s}r{r}.pt") for r in range(dp)] for s in range(pp)]


def _params(res, pp):
    """Per-parameter tensors of the whole model from the stages' weight arenas."""
    from shallowspeed_b200.layers import MLP

    got = []
    for s in range(pp):
        stage = MLP(REF, s, pp, GBS, residual=True)
        stage.arena.weights.copy_(res[s][0]["w"])
        got += [p.data.clone() for p in stage.parameters()]
    return got


LAYOUTS = {
    "dp2-fused": (2, 1, "fused", None, "gpipe"), "dp4-fused": (4, 1, "fused", None, "gpipe"),
    "dp8-fused": (8, 1, "fused", None, "gpipe"), "dp2-nccl": (2, 1, "nccl", None, "gpipe"),
    "dp4-nccl": (4, 1, "nccl", None, "gpipe"), "dp2-nvls": (2, 1, "nvls", None, "gpipe"),
    "dp8-nvls": (8, 1, "nvls", None, "gpipe"),
    "pp2-peer-gpipe": (1, 2, "fused", "peer", "gpipe"), "pp2-nccl-1f1b": (1, 2, "fused", "nccl", "1f1b"),
    "pp4-peer-1f1b": (1, 4, "fused", "peer", "1f1b"), "pp4-nccl-gpipe": (1, 4, "fused", "nccl", "gpipe"),
}
_SEQ = {}


@pytest.mark.parametrize("act", ["gelu", "relu"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_residual_layout_matches_one_gpu_engine(layout, act, tmp_path):
    from shallowspeed_b200.layers import MLP

    dp, pp, comm, transport, sched = LAYOUTS[layout]
    if torch.cuda.device_count() < dp * pp:
        pytest.skip(f"needs {dp * pp} GPUs")
    if comm == "nvls":
        from shallowspeed_b200 import _C

        if not _C.NvlsContext.supported():
            pytest.skip("no NVLink multicast on this machine")
    if act not in _SEQ:
        _SEQ[act] = _spawn(tmp_path, 1, 1, act)
    seq = _SEQ[act]
    res = _spawn(tmp_path, dp, pp, act, comm, transport, sched)
    runs = [r for stage in res for r in stage]
    assert all(r["chain"] for r in runs)
    init = [p.data.clone() for p in MLP(REF, 0, 1, GBS, residual=True).parameters()]
    ref, got = _params(seq, 1), _params(res, pp)
    assert len(got) == len(ref) == len(init)
    for i, (p0, pr, pg) in enumerate(zip(init, ref, got)):
        err = _frob(pg - p0, pr - p0)
        assert err < 1e-4, (i, err)
    # each replica's loss covers its share of the global batch (scaled by 1 / GBS): their sum is the step's loss
    losses = [sum(r["losses"][i] for r in res[-1]) for i in range(STEPS)]
    for a, b in zip(losses, seq[0][0]["losses"]):
        assert abs(a - b) <= 1e-5 * abs(b), (a, b)
