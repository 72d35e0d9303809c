"""Learning-rate schedules on several H100s: a warmup + cosine schedule through every data-parallel transport (LL, the
flag protocol on the wide model, NCCL, NVLS) at dp 2 / 4 / 8 and through pipeline layouts (GPipe, 1F1B) with the peer
and the NCCL boundary transport; replicas bit-identical and equal to the sequential CPU oracle under the same schedule;
a checkpoint resume mid-schedule in a fresh process group equals the uninterrupted run."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

REF = [784, 128, 127, 126, 125, 124, 123, 10]
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]
MOM = dict(momentum=0.9, weight_decay=1e-3, nesterov=True)
LR, GBS, N_MU, STEPS = 0.05, 128, 4, 5
SCHEDULE = dict(kind="cosine", total_steps=STEPS, warmup_steps=2, warmup_start_factor=0.25, min_lr=0.0)
TOL = 2e-2                                   # relative error of the update after STEPS steps (tests/test_gpu_momentum.py)


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _schedule():
    from shallowspeed_b200.lr_schedule import LRSchedule

    return LRSchedule(LR, **SCHEDULE)


def _data():
    from shallowspeed_b200.dataset import synthetic_mnist

    return synthetic_mnist(n=GBS * STEPS)


def _rank_main(rank, world, dp, pp, port, comm, transport, env, sizes, sched_name, steps, out_dir, ckpt):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), **env)
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS
    from shallowspeed_b200.utils import assert_sync, get_model_hash
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(dp, pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    model = MLP(sizes, grid.stage, pp, GBS).to("cuda")
    opt = SGD(model.parameters(), LR, arena=model.arena, **MOM)
    schedule = _schedule()
    hparams = dict(lr=LR, lr_schedule=schedule.spec(), **MOM)
    first = 0
    if ckpt is not None and ckpt[0] == "load":
        first = load_stage(model, ckpt[1], grid.stage, pp, expect_hparams=hparams)
    x, y = _data()
    ds = Dataset(None, GBS, GBS // dp // N_MU, device="cuda")
    ds.local_batch_size = GBS // dp
    ds.from_arrays(x[grid.replica::dp], y[grid.replica::dp])
    w = NativeWorker(dp_comm if dp > 1 else None, pp_comm if pp > 1 else None, model, ds, opt, grid=grid, comm_mode=comm,
                     pp_transport=transport)
    sched = SCHEDULE_NAME_TO_CLS[sched_name](N_MU, pp, grid.stage)
    for b in range(first, steps):
        opt.lr = schedule(b)
        w.execute(sched, b)
    w.sync_to_model()
    assert_sync(dp_comm, get_model_hash(model))
    state = w.optimizer_state()
    if ckpt is not None and ckpt[0] == "save" and grid.replica == 0:
        save_stage(model, ckpt[1], grid.stage, pp, step=steps, hparams=hparams, momentum=state)
    if grid.replica == 0:
        torch.save({"w": model.arena.weights[: model.arena.numel].cpu(), "v": state}, os.path.join(out_dir, f"s{grid.stage}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp, dp, pp, comm="fused", transport="nccl", env=None, sizes=REF, sched="gpipe", steps=STEPS, ckpt=None):
    import torch.multiprocessing as mp

    world = dp * pp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29400 + (os.getpid() + world * 7 + len(os.listdir(tmp))) % 300
    out = tmp / f"run{len(os.listdir(tmp))}"
    out.mkdir()
    mp.spawn(_rank_main, args=(world, dp, pp, port, comm, transport, env or {}, sizes, sched, steps, str(out), ckpt),
             nprocs=world, join=True)
    return [torch.load(out / f"s{s}.pt") for s in range(pp)]


def _oracle(sizes):
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.pipe import NaiveParallelSchedule, Worker

    x, y = _data()
    model = MLP(sizes, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena, **MOM)
    init = model.arena.weights.clone()
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(x, y)
    wk = Worker(None, None, model, ds, opt)
    schedule = _schedule()
    for b in range(STEPS):
        opt.lr = schedule(b)
        wk.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    return model, init


def _check_against_oracle(res, sizes, pp):
    from shallowspeed_b200.layers import MLP

    oracle, init = _oracle(sizes)
    init_model = MLP(sizes, 0, 1, GBS)
    init_model.arena.weights.copy_(init)
    got = []
    for s in range(pp):
        stage = MLP(sizes, s, pp, GBS)
        stage.arena.weights.copy_(res[s]["w"])
        got += list(stage.parameters())
    for i, (p0, pc, pg) in enumerate(zip(init_model.parameters(), oracle.parameters(), got)):
        assert _frob(pg.data - p0.data, pc.data - p0.data) < TOL, i


CASES = {
    "dp2-ll": dict(dp=2, pp=1),
    "dp4-ll": dict(dp=4, pp=1),
    "dp8-ll": dict(dp=8, pp=1),
    "dp2-wide-flags": dict(dp=2, pp=1, sizes=WIDE),
    "dp4-wide-flags": dict(dp=4, pp=1, sizes=WIDE),
    "dp8-two-shot": dict(dp=8, pp=1, env={"SSB_DP_TWO_SHOT": "1", "SSB_DP_LL": "0"}),
    "dp2-nccl": dict(dp=2, pp=1, comm="nccl"),
    "dp4-nccl": dict(dp=4, pp=1, comm="nccl"),
    "dp8-nccl": dict(dp=8, pp=1, comm="nccl"),
    "pp2-gpipe-peer": dict(dp=1, pp=2, transport="peer"),
    "pp2-gpipe-nccl": dict(dp=1, pp=2),
    "pp4-1f1b-peer": dict(dp=1, pp=4, sched="pipedream", transport="peer"),
    "pp4-1f1b-nccl": dict(dp=1, pp=4, sched="pipedream"),
    "pp4-gpipe-peer": dict(dp=1, pp=4, transport="peer"),
    "dp2xpp2-1f1b-peer": dict(dp=2, pp=2, sched="pipedream", transport="peer"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_schedule_matches_oracle(case, tmp_path):
    kw = dict(CASES[case])
    res = _spawn(tmp_path, **kw)
    _check_against_oracle(res, kw.get("sizes", REF), kw["pp"])


@pytest.mark.parametrize("dp", [2, 4, 8])
def test_schedule_nvls(dp, tmp_path):
    from shallowspeed_b200 import _C

    if torch.cuda.device_count() < dp or not _C.NvlsContext.supported():
        pytest.skip(f"needs {dp} GPUs with NVLink multicast")
    _check_against_oracle(_spawn(tmp_path, dp=dp, pp=1, comm="nvls"), REF, 1)


def test_checkpoint_resume_mid_schedule_is_bitwise(tmp_path):
    straight = _spawn(tmp_path, dp=2, pp=1)
    ck = tmp_path / "ck"
    _spawn(tmp_path, dp=2, pp=1, steps=3, ckpt=("save", str(ck)))
    resumed = _spawn(tmp_path, dp=2, pp=1, ckpt=("load", str(ck)))
    assert torch.equal(straight[0]["w"], resumed[0]["w"]) and torch.equal(straight[0]["v"], resumed[0]["v"])
