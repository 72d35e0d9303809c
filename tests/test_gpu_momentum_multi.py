"""SGD momentum on several H100s: every data-parallel transport (LL, two-shot, flag protocol on the wide model, NCCL,
NVLS) and pipeline layouts against the CPU oracle, with momentum seeded non-zero so that one step exercises mu * v;
replicas bit-identical; the canonical momentum assembled by ``optimizer_state()`` equals the oracle's; a checkpoint
resume in a fresh process group equals the uninterrupted run."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

REF = [784, 128, 127, 126, 125, 124, 123, 10]
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]
MOM = dict(momentum=0.9, weight_decay=1e-2, nesterov=True)
LR, GBS, N_MU = 0.05, 128, 4


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _seed_v(arena):
    v0 = torch.zeros(arena.numel)
    gen = torch.Generator().manual_seed(3)
    for i, (o, k) in enumerate(arena.blocks):
        off, ld = arena.offsets[i], arena.lds[i]
        v0[off:off + o * ld].view(o, ld)[:, : k + 1] = torch.randn(o, k + 1, generator=gen) * 1e-3
    return v0


def _data(steps):
    from shallowspeed_b200.dataset import synthetic_mnist

    return synthetic_mnist(n=GBS * steps)


def _rank_main(rank, world, dp, pp, port, comm, env, sizes, sched_name, steps, out_dir, ckpt):
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
    model.arena.momentum.copy_(_seed_v(model.arena).cuda())
    first = 0
    if ckpt is not None and ckpt[0] == "load":
        first = load_stage(model, ckpt[1], grid.stage, pp, expect_hparams=MOM)
    x, y = _data(steps)
    ds = Dataset(None, GBS, GBS // dp // N_MU, device="cuda")
    ds.local_batch_size = GBS // dp
    ds.from_arrays(x[grid.replica::dp], y[grid.replica::dp])
    w = NativeWorker(dp_comm if dp > 1 else None, pp_comm if pp > 1 else None, model, ds, opt, grid=grid, comm_mode=comm)
    sched = SCHEDULE_NAME_TO_CLS[sched_name](N_MU, pp, grid.stage)
    for b in range(first, steps):
        w.execute(sched, b)
    w.sync_to_model()
    assert_sync(dp_comm, get_model_hash(model))
    state = w.optimizer_state()
    if ckpt is not None and ckpt[0] == "save" and grid.replica == 0:
        save_stage(model, ckpt[1], grid.stage, pp, step=steps, hparams=MOM, momentum=state)
    if grid.replica == 0:
        torch.save({"w": model.arena.weights[: model.arena.numel].cpu(), "v": state}, os.path.join(out_dir, f"s{grid.stage}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp, dp, pp, comm="fused", env=None, sizes=REF, sched="gpipe", steps=1, ckpt=None):
    import torch.multiprocessing as mp

    world = dp * pp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29700 + (os.getpid() + world * 7 + len(os.listdir(tmp))) % 300
    out = tmp / f"run{len(os.listdir(tmp))}"
    out.mkdir()
    mp.spawn(_rank_main, args=(world, dp, pp, port, comm, env or {}, sizes, sched, steps, str(out), ckpt), nprocs=world,
             join=True)
    return [torch.load(out / f"s{s}.pt") for s in range(pp)]


def _oracle(sizes, pp, steps=1):
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.pipe import NaiveParallelSchedule, Worker

    x, y = _data(steps)
    model = MLP(sizes, 0, 1, GBS)
    opt = SGD(model.parameters(), LR, arena=model.arena, **MOM)
    model.arena.momentum.copy_(_seed_v(model.arena))
    init = model.arena.weights.clone()
    ds = Dataset(None, GBS, GBS // N_MU)
    ds.local_batch_size = GBS
    ds.from_arrays(x, y)
    wk = Worker(None, None, model, ds, opt)
    for b in range(steps):
        wk.execute(NaiveParallelSchedule(N_MU, 1, 0), b)
    return model, init


def _check_against_oracle(res, sizes, pp):
    from shallowspeed_b200.layers import MLP

    oracle, init = _oracle(sizes, pp)
    ref_params = list(oracle.parameters())
    init_model = MLP(sizes, 0, 1, GBS)
    init_model.arena.weights.copy_(init)
    got, idx = [], 0
    for s in range(pp):
        stage = MLP(sizes, s, pp, GBS)
        stage.arena.weights.copy_(res[s]["w"])
        got += list(stage.parameters())
        # momentum of this stage against the oracle's, per block
        for i, (o, k) in enumerate(stage.arena.blocks):
            off, ld = stage.arena.offsets[i], stage.arena.lds[i]
            oi = idx + i
            vg = res[s]["v"][off:off + o * ld].view(o, ld)[:, : k + 1]
            ooff, old = oracle.arena.offsets[oi], oracle.arena.lds[oi]
            vc = oracle.arena.momentum[ooff:ooff + o * old].view(o, old)[:, : k + 1]
            v0 = _seed_v(oracle.arena)[ooff:ooff + o * old].view(o, old)[:, : k + 1]
            assert _frob(vg - 0.9 * v0, vc - 0.9 * v0) < 3e-3
        idx += len(stage.arena.blocks)
    for i, (p0, pc, pg) in enumerate(zip(init_model.parameters(), ref_params, got)):
        err = _frob(pg.data - p0.data, pc.data - p0.data)
        assert err < (1e-4 if i % 2 == 1 else 3e-3), (i, err)


CASES = {
    "dp2-ll": dict(dp=2, pp=1),
    "dp2-two-shot": dict(dp=2, pp=1, env={"SSB_DP_TWO_SHOT": "1", "SSB_DP_LL": "0"}),
    "dp2-nccl": dict(dp=2, pp=1, comm="nccl"),
    "pp2-gpipe": dict(dp=1, pp=2),
    "dp2xpp2-gpipe": dict(dp=2, pp=2),
    "dp8": dict(dp=8, pp=1),
    "dp2-wide": dict(dp=2, pp=1, sizes=WIDE),
}


@pytest.mark.parametrize("case", list(CASES))
def test_momentum_one_step_matches_oracle(case, tmp_path):
    kw = dict(CASES[case])
    res = _spawn(tmp_path, **kw)
    _check_against_oracle(res, kw.get("sizes", REF), kw["pp"])


def test_momentum_nvls(tmp_path):
    from shallowspeed_b200 import _C

    if torch.cuda.device_count() < 2 or not _C.NvlsContext.supported():
        pytest.skip("needs 2 GPUs with NVLink multicast")
    _check_against_oracle(_spawn(tmp_path, dp=2, pp=1, comm="nvls"), REF, 1)


def test_sharded_momentum_checkpoint_resume_is_bitwise(tmp_path):
    straight = _spawn(tmp_path, dp=2, pp=1, steps=4)
    ck = tmp_path / "ck"
    _spawn(tmp_path, dp=2, pp=1, steps=2, ckpt=("save", str(ck)))
    resumed = _spawn(tmp_path, dp=2, pp=1, steps=4, ckpt=("load", str(ck)))
    assert torch.equal(straight[0]["w"], resumed[0]["w"]) and torch.equal(straight[0]["v"], resumed[0]["v"])
