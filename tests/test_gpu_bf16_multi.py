"""``precision="bf16"`` on two H100s: data parallel (dp = 2) with the fused in-kernel reduction.  Each element is reduced
and updated once, by its owner, and published to the other replica, so the replicas must hold bit-identical weights
after every step; the run must also train (finite losses) and use the chain kernel.  Skipped below two GPUs."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

REF = [784, 128, 127, 126, 125, 124, 123, 10]
LR, GBS, N_MU, STEPS = 0.05, 128, 4, 4


def _rank_main(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import GPipeSchedule

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(world, 1, rank)
    dp_comm, _ = make_torch_comms(grid)
    model = MLP(REF, 0, 1, GBS).to("cuda")
    opt = SGD(model.parameters(), LR, arena=model.arena)
    x, y = synthetic_mnist(n=GBS * STEPS)
    ds = Dataset(None, GBS, GBS // world // N_MU, device="cuda")
    ds.local_batch_size = GBS // world
    ds.from_arrays(x[grid.replica::world], y[grid.replica::world])
    w = NativeWorker(dp_comm, None, model, ds, opt, grid=grid, comm_mode="fused", precision="bf16")
    sched = GPipeSchedule(N_MU, 1, 0)
    weights, losses = [], []
    for b in range(STEPS):
        w.execute(sched, b)
        losses.append(w.batch_loss())
        w.sync_to_model()
        weights.append(model.arena.weights[: model.arena.numel].cpu().clone())
    eng = w.engine_for(sched)
    torch.save({"w": weights, "losses": losses, "chain": bool(eng.uses_chain()), "describe": eng.describe()},
               os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_dp2_fused_replicas_are_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29400 + (os.getpid() + 7) % 300
    mp.spawn(_rank_main, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0, r1 = (torch.load(tmp_path / f"r{r}.pt") for r in range(world))
    assert r0["chain"] and r1["chain"], r0["describe"]
    assert all(torch.isfinite(torch.tensor(l)) for l in r0["losses"]), r0["losses"]
    for step, (a, b) in enumerate(zip(r0["w"], r1["w"])):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"replicas differ after step {step + 1}"
    assert not torch.equal(r0["w"][0], r0["w"][-1])
