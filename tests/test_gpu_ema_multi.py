"""EMA of the weights on several H100s: every data-parallel transport (fused LL / flag protocol, NCCL, NVLS) and
pipeline layouts.  ``ema_state()`` must be identical on every replica and equal, bit for bit, to the reference lerp
replayed over the run's own per-step weights; the weights must equal those of the same run without EMA.  A layout
that needs more GPUs than the machine has is skipped."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

REF = [784, 128, 127, 126, 125, 124, 123, 10]
WIDE = [784, 1024, 1000, 1024, 520, 1024, 130, 10]
LR, GBS, N_MU, STEPS, DECAY = 0.05, 128, 4, 4, 0.6


def _rank_main(rank, world, dp, pp, port, comm, sizes, sched_name, opt_kw, ema, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.comm import ProcessGrid, make_torch_comms
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    grid = ProcessGrid(dp, pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    model = MLP(sizes, grid.stage, pp, GBS).to("cuda")
    opt = SGD(model.parameters(), LR, arena=model.arena, ema_decay=DECAY if ema else None, **opt_kw)
    x, y = synthetic_mnist(n=GBS * STEPS)
    ds = Dataset(None, GBS, GBS // dp // N_MU)
    ds.local_batch_size = GBS // dp
    ds.from_arrays(x[grid.replica::dp], y[grid.replica::dp])
    worker = NativeWorker(dp_comm, pp_comm, model, ds, opt, grid=grid, comm_mode=comm)
    sched = SCHEDULE_NAME_TO_CLS[sched_name](N_MU, pp, grid.stage)
    n = model.arena.numel
    weights = [model.arena.weights[:n].cpu().clone()]
    for b in range(STEPS):
        worker.execute(sched, b)
        worker.sync_to_model()
        weights.append(model.arena.weights[:n].cpu().clone())
    state = worker.ema_state()
    torch.save({"weights": weights, "ema": state, "blocks": model.arena.blocks, "offsets": model.arena.offsets,
                "lds": model.arena.lds, "updates": opt.ema_updates},
               os.path.join(out_dir, f"r{rank}_{int(ema)}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp_path, dp, pp, comm, sizes, sched, opt_kw, ema, port):
    import torch.multiprocessing as mp

    mp.spawn(_rank_main, args=(dp * pp, dp, pp, port, comm, sizes, sched, opt_kw, ema, str(tmp_path)), nprocs=dp * pp,
             join=True)


LAYOUTS = [(2, 1, "fused", REF, "naive"), (4, 1, "fused", REF, "naive"), (8, 1, "fused", REF, "naive"),
           (2, 1, "fused", WIDE, "naive"), (2, 1, "nccl", REF, "naive"), (4, 1, "nccl", REF, "naive"),
           (2, 1, "nvls", REF, "naive"), (4, 1, "nvls", REF, "naive"), (8, 1, "nvls", REF, "naive"),
           (1, 2, "fused", REF, "gpipe"), (1, 4, "fused", REF, "pipedream"), (2, 2, "fused", REF, "gpipe")]


@pytest.mark.parametrize("opt_kw", [{}, dict(momentum=0.9, weight_decay=1e-2)], ids=["plain", "momentum_wd"])
@pytest.mark.parametrize("dp,pp,comm,sizes,sched", LAYOUTS,
                         ids=[f"dp{d}_pp{p}_{c}_{'wide' if s is WIDE else 'ref'}" for d, p, c, s, _ in LAYOUTS])
def test_ema_state_is_the_replayed_reference(tmp_path, dp, pp, comm, sizes, sched, opt_kw):
    from shallowspeed_b200.ops.functional import ema_alpha, ema_lerp_ref

    if torch.cuda.device_count() < dp * pp:
        pytest.skip(f"needs {dp * pp} GPUs")
    port = 29700 + (hash((dp, pp, comm, sched, len(opt_kw), len(sizes))) % 200)
    _spawn(tmp_path, dp, pp, comm, sizes, sched, opt_kw, True, port)
    _spawn(tmp_path, dp, pp, comm, sizes, sched, opt_kw, False, port + 1)
    for rank in range(dp * pp):
        stage, replica = rank % pp, rank // pp
        a = torch.load(tmp_path / f"r{rank}_1.pt")
        b = torch.load(tmp_path / f"r{rank}_0.pt")
        assert a["updates"] == STEPS
        for wa, wb in zip(a["weights"], b["weights"]):
            assert torch.equal(wa, wb), "the EMA changed the weights"
        first = torch.load(tmp_path / f"r{stage}_1.pt")                 # replica 0 of the same stage
        assert torch.equal(a["ema"], first["ema"]), "ema_state() differs between replicas"
        mask = torch.zeros(a["ema"].numel(), dtype=torch.bool)
        for i, (o, k) in enumerate(a["blocks"]):
            mask[a["offsets"][i]: a["offsets"][i] + o * a["lds"][i]].view(o, a["lds"][i])[:, : k + 1] = True
        e = a["weights"][0].clone()
        for t in range(STEPS):
            e = ema_lerp_ref(e, a["weights"][t + 1], ema_alpha(DECAY, t))
        assert torch.equal(a["ema"][mask], e[mask])
        assert not bool(a["ema"][~mask].any())
