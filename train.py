#!/usr/bin/env python
"""Training driver.  Same CLI as the reference's ``train.py`` (``--dp/--pp/--schedule``,
train.py:63-76) - plus the knobs the reference hard-codes as module constants
(train.py:56-59, 98, 107, 111) and the GPU runtime options.

Launch (one process per GPU / per (dp, pp) cell):

    python train.py                                          # sequential, dp=1 pp=1
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 train.py --dp 8
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 train.py --dp 2 --pp 4 --schedule gpipe
    python train.py --spawn --dp 2 --pp 2 --device cpu        # self-spawning (gloo) for laptops

The reference is launched with ``mpirun -n DP*PP`` (README.md:29-38); ``torchrun`` (or
``--spawn``) replaces it, ``torch.distributed`` process groups replace ``COMM_WORLD.Split``.
"""
from __future__ import annotations

import argparse
import os
import time
from pathlib import Path

import torch

from shallowspeed_b200.dataset import Dataset
from shallowspeed_b200.layers import MLP, mlp_sizes
from shallowspeed_b200.lr_schedule import DEFAULT_WARMUP_START_FACTOR, KINDS as LR_SCHEDULES, LRSchedule
from shallowspeed_b200.models.mlp import DEFAULT_LAYER_SIZES
from shallowspeed_b200.optimizer import SGD
from shallowspeed_b200.parallel.comm import ProcessGrid, SelfComm, make_torch_comms
from shallowspeed_b200.pipe import (GPipeSchedule, InferenceSchedule, NaiveParallelSchedule,
                                    PipeDreamSchedule, Worker)
from shallowspeed_b200.utils import StepLogger, assert_sync, get_model_hash

SCHEDULE_NAME_TO_CLS = {
    "naive": NaiveParallelSchedule,
    "gpipe": GPipeSchedule,
    "pipedream": PipeDreamSchedule,
    "pipedream-flush": PipeDreamSchedule,
}

EPOCHS = 20
GLOBAL_BATCH_SIZE = 128
N_MUBATCHES = 4
LEARNING_RATE = 0.006


def compute_accuracy(model, worker, dataset):
    """Forward the whole validation set through the pipeline (InferenceSchedule), compare
    argmax(pred) with argmax(target) on the last stage (reference train.py:21-47)."""
    model.eval()
    correct = 0
    total = 0
    for batch_id in range(dataset.get_num_batches()):
        schedule = InferenceSchedule(num_micro_batches=1, num_stages=worker.pipeline_depth,
                                     stage_id=worker.stage_id)
        worker.execute(schedule, batch_id)
        if worker.stage_id == worker.pipeline_depth - 1:
            pred = worker.output_buffers[0].argmax(dim=-1)
            target = dataset.load_micro_batch_target(batch_id, 0).to(pred.device).argmax(dim=-1)
            correct += int((pred == target).sum())
            total += pred.shape[0]
    model.train()
    if worker.stage_id == worker.pipeline_depth - 1:
        return correct / total


def build_parser():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--dp", type=int, default=1, help="Degree of data parallelism (=number of full model replicas)")
    p.add_argument("--pp", type=int, default=1, help="Number of pipeline stages")
    p.add_argument("--schedule", type=str, choices=sorted(SCHEDULE_NAME_TO_CLS), default="naive")
    # knobs the reference hard-codes
    p.add_argument("--epochs", type=int, default=EPOCHS)
    p.add_argument("--steps", type=int, default=None, help="stop after this many training steps (overrides --epochs)")
    p.add_argument("--global-batch-size", type=int, default=GLOBAL_BATCH_SIZE)
    p.add_argument("--n-mubatches", type=int, default=N_MUBATCHES)
    p.add_argument("--lr", type=float, default=LEARNING_RATE)
    p.add_argument("--lr-schedule", choices=LR_SCHEDULES, default="constant",
                   help="learning rate after the warmup: constant, step (StepLR), cosine (CosineAnnealingLR to --lr-min) "
                        "or linear (linear decay to --lr-min); --lr is the base rate")
    p.add_argument("--warmup-steps", type=int, default=0, help="linear warmup over this many steps (LinearLR)")
    p.add_argument("--warmup-start-factor", type=float, default=DEFAULT_WARMUP_START_FACTOR,
                   help="the first warmup step runs at this fraction of --lr, in (0, 1]")
    p.add_argument("--lr-min", type=float, default=0.0, help="cosine / linear: the rate the decay ends at")
    p.add_argument("--lr-step-size", type=int, default=None, help="step: steps between two decays by --lr-gamma")
    p.add_argument("--lr-gamma", type=float, default=0.1, help="step: decay factor")
    p.add_argument("--lr-total-steps", type=int, default=None,
                   help="cosine / linear: the schedule's horizon in steps (default: this run's total steps; set it when "
                        "a run is split into several invocations with --save / --resume)")
    p.add_argument("--momentum", type=float, default=0.0, help="SGD momentum (torch.optim.SGD semantics, dampening 0)")
    p.add_argument("--weight-decay", type=float, default=0.0, help="L2 penalty added to the gradient (biases included)")
    p.add_argument("--nesterov", action="store_true", help="Nesterov momentum (needs --momentum > 0)")
    p.add_argument("--loss", choices=["mse", "cross-entropy"], default="mse",
                   help="mse: the reference's softmax + MSE; cross-entropy: softmax cross-entropy on the logits")
    p.add_argument("--layer-sizes", type=int, nargs="+", default=None, help="explicit layer widths (default: reference MLP)")
    p.add_argument("--hidden", type=int, default=None, help="with --n-layers: 784 -> hidden x (n-1) -> 10")
    p.add_argument("--n-layers", type=int, default=None)
    p.add_argument("--seed-mode", choices=["shape", "index"], default="shape")
    p.add_argument("--data-dir", type=str, default="data/mnist_784/")
    p.add_argument("--synthetic", action="store_true", help="force synthetic MNIST-shaped data")
    p.add_argument("--no-eval", action="store_true", help="skip the per-epoch validation pass")
    # runtime
    p.add_argument("--device", choices=["auto", "cpu", "cuda"], default="auto")
    p.add_argument("--engine", choices=["auto", "python", "native"], default="auto",
                   help="python = portable instruction VM; native = C++ executor + sm_90a kernels")
    p.add_argument("--comm", choices=["fused", "nccl", "nvls"], default="fused",
                   help="native engine DP path: in-kernel reduction over peer memory, or plain NCCL all-reduce (A/B baseline)")
    p.add_argument("--pp-transport", choices=["nccl", "peer"], default=None,
                   help="native engine, stage boundaries: one-sided pushes into the neighbour's memory over NVLink with "
                        "epoch flags (peer; the default through SSB_PP_PEER in tuning.json) or NCCL send/recv")
    p.add_argument("--no-graph", action="store_true", help="native engine: do not capture the step in a CUDA graph")
    p.add_argument("--precision", choices=["tf32", "fp32"], default="fp32",
                   help="tensor-core math: fp32 = 3xTF32 split (fp32-equivalent, the reference's contract); tf32 = single pass")
    p.add_argument("--watchdog-s", type=float, default=None,
                   help="native engine: abort (and tear the NCCL communicators down) if an epoch's work is still in "
                        "flight after this many seconds; default: SSB_WATCHDOG_S or disabled")
    p.add_argument("--spawn", action="store_true", help="spawn dp*pp local processes instead of relying on torchrun")
    p.add_argument("--log-json", type=str, default=None, help="write JSON-lines metrics here (rank 0)")
    p.add_argument("--save", type=str, default=None, help="directory for per-stage checkpoints at the end of training")
    p.add_argument("--resume", type=str, default=None, help="directory with per-stage checkpoints to load")
    return p


def resolve_sizes(args):
    if args.layer_sizes:
        return list(args.layer_sizes)
    if args.hidden or args.n_layers:
        return mlp_sizes(args.hidden or 128, args.n_layers or 7)
    return list(DEFAULT_LAYER_SIZES)


def init_distributed(args, device_type):
    import torch.distributed as dist

    world = args.dp * args.pp
    env_world = int(os.environ.get("WORLD_SIZE", "1"))
    assert env_world == world, (
        f"Number of started workers is {env_world}, but should be {world} (DP * PP)")
    if world == 1:
        return ProcessGrid(1, 1, 0), SelfComm(), SelfComm()
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29511")
    rank = int(os.environ["RANK"])
    if device_type == "cuda":
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    else:  # several CPU ranks on one host: do not oversubscribe the cores
        torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))
    if not dist.is_initialized():
        dist.init_process_group("nccl" if device_type == "cuda" else "gloo", rank=rank, world_size=world)
    grid = ProcessGrid(args.dp, args.pp, rank)
    dp_comm, pp_comm = make_torch_comms(grid)
    assert dp_comm.Get_size() == args.dp and pp_comm.Get_size() == args.pp
    return grid, dp_comm, pp_comm


def main(args):
    assert args.dp >= 1 and args.pp >= 1
    assert args.global_batch_size % args.dp == 0, "Batch size must be properly divisible by DP"
    device_type = args.device
    if device_type == "auto":
        device_type = "cuda" if torch.cuda.is_available() else "cpu"
    grid, dp_comm, pp_comm = init_distributed(args, device_type)
    device = torch.device("cuda", torch.cuda.current_device()) if device_type == "cuda" else torch.device("cpu")
    engine = args.engine
    if engine == "auto":
        engine = "native" if device_type == "cuda" else "python"

    layer_sizes = resolve_sizes(args)
    sched_cls = SCHEDULE_NAME_TO_CLS[args.schedule]
    local_batch_size = args.global_batch_size // args.dp
    assert local_batch_size % args.n_mubatches == 0, "n-mubatches must divide the DP-local batch"
    save_dir = Path(args.data_dir)
    synthetic = args.synthetic or not (save_dir / "x_train.parquet").exists()
    logger = StepLogger(args.log_json, rank=grid.rank)
    is_last = pp_comm.Get_rank() == args.pp - 1

    loss = args.loss.replace("-", "_")
    model = MLP(layer_sizes, stage_idx=pp_comm.Get_rank(), n_stages=args.pp,
                batch_size=args.global_batch_size, seed_mode=args.seed_mode,
                verbose=(grid.rank == 0 or is_last), loss=loss)
    model.to(device)
    model.train()
    # before the resume: the momentum arena it restores is allocated here
    optimizer = SGD(model.parameters(), lr=args.lr, momentum=args.momentum, weight_decay=args.weight_decay,
                    nesterov=args.nesterov, arena=model.arena)

    dataset = Dataset(save_dir, global_batch_size=args.global_batch_size,
                      mubatch_size=local_batch_size // args.n_mubatches, validation=False,
                      synthetic=synthetic, device=device)
    dataset.load(dp_comm.Get_rank(), dp_comm.Get_size())
    val_dataset = Dataset(save_dir, global_batch_size=args.global_batch_size,
                          mubatch_size=args.global_batch_size, validation=True,
                          synthetic=synthetic, device=device)
    val_dataset.load(DP_rank=0, DP_size=1)

    n_batches = dataset.get_num_batches()
    total_steps = args.steps if args.steps is not None else args.epochs * n_batches
    lr_schedule = LRSchedule(args.lr, args.lr_schedule, total_steps=args.lr_total_steps or total_steps,
                             warmup_steps=args.warmup_steps, warmup_start_factor=args.warmup_start_factor,
                             min_lr=args.lr_min, step_size=args.lr_step_size, gamma=args.lr_gamma)
    hparams = {"lr": float(args.lr), "global_batch_size": int(args.global_batch_size), "seed_mode": str(args.seed_mode),
               "n_mubatches": int(args.n_mubatches), "momentum": float(args.momentum),
               "weight_decay": float(args.weight_decay), "nesterov": bool(args.nesterov), "loss": loss,
               "lr_schedule": lr_schedule.spec()}
    resumed_step = 0
    if args.resume:
        from shallowspeed_b200.utils.checkpoint import load_stage

        resumed_step = load_stage(model, args.resume, pp_comm.Get_rank(), args.pp, expect_hparams=hparams)

    if engine == "native":
        from shallowspeed_b200.parallel.engine import NativeWorker

        worker = NativeWorker(dp_comm, pp_comm, model, dataset, optimizer, grid=grid, comm_mode=args.comm,
                              use_graph=not args.no_graph, precision=args.precision, pp_transport=args.pp_transport)
        val_worker = NativeWorker(None, pp_comm, model, val_dataset, None, grid=grid, comm_mode="nccl",
                                  use_graph=not args.no_graph, precision=args.precision, share=worker,
                                  pp_transport=args.pp_transport)
    else:
        worker = Worker(dp_comm, pp_comm, model, dataset, optimizer, device=device)
        val_worker = Worker(None, pp_comm, model, val_dataset, None, device=device)

    start_time = time.time()
    # a resumed run continues where the checkpoint stopped: same global step, same position in the data
    step = min(resumed_step, total_steps)
    epoch = step // n_batches
    first_batch = step % n_batches
    # the schedule is identical for every batch: build it once (the reference rebuilds
    # a Python object per batch, train.py:140-144)
    schedule = sched_cls(num_micro_batches=args.n_mubatches, num_stages=args.pp, stage_id=pp_comm.Get_rank())
    while step < total_steps:
        if not args.no_eval:
            accuracy = compute_accuracy(model, val_worker, val_dataset)
            if accuracy is not None:
                print(f"Epoch: {epoch}, Time Spent: {time.time() - start_time:.2f}s, Accuracy: {accuracy * 100:.2f}%",
                      flush=True)
                if dp_comm.Get_rank() == 0:
                    logger.log(event="eval", epoch=epoch, step=step, accuracy=accuracy,
                               time_s=time.time() - start_time)
        t_epoch = time.time()
        steps_this_epoch = min(n_batches - first_batch, total_steps - step)
        for batch_id in range(first_batch, first_batch + steps_this_epoch):
            optimizer.lr = lr_schedule(step)        # both engines read the optimizer's rate when the step starts
            worker.execute(schedule, batch_id)
            step += 1
        first_batch = 0
        if engine == "native":
            from shallowspeed_b200.parallel.engine import watchdog_seconds

            worker.guard(worker._last_engine, watchdog_seconds(args.watchdog_s), what=f"epoch {epoch}")
        if device_type == "cuda":
            torch.cuda.synchronize()
        dt = time.time() - t_epoch
        logger.log(event="epoch", epoch=epoch, steps=steps_this_epoch,
                   samples_per_s=steps_this_epoch * args.global_batch_size / max(dt, 1e-9),
                   ms_per_step=1e3 * dt / max(steps_this_epoch, 1), loss=worker.batch_loss())
        epoch += 1

    if not args.no_eval:
        accuracy = compute_accuracy(model, val_worker, val_dataset)
        if accuracy is not None:
            print(f"Epoch: {epoch}, Time Spent: {time.time() - start_time:.2f}s, Accuracy: {accuracy * 100:.2f}%",
                  flush=True)

    if hasattr(worker, "sync_to_model"):
        worker.sync_to_model()
    # Sanity check: data parallel replicas must hold bit-identical weights
    assert_sync(dp_comm, get_model_hash(model))
    if args.save:
        from shallowspeed_b200.utils.checkpoint import save_stage

        if engine == "native":
            momentum = worker.optimizer_state()
        else:
            momentum = model.arena.momentum if optimizer.momentum > 0.0 else None
        if dp_comm.Get_rank() == 0:
            save_stage(model, args.save, pp_comm.Get_rank(), args.pp, step=step, hparams=hparams, momentum=momentum)
    logger.close()
    if args.dp * args.pp > 1:
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()


def _spawn_entry(rank, args, port):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(args.dp * args.pp),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    main(args)


if __name__ == "__main__":
    args = build_parser().parse_args()
    if args.spawn and args.dp * args.pp > 1:
        import torch.multiprocessing as mp

        port = 29500 + (os.getpid() % 2000)
        args.spawn = False
        mp.spawn(_spawn_entry, args=(args, port), nprocs=args.dp * args.pp, join=True)
    else:
        if args.dp * args.pp == 1:
            os.environ.setdefault("WORLD_SIZE", "1")
        main(args)
