"""Python face of the native pipeline executor (``csrc/runtime/pipe_engine.cpp``).

``NativeWorker`` has the surface of the reference's ``Worker`` (``execute(sched,
batch_id)``, ``output_buffers``, ``stage_id``, ``pipeline_depth``; pipe.py:330-466) but
lowers each distinct schedule ONCE into a static CUDA-graph plan and replays it.

``Trainer`` is the user-facing end-to-end API (``trainer.step(x_host, y_host) -> loss``):
inputs come from pinned host memory, one H2D copy per step, loss read back per step.
"""
from __future__ import annotations

from typing import Optional

import torch

from ..ops.functional import ACTIVATION_CODES, LOSS_CODES, precision_code
from .comm import Comm, ProcessGrid, SelfComm, TorchComm
from .instructions import encode, flatten
from .schedules import Schedule
from .validate import simulate

DP_MODE = {"none": 0, "nccl": 1, "fused": 2, "nvls": 3}


class StepTimeout(RuntimeError):
    """A training step did not finish within the watchdog's bound (dead peer, lost message, schedule bug)."""


def watchdog_seconds(explicit=None):
    """Watchdog bound in seconds: the explicit argument, else ``SSB_WATCHDOG_S``, else None (disabled)."""
    import os

    if explicit is not None:
        return float(explicit) if explicit > 0 else None
    env = os.environ.get("SSB_WATCHDOG_S", "")
    return float(env) if env and float(env) > 0 else None


def _C():
    from .. import _C as mod

    return mod


def make_dp_context(comm: Comm, model, lr: float):
    """Symmetric memory for the fused DP kernels: allocate, exchange CUDA IPC handles over
    torch.distributed, map the peers, and move the model's weight arena into it."""
    assert isinstance(comm, TorchComm)
    import torch.distributed as dist

    arena = model.arena
    layers = [(lin.in_dims, lin.out_dims, int(arena.offsets[lin.block_index]), int(arena.lds[lin.block_index]))
              for lin in model.linears]
    ctx = _C().DpContext(comm.size, comm.rank, int(arena.weights.numel()), layers, float(lr))
    blobs = [None] * comm.size
    dist.all_gather_object(blobs, bytes(ctx.export_handles()), group=comm.group)
    ctx.open_peers(blobs)
    arena.rebind(ctx.weights(), arena.grads, copy=True)      # weights now live in symmetric memory
    torch.cuda.synchronize()
    dist.barrier(group=comm.group)
    return ctx


# ----------------------------------------------------------------------------------------------------------
# NVLS (switch-side reduction): the multicast object is created by the DP group's leader and reaches the other
# replicas as a POSIX file descriptor over an AF_UNIX socket (SCM_RIGHTS) - file descriptors cannot travel
# through torch.distributed.
# ----------------------------------------------------------------------------------------------------------
def serve_fd(path: str, fd: int, n_peers: int, timeout_s: float = 120.0):
    """Leader side: hand ``fd`` to ``n_peers`` clients connecting to the unix socket ``path``."""
    import os
    import socket

    if os.path.exists(path):
        os.unlink(path)
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(path)
    srv.listen(max(1, n_peers))
    srv.settimeout(timeout_s)
    return srv


def serve_fd_finish(srv, path: str, fd: int, n_peers: int):
    import os
    import socket

    import struct

    try:
        for _ in range(n_peers):
            conn, _addr = srv.accept()
            with conn:
                # only processes of the same user may receive the multicast handle
                cred = conn.getsockopt(socket.SOL_SOCKET, socket.SO_PEERCRED, struct.calcsize("3i"))
                _pid, uid, _gid = struct.unpack("3i", cred)
                if uid != os.getuid():
                    raise PermissionError(f"NVLS fd exchange: connection from uid {uid}, expected {os.getuid()}")
                socket.send_fds(conn, [b"ssb-nvls"], [fd])
    finally:
        srv.close()
        if os.path.exists(path):
            os.unlink(path)


def recv_fd(path: str, timeout_s: float = 120.0) -> int:
    """Peer side: connect to the leader's socket and receive one file descriptor."""
    import socket
    import time

    deadline = time.time() + timeout_s
    while True:
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        try:
            c.connect(path)
            break
        except (FileNotFoundError, ConnectionRefusedError):
            c.close()
            if time.time() > deadline:
                raise
            time.sleep(0.01)
    with c:
        c.settimeout(timeout_s)
        msg, fds, _flags, _addr = socket.recv_fds(c, 64, 1)
    if msg != b"ssb-nvls" or len(fds) != 1:
        raise RuntimeError(f"NVLS fd exchange: unexpected message {msg!r} with {len(fds)} descriptors")
    return fds[0]


def make_nvls_context(comm: Comm, model, lr: float):
    """Collective over the DP group: create / import the multicast object, bind this replica's memory, and move the
    model's weight AND gradient arenas into it (the NVLS kernel reduces G through the switch and multicasts W)."""
    assert isinstance(comm, TorchComm)
    import os

    import torch.distributed as dist

    C = _C()
    if not C.NvlsContext.supported():
        raise RuntimeError("--comm nvls: this device / driver does not support NVLink multicast (NVLS); use --comm fused")
    arena = model.arena
    ctx = C.NvlsContext(comm.size, comm.rank, int(arena.weights.numel()), float(lr))
    leader = comm.rank == 0
    box = [None]
    srv = fd = None
    sock_dir = None
    if leader:
        import tempfile

        fd = ctx.export_fd()
        sock_dir = tempfile.mkdtemp(prefix="ssb_nvls_")  # mode 0700, unpredictable name: no symlink / squatting games in /tmp
        box[0] = os.path.join(sock_dir, "fd.sock")
        srv = serve_fd(box[0], fd, comm.size - 1)       # listening BEFORE the path is announced
    dist.broadcast_object_list(box, src=comm.ranks[0], group=comm.group)
    if leader:
        serve_fd_finish(srv, box[0], fd, comm.size - 1)
        os.close(fd)
        os.rmdir(sock_dir)
    else:
        got = recv_fd(box[0])
        ctx.import_fd(got)
        os.close(got)                                    # the imported handle keeps its own reference
    dist.barrier(group=comm.group)
    ctx.add_device()
    dist.barrier(group=comm.group)                       # every device is part of the team before anyone binds
    ctx.bind_and_map()
    dist.barrier(group=comm.group)
    arena.rebind(ctx.weights(), ctx.grads(), copy=True)  # parameters and gradients now live in NVLS memory
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    dist.barrier(group=comm.group)
    return ctx


def make_pp_context(comm: Comm, eng, n_mu: int, mb_rows: int, is_first: bool, is_last: bool):
    """Collective over the pipeline group: receive slots + flags of this stage in IPC-shared memory, mapped by the two
    neighbours (peer-memory boundary transport, ``--pp-transport peer``)."""
    assert isinstance(comm, TorchComm)
    import torch.distributed as dist

    ld_in, ld_out = eng.boundary_lds()
    ctx = _C().PpContext(int(n_mu), int(mb_rows), int(ld_in), int(ld_out), bool(is_first), bool(is_last))
    blobs = [None] * comm.size
    dist.all_gather_object(blobs, (bytes(ctx.export_handles()), int(ld_in), int(ld_out)), group=comm.group)
    if not is_first:
        h, _pin, pout = blobs[comm.rank - 1]
        assert pout == ld_in, f"stage boundary mismatch: predecessor writes rows of {pout} floats, this stage reads {ld_in}"
        ctx.open_prev(h)
    if not is_last:
        h, nin, _nout = blobs[comm.rank + 1]
        assert nin == ld_out, f"stage boundary mismatch: successor reads rows of {nin} floats, this stage writes {ld_out}"
        ctx.open_next(h)
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    dist.barrier(group=comm.group)
    return ctx


def make_nccl_comm(comm: Comm):
    """Create a native ncclComm for the ranks of a ``TorchComm`` (unique id travels over
    torch.distributed).  Returns None for size-1 communicators."""
    if comm is None or comm.Get_size() == 1:
        return None
    assert isinstance(comm, TorchComm), "native engine needs torch.distributed (NCCL) communicators"
    import torch.distributed as dist

    box = [_C().NcclComm.unique_id() if comm.rank == 0 else None]
    dist.broadcast_object_list(box, src=comm.ranks[0], group=comm.group)
    nc = _C().NcclComm(box[0], comm.size, comm.rank)
    nc.warmup()
    return nc


class NativeWorker:
    def __init__(self, dp_comm, pp_comm, model, dataset, optimizer, grid: Optional[ProcessGrid] = None,
                 comm_mode: str = "fused", use_graph: bool = True, precision: str = "fp32", share=None,
                 validate_schedules: bool = True, pp_transport: Optional[str] = None):
        self.dp_comm = dp_comm if dp_comm is not None else SelfComm()
        self.pp_comm = pp_comm if pp_comm is not None else SelfComm()
        self.stage_id = self.pp_comm.Get_rank()
        self.pipeline_depth = self.pp_comm.Get_size()
        self.model, self.dataset, self.optimizer = model, dataset, optimizer
        self.use_graph, self.precision = use_graph, precision
        precision_code(precision)   # ValueError now for a name the engine does not know
        self.validate_schedules = validate_schedules
        # pipeline boundaries: one-sided pushes into the neighbour's memory (None = "peer") or NCCL send/recv ("nccl")
        self.pp_transport = pp_transport or "peer"
        assert self.pp_transport in ("nccl", "peer")
        self.device = model.arena.weights.device
        assert self.device.type == "cuda", "NativeWorker needs the model on a CUDA device (model.to('cuda'))"
        if self.dp_comm.Get_size() == 1:
            self.dp_mode = "none"
        else:
            self.dp_mode = comm_mode
        # native communicators are shared between the train and the validation worker
        # the update rule beyond lr (optimizer.SGD); the engine keeps the momentum in the model arena's buffer
        self.momentum = float(getattr(optimizer, "momentum", 0.0) or 0.0)
        self.weight_decay = float(getattr(optimizer, "weight_decay", 0.0) or 0.0)
        self.nesterov = bool(getattr(optimizer, "nesterov", False))
        if self.momentum > 0.0 and getattr(optimizer, "arena", None) is not model.arena:
            raise ValueError("NativeWorker: SGD with momentum must be built with arena=model.arena (the engine keeps the "
                             "momentum in the arena's buffer)")
        self.ema_decay = getattr(optimizer, "ema_decay", None)
        if self.ema_decay is not None and getattr(optimizer, "arena", None) is not model.arena:
            raise ValueError("NativeWorker: SGD with an EMA must be built with arena=model.arena (the engine keeps the "
                             "EMA in the arena's buffer)")
        self._dp_ctx = None
        self._nvls_ctx = None
        # Engines that share a communicator (train + validation worker on one pipeline group) run on their own
        # non-blocking streams.  NCCL matches p2p operations in issue order per peer and forbids concurrent use of one
        # communicator, so successive engines are ordered explicitly: ``_order["last"]`` is the engine whose work was
        # enqueued last on the shared communicators (see ``_enter``).
        self._order = share._order if share is not None else {"last": None}
        if share is not None:
            self._pp_nccl, self._dp_nccl = share._pp_nccl, share._dp_nccl
        else:
            self._pp_nccl = make_nccl_comm(self.pp_comm)
            self._dp_nccl = None
            if dp_comm is not None and self.dp_comm.Get_size() > 1:
                if self.dp_mode == "fused":
                    self._dp_ctx = make_dp_context(self.dp_comm, model, self.lr)
                elif self.dp_mode == "nvls":
                    self._nvls_ctx = make_nvls_context(self.dp_comm, model, self.lr)
                else:
                    self._dp_nccl = make_nccl_comm(self.dp_comm)
        self._engines = {}
        self._last_engine = None
        self._train_engine = None      # the training plan whose DP protocols decide who owns which momentum entries

    @property
    def lr(self):
        """The optimizer's current learning rate: the rate the next training step runs with."""
        return self.optimizer.lr if self.optimizer is not None else 0.0

    def set_lr(self, eng, sched: Schedule):
        """Hand the optimizer's current learning rate to ``eng`` before it runs a training step (the engine rewrites
        its device slot only when the value changed).  Every call precedes exactly one run of ``eng``, so a training
        call also hands over the alpha of that step's EMA update and counts the update."""
        if sched.training and self.optimizer is not None:
            eng.set_lr(float(self.optimizer.lr))
            if self.ema_decay is not None:
                eng.set_ema_alpha(float(self.optimizer.ema_alpha))
                self.optimizer.ema_updates += 1
        if sched.training and getattr(self.model, "dropout", 0.0) > 0.0:   # the step whose dropout masks this step draws
            eng.set_dropout_step(int(self.model.dropout_step))

    # ------------------------------------------------------------------ plan cache
    def _key(self, sched: Schedule):
        return (type(sched).__name__, sched.num_micro_batches, sched.num_stages, sched.stage_id,
                self.dataset.mubatch_size)

    def _build(self, sched: Schedule):
        if self.validate_schedules:   # prove the whole pipeline deadlock-free before touching the GPU
            simulate([type(sched)(sched.num_micro_batches, sched.num_stages, s) for s in range(sched.num_stages)])
        m = self.model
        specs = []
        for lin in m.linears:
            specs.append((lin.in_dims, lin.out_dims, 1 if lin.activation is not None else 0,
                          int(m.arena.offsets[lin.block_index]), int(m.arena.lds[lin.block_index])))
        training = bool(sched.training)
        cfg = dict(is_first=int(sched.is_first_stage), is_last=int(sched.is_last_stage), stage=sched.stage_id,
                   n_stages=sched.num_stages, mb_rows=self.dataset.mubatch_size, n_mu=sched.num_micro_batches,
                   global_batch=m.batch_size, lr=float(self.lr), training=int(training), use_graph=int(self.use_graph),
                   dp_size=self.dp_comm.Get_size(), dp_rank=self.dp_comm.Get_rank(),
                   dp_mode=DP_MODE[self.dp_mode] if training else 0, in_dim=m.in_dim, out_dim=m.out_dim,
                   prec=precision_code(self.precision))
        momentum = None
        if training and (self.momentum != 0.0 or self.weight_decay != 0.0):
            cfg.update(momentum=self.momentum, weight_decay=self.weight_decay, nesterov=int(self.nesterov))
            momentum = m.arena.momentum if self.momentum > 0.0 else None
        ema = None
        if training and self.ema_decay is not None:
            cfg.update(ema_decay=self.ema_decay)
            ema = m.arena.ema
        if m.loss != "mse":   # the head's loss kind (training and inference: the probabilities depend on it)
            cfg.update(loss=LOSS_CODES[m.loss])
        if getattr(m, "activation", "relu") != "relu":   # training and inference: f applies in both
            cfg.update(activation=ACTIVATION_CODES[m.activation])
        if getattr(m, "residual", False):   # training and inference: the skips apply in both
            cfg.update(residual=[int(lin.residual) for lin in m.linears])
        if training and getattr(m, "dropout", 0.0) > 0.0:   # inference plans run without dropout
            cfg.update(dropout=m.dropout, dropout_seed=m.dropout_seed, layer_base=m.layer_base)
        eng = _C().PipeEngine(specs, cfg, m.arena.weights, m.arena.grads, momentum, ema)
        if self._pp_nccl is not None:
            eng.set_pp_comm(self._pp_nccl)
        if self._dp_nccl is not None and training:
            eng.set_dp_comm(self._dp_nccl)
        if self._dp_ctx is not None and training:
            eng.set_dp_context(self._dp_ctx)
        if self._nvls_ctx is not None and training:
            eng.set_nvls_context(self._nvls_ctx)
        if self.pp_transport == "peer" and self.pipeline_depth > 1:
            eng.set_pp_context(make_pp_context(self.pp_comm, eng, sched.num_micro_batches, self.dataset.mubatch_size,
                                               sched.is_first_stage, sched.is_last_stage))
        torch.cuda.synchronize(self.device)
        eng.build([encode(i) for i in flatten(list(sched.steps()))])
        if training:
            self._train_engine = eng
        return eng

    def engine_for(self, sched: Schedule):
        key = self._key(sched)
        eng = self._engines.get(key)
        if eng is None:
            eng = self._engines[key] = self._build(sched)
        return eng

    # ------------------------------------------------------------------ Worker surface
    def _enter(self, eng):
        """Order ``eng`` behind whichever engine used the shared communicators last (train <-> validation switches).
        An engine's main stream joins all of its side streams at the end of a run, and its next run forks from the main
        stream, so one event edge main(prev) -> main(eng) serialises every NCCL operation of the two engines, on every
        stage, without a host synchronisation."""
        prev = self._order["last"]
        if prev is not None and prev is not eng:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.ExternalStream(prev.main_stream(), device=self.device))
            torch.cuda.ExternalStream(eng.main_stream(), device=self.device).wait_event(ev)
        self._order["last"] = eng

    def execute(self, sched: Schedule, batch_id: int):
        eng = self.engine_for(sched)
        ds = self.dataset
        if getattr(ds, "shuffle", False):
            # the whole file stays on the device; the engine gathers this rank's rows of the epoch's permutation itself
            if ds.input_X.device != self.device:
                raise ValueError(f"a shuffled dataset must live on the engine's device {self.device}, "
                                 f"not {ds.input_X.device} (Dataset(..., device=...))")
            assert 0 <= batch_id < ds.get_num_batches()
            self._enter(eng)
            self.set_lr(eng, sched)
            eng.stage_gather(ds.input_X if sched.is_first_stage else None, ds.target_y if sched.is_last_stage else None,
                             ds.shuffle_seed, ds.epoch, ds.global_batch_size, ds.dp_size, ds.dp_rank, batch_id)
            eng.run()
            self._last_engine = eng
            return
        x, y = ds.load_batch(batch_id)
        self._enter(eng)
        self.set_lr(eng, sched)
        eng.stage_inputs(x if sched.is_first_stage else None, y if sched.is_last_stage else None)
        eng.run()
        self._last_engine = eng

    def step_from(self, sched: Schedule, x, y):
        """Run one step on explicit (pinned-host or device) batch tensors."""
        eng = self.engine_for(sched)
        self._enter(eng)
        self.set_lr(eng, sched)
        eng.stage_inputs(x if sched.is_first_stage else None, y if sched.is_last_stage else None)
        eng.run()
        self._last_engine = eng
        return eng

    @property
    def output_buffers(self):
        """Inference: softmax output of micro-batch 0 on the last stage (train.py reads
        ``worker.output_buffers[0]``)."""
        eng = self._last_engine
        eng.synchronize()
        return [eng.probs(mu) for mu in range(int(eng.n_mubatches()))]

    def batch_loss(self):
        if self._last_engine is None or self.stage_id != self.pipeline_depth - 1:
            return None
        return float(self._last_engine.last_loss())

    def synchronize(self):
        for e in self._engines.values():
            e.synchronize()

    # ------------------------------------------------------------------ failure detection
    def guard(self, eng, timeout_s, what="step"):
        """Bounded wait for the work in flight on ``eng``.  On timeout: report what the communicators know,
        abort them (so the peers blocked in the matching operations fail instead of hanging with us) and raise
        ``StepTimeout``.  Device-side spins (fused DP flags) carry their own bound and surface as CUDA errors."""
        if timeout_s is None or eng.wait(float(timeout_s)):
            return
        status = eng.comm_status()
        self.abort_comms()
        raise StepTimeout(f"{what} did not finish within {timeout_s:g} s on stage {self.stage_id} "
                          f"(dp rank {self.dp_comm.Get_rank()}); communicators: {status or 'none'}; plan: {eng.describe()[:200]}")

    def abort_comms(self):
        for nc in (self._pp_nccl, self._dp_nccl):
            if nc is not None:
                nc.abort()

    def sync_to_model(self):
        """Weights live in the model's arena already; just drain the streams."""
        self.synchronize()
        torch.cuda.synchronize(self.device)

    def kernels_per_step(self, sched):
        return int(self.engine_for(sched).kernels_per_step())

    # ------------------------------------------------------------------ optimizer state (checkpoints)
    def optimizer_state(self):
        """Collective over the DP group: the canonical full momentum arena of this stage (CPU, None without momentum),
        each entry taken from the replica that owns it, so the result does not depend on the DP transport.  Entries
        every replica owns come from DP rank 0; the rest of the arena (padding) is zero everywhere."""
        if self.momentum == 0.0:
            return None
        return self._owned_state(self.model.arena.momentum)

    def ema_state(self):
        """Collective over the DP group: the stage's full EMA arena (CPU, None without an EMA), assembled from the
        owners exactly like ``optimizer_state``."""
        if self.ema_decay is None:
            return None
        return self._owned_state(self.model.arena.ema)

    def _owned_state(self, buf):
        """The full arena of a per-element optimizer buffer whose entries live with their owners (see
        ``optimizer_state``)."""
        if buf is None:
            return None
        self.sync_to_model()
        n = self.model.arena.numel
        dp, rank = self.dp_comm.Get_size(), self.dp_comm.Get_rank()
        if dp == 1:
            return buf[:n].detach().cpu().clone()
        eng = self._train_engine
        protos = list(eng.layer_protocols()) if eng is not None else [0] * len(self.model.linears)
        mine = owned_elements(self.model.arena, self.model.linears, protos, dp, rank, shared_to_rank0=True).to(buf.device)
        part = torch.where(mine, buf[:n], torch.zeros_like(buf[:n]))
        import torch.distributed as dist

        dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.dp_comm.group)   # exactly one non-zero term per entry
        return part.cpu()

    def load_optimizer_state(self, full):
        """Restore a buffer returned by ``optimizer_state`` into this replica (every replica loads the full buffer; the
        entries it does not own are never read)."""
        self._load_owned_state(full, self.model.arena.momentum, "momentum")

    def load_ema_state(self, full):
        """Restore a buffer returned by ``ema_state`` into this replica, like ``load_optimizer_state``."""
        self._load_owned_state(full, self.model.arena.ema, "EMA")

    def _load_owned_state(self, full, buf, what):
        if full is None:
            return
        if buf is None or full.numel() != self.model.arena.numel:
            raise ValueError(f"optimizer state does not match this model's {what} arena")
        self.sync_to_model()
        buf[: full.numel()].copy_(full.to(buf.device))
        torch.cuda.synchronize(self.device)

    def describe(self, sched):
        return self.engine_for(sched).describe()


def owned_elements(arena, linears, protocols, dp, rank, shared_to_rank0=False):
    """Bool mask over ``arena`` (CPU): the parameter elements (weights and bias columns) replica ``rank`` of ``dp``
    owns when layer i's update runs under ``protocols[i]`` (``_C.DP_PROTO_*``; the rule is ``dp_element_owner`` in
    ``csrc/kernels/fused_dp.cu``).  Elements every replica owns count for every rank, or only for rank 0 with
    ``shared_to_rank0``.  Padding belongs to rank 0 only with ``shared_to_rank0``."""
    C = _C()
    mask = torch.zeros(arena.numel, dtype=torch.bool)
    if shared_to_rank0 and rank == 0:
        mask[:] = True                                     # padding and alignment gaps: zero on every replica
    for lin, proto in zip(linears, protocols):
        i = lin.block_index
        off, ld = int(arena.offsets[i]), int(arena.lds[i])
        o, k = arena.blocks[i]
        owners = C.dp_owner_map(int(proto), k, o, ld, off, int(dp))            # [out, in + 1], -1 = every replica
        shared = owners < 0
        own = (owners == rank) | (shared if (not shared_to_rank0 or rank == 0) else torch.zeros_like(shared))
        mask[off:off + o * ld].view(o, ld)[:, : k + 1] = own
    return mask


class Trainer:
    """End-to-end training API: the call a user makes.

        trainer = Trainer(layer_sizes, dp=1, pp=1, schedule="naive", ...)
        loss = trainer.step(x_host, y_host)        # pinned host tensors of the DP-local batch

    Every step copies its inputs host->device and reads its loss device->host.

    ``lr`` is the base learning rate.  ``lr_schedule`` (an ``lr_schedule.LRSchedule`` or any callable ``step -> lr``)
    sets ``optimizer.lr`` before every step from the number of steps run so far; ``Trainer.lr`` is the rate of the
    next step.

    ``dropout`` / ``dropout_seed``: inverted dropout on every hidden layer (``models.mlp.MLP``); step i draws the masks
    of ``dropout_step`` i, the number of steps run so far.

    ``activation``: the hidden layers' activation, "relu" (default), "gelu", "silu" or "tanh" (``models.mlp.MLP``).

    ``residual``: an identity skip around every hidden layer whose width does not change (``models.mlp.MLP``).

    ``ema_decay``: keep an exponential moving average of the weights (``optimizer.SGD``), updated inside the update
    kernels; ``ema_state()`` returns it.
    """

    def __init__(self, layer_sizes, global_batch_size=128, n_mubatches=4, lr=0.006, schedule="naive",
                 dp_comm=None, pp_comm=None, grid: Optional[ProcessGrid] = None, comm_mode="fused",
                 use_graph=True, device=None, seed_mode="shape", precision="fp32", watchdog_s=None, pp_transport=None,
                 local_batch_size=None, momentum=0.0, weight_decay=0.0, nesterov=False, loss="mse", lr_schedule=None,
                 dropout=0.0, dropout_seed=0, activation="relu", residual=False, ema_decay=None):
        from ..models.mlp import MLP
        from ..optimizer import SGD
        from .schedules import SCHEDULE_NAME_TO_CLS

        self.dp_comm = dp_comm if dp_comm is not None else SelfComm()
        self.pp_comm = pp_comm if pp_comm is not None else SelfComm()
        dp, pp = self.dp_comm.Get_size(), self.pp_comm.Get_size()
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.global_batch_size, self.n_mubatches = global_batch_size, n_mubatches
        # local_batch_size: rows this replica processes per step.  Defaults to global / dp; an explicit value lets a
        # communication-free engine do one replica's share of a bigger job (bench.py's exposed-comm twin): the loss
        # scale stays 1 / global_batch_size.
        self.local_batch_size = int(local_batch_size) if local_batch_size else global_batch_size // dp
        self.model = MLP(layer_sizes, self.pp_comm.Get_rank(), pp, global_batch_size, seed_mode=seed_mode,
                         loss=loss, dropout=dropout, dropout_seed=dropout_seed, activation=activation,
                         residual=residual).to(self.device)
        self.optimizer = SGD(self.model.parameters(), lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov,
                             arena=self.model.arena, ema_decay=ema_decay)

        class _Shape:  # the worker only needs the micro-batch size from the dataset
            mubatch_size = self.local_batch_size // n_mubatches

        self.worker = NativeWorker(dp_comm, pp_comm, self.model, _Shape(), self.optimizer, grid=grid,
                                   comm_mode=comm_mode, use_graph=use_graph, precision=precision, pp_transport=pp_transport)
        cls = SCHEDULE_NAME_TO_CLS[schedule] if isinstance(schedule, str) else schedule
        self.schedule = cls(n_mubatches, pp, self.pp_comm.Get_rank())
        self.engine = self.worker.engine_for(self.schedule)
        self.is_first, self.is_last = self.schedule.is_first_stage, self.schedule.is_last_stage
        self._steps = 0
        self.lr_schedule = lr_schedule
        self.watchdog_s = watchdog_seconds(watchdog_s)   # None = plain stream synchronisation (default)

    @property
    def lr(self):
        """The learning rate of the next step."""
        return self.lr_schedule(self._steps) if self.lr_schedule is not None else self.optimizer.lr

    def step_async(self, x_host, y_host):
        if self.lr_schedule is not None:
            self.optimizer.lr = self.lr_schedule(self._steps)
        self.model.dropout_step = self._steps
        self.worker.set_lr(self.engine, self.schedule)
        self.engine.stage_inputs(x_host if self.is_first else None, y_host if self.is_last else None)
        self.engine.run()
        self._steps += 1

    def step(self, x_host, y_host):
        """Run one step and return its loss (synchronises with the device)."""
        self.step_async(x_host, y_host)
        if self.watchdog_s is not None:
            self.worker.guard(self.engine, self.watchdog_s, what=f"step {self._steps}")
        return self.engine.last_loss() if self.is_last else None

    def step_pipelined(self, x_host, y_host):
        """Enqueue one step (H2D of its inputs, compute, D2H of its loss) and return the loss of the
        PREVIOUS step, read from pinned host memory after waiting only for that step's event.  The
        device queue never drains: copy-in of step i+1, compute of step i and read-back of step i-1
        overlap.  The first call returns None; ``flush()`` returns the final loss."""
        self.step_async(x_host, y_host)
        if not self.is_last or self._steps < 2:
            return None
        return self.engine.prev_loss()

    def flush(self):
        return self.engine.last_loss() if self.is_last else None

    def loss(self):
        return self.engine.last_loss() if self.is_last else None

    def ema_state(self):
        """Collective over the DP group: this stage's full EMA arena (CPU), or None without an EMA."""
        return self.worker.ema_state()

    def synchronize(self):
        if self.watchdog_s is not None:
            self.worker.guard(self.engine, self.watchdog_s, what="synchronize")
        self.engine.synchronize()
