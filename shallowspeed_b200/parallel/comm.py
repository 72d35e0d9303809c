"""Communication plumbing: process grid + communicators.

The reference uses mpi4py communicators obtained by ``COMM_WORLD.Split`` (train.py:89-92)
and touches this surface: ``Get_rank/Get_size/rank``, ``Iallreduce`` + ``Waitall``,
blocking ``Send/Recv`` and a pickle ``gather`` (SURVEY.md section 2.4, C1-C11).

Here the plumbing is ``torch.distributed`` (one process per GPU, backend ``nccl``; ``gloo``
for the CPU path / tests) wrapped in a tiny communicator interface so that the pipeline
VM is backend agnostic.  Three implementations:

* ``SelfComm``    - size-1 communicator (sequential training, no-ops).
* ``TorchComm``   - a ``torch.distributed`` process group (NCCL over NVLink/NVSwitch on
                    GPUs, gloo on CPU).
* ``ThreadComm``  - in-process fabric for fast multi-"rank" tests (threads + queues).

The *hot* DP path on GPUs does not go through this file at all: the native engine
reduces gradients inside the wgrad kernel over peer memory (``csrc/kernels``).
"""
from __future__ import annotations

import queue
import threading
from dataclasses import dataclass
from typing import Any, List, Optional, Sequence

import torch


# ----------------------------------------------------------------------------
# process grid
# ----------------------------------------------------------------------------
@dataclass(frozen=True)
class ProcessGrid:
    """DP x PP layout with the reference's rank mapping (train.py:89-92):
    ``stage = rank % pp`` (pipeline neighbours are *adjacent* world ranks, i.e. adjacent
    GPUs) and ``replica = rank // pp``."""

    dp: int
    pp: int
    rank: int

    def __post_init__(self):
        assert self.dp >= 1 and self.pp >= 1
        assert 0 <= self.rank < self.dp * self.pp

    @property
    def world_size(self):
        return self.dp * self.pp

    @property
    def stage(self):
        return self.rank % self.pp

    @property
    def replica(self):
        return self.rank // self.pp

    def dp_group_ranks(self, stage: Optional[int] = None) -> List[int]:
        """world ranks that hold the same stage (all-reduce peers)."""
        stage = self.stage if stage is None else stage
        return [r * self.pp + stage for r in range(self.dp)]

    def pp_group_ranks(self, replica: Optional[int] = None) -> List[int]:
        """world ranks that form one pipeline (send/recv peers), in stage order."""
        replica = self.replica if replica is None else replica
        return [replica * self.pp + s for s in range(self.pp)]


# ----------------------------------------------------------------------------
# communicator interface
# ----------------------------------------------------------------------------
class Request:
    def wait(self):
        pass


class Comm:
    rank: int = 0
    size: int = 1

    def Get_rank(self):
        return self.rank

    def Get_size(self):
        return self.size

    # collectives
    def iallreduce(self, tensor: torch.Tensor) -> Request:
        """in-place SUM all-reduce, non-blocking (MPI Iallreduce analogue)."""
        raise NotImplementedError

    def allreduce(self, tensor):
        self.iallreduce(tensor).wait()

    def gather(self, obj: Any, root: int = 0) -> Optional[list]:
        raise NotImplementedError

    def barrier(self):
        pass

    # point to point (peer = rank inside this communicator)
    def send(self, tensor, dst: int):
        self.batch([("send", tensor, dst)])

    def recv(self, tensor, src: int):
        self.batch([("recv", tensor, src)])

    def batch(self, ops: Sequence[tuple]):
        """ops = [("send"|"recv", tensor, peer)].  All operations progress concurrently
        (ncclGroup semantics); returns when every one has completed."""
        raise NotImplementedError


class SelfComm(Comm):
    """Size-1 communicator."""

    def iallreduce(self, tensor):
        return Request()

    def gather(self, obj, root=0):
        return [obj]

    def batch(self, ops):
        if ops:
            raise RuntimeError("point-to-point on a size-1 communicator")


# ----------------------------------------------------------------------------
# torch.distributed
# ----------------------------------------------------------------------------
class _WorkRequest(Request):
    def __init__(self, work):
        self.work = work

    def wait(self):
        if self.work is not None:
            self.work.wait()
            self.work = None


class TorchComm(Comm):
    def __init__(self, ranks: Sequence[int], group=None):
        import torch.distributed as dist

        self.dist = dist
        self.ranks = list(ranks)
        self.group = group
        self.size = len(self.ranks)
        self.rank = self.ranks.index(dist.get_rank())

    def iallreduce(self, tensor):
        if self.size == 1:
            return Request()
        assert tensor.is_contiguous(), "all-reduce needs a contiguous buffer (use the arena block)"
        return _WorkRequest(self.dist.all_reduce(tensor, op=self.dist.ReduceOp.SUM, group=self.group, async_op=True))

    def gather(self, obj, root=0):
        out = [None] * self.size
        self.dist.all_gather_object(out, obj, group=self.group)
        return out if self.rank == root else None

    def barrier(self):
        if self.size > 1:
            self.dist.barrier(group=self.group)

    def batch(self, ops):
        if not ops:
            return
        p2p = []
        for kind, tensor, peer in ops:
            assert tensor.is_contiguous()
            fn = self.dist.isend if kind == "send" else self.dist.irecv
            p2p.append(self.dist.P2POp(fn, tensor, self.ranks[peer], self.group))
        for w in self.dist.batch_isend_irecv(p2p):
            w.wait()


def make_torch_comms(grid: ProcessGrid):
    """Create the DP and PP communicators of this rank.  Every rank must create ALL
    groups (torch.distributed.new_group is collective over the world)."""
    import torch.distributed as dist

    assert dist.is_initialized() and dist.get_world_size() == grid.world_size
    dp_comm = pp_comm = None
    for stage in range(grid.pp):
        ranks = grid.dp_group_ranks(stage)
        g = dist.new_group(ranks) if grid.dp > 1 else None
        if stage == grid.stage:
            dp_comm = TorchComm(ranks, g) if grid.dp > 1 else SelfComm()
    for rep in range(grid.dp):
        ranks = grid.pp_group_ranks(rep)
        g = dist.new_group(ranks) if grid.pp > 1 else None
        if rep == grid.replica:
            pp_comm = TorchComm(ranks, g) if grid.pp > 1 else SelfComm()
    if isinstance(dp_comm, SelfComm):
        dp_comm.rank, dp_comm.size = 0, 1
    if isinstance(pp_comm, SelfComm):
        pp_comm.rank, pp_comm.size = 0, 1
    return dp_comm, pp_comm


# ----------------------------------------------------------------------------
# in-process fabric (tests, debugging)
# ----------------------------------------------------------------------------
class ThreadFabric:
    """Shared state of a group of ``ThreadComm``s living in one process."""

    def __init__(self, size: int):
        self.size = size
        self.queues = {(a, b): queue.Queue() for a in range(size) for b in range(size) if a != b}
        self.barrier = threading.Barrier(size)
        self.lock = threading.Lock()
        self.slots: dict = {}
        self.timeout = 60.0

    def comm(self, rank: int) -> "ThreadComm":
        return ThreadComm(self, rank)


class ThreadComm(Comm):
    def __init__(self, fabric: ThreadFabric, rank: int):
        self.fabric, self.rank, self.size = fabric, rank, fabric.size
        self._seq = 0

    def _exchange(self, value):
        """all ranks contribute a value; everyone gets the rank-ordered list."""
        f = self.fabric
        key = ("x", self._seq)
        self._seq += 1
        with f.lock:
            f.slots.setdefault(key, {})[self.rank] = value
        f.barrier.wait(f.timeout)
        vals = [f.slots[key][r] for r in range(self.size)]
        f.barrier.wait(f.timeout)
        if self.rank == 0:
            with f.lock:
                del f.slots[key]
        return vals

    def iallreduce(self, tensor):
        if self.size > 1:
            vals = self._exchange(tensor.detach().clone())
            total = vals[0].clone()
            for v in vals[1:]:
                total += v          # fixed rank order -> bit-identical on every rank
            tensor.copy_(total)
        return Request()

    def gather(self, obj, root=0):
        vals = self._exchange(obj)
        return vals if self.rank == root else None

    def barrier(self):
        self.fabric.barrier.wait(self.fabric.timeout)

    def batch(self, ops):
        f = self.fabric
        for kind, tensor, peer in ops:       # post all sends first (eager buffered)
            if kind == "send":
                f.queues[(self.rank, peer)].put(tensor.detach().clone())
        for kind, tensor, peer in ops:
            if kind == "recv":
                tensor.copy_(f.queues[(peer, self.rank)].get(timeout=f.timeout))
