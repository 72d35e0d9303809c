"""Python pipeline VM: executes a Schedule's instruction stream for one stage.

Parity with the reference's ``Worker`` (``shallowspeed/pipe.py:330-466``) and the two DP
hook functions (pipe.py:302-327): same constructor ``Worker(dp_comm, pp_comm, model,
dataset, optimizer)``, same ``execute(sched, batch_id)``, one method per instruction,
``input_buffers`` / ``output_buffers`` readable after ``execute`` (train.py reads
``output_buffers[0]`` to compute accuracy).

This VM is the portable path (CPU/gloo, debugging, numerics oracle).  On a GPU the same
instruction stream is lowered once into a static plan and run by the native executor
(``parallel.engine`` -> ``csrc/runtime``) on CUDA streams + NCCL p2p + the fused
in-kernel DP reduction.

Differences to the reference VM, all deliberate:
* buffers are persistent per (slot, direction) instead of re-allocated every batch
  (the reference's own TODO, pipe.py:443-445), and activations / gradients use
  separate buffers so a send of slot i may overlap a receive into slot i;
* consecutive communication instructions are issued as ONE batched group
  (deadlock-free under rendezvous semantics, see ``parallel.validate``);
* the reference's stage>0 GPipe path receives in place into the array its first Linear
  cached by reference (pipe.py:371-373 + layers.py:116-117), silently corrupting the
  stashed input of earlier micro-batches; here every in-flight micro-batch owns a slot.

The instruction -> handler table and the handler names mirror the reference's ``Worker`` (pipe.py:389-432) by design:
it is the portable, debuggable VM with the reference's surface.  Slots, grouped communication, per-layer bucketing and
everything performance-relevant live in the native executor (``parallel/engine.py`` + ``csrc/runtime``).
"""
from __future__ import annotations

import dataclasses

import torch

from .comm import Comm, SelfComm
from .instructions import (BackwardGradAcc, BackwardGradAllReduce, COMM_INSTRUCTIONS, Forward,
                           LoadInstruction, LoadMuBatchInput, LoadMuBatchTarget, OptimizerStep,
                           RecvActivations, RecvOutputGrad, SendActivations, SendInputGrad, ZeroGrad)


# ----------------------------------------------------------------------------
# DP hooks (same names as the reference)
# ----------------------------------------------------------------------------
def backprop_allreduce_gradient(comm: Comm, param):
    """Start a non-blocking SUM all-reduce for a parameter whose gradient just became
    final.  Parameters that live in a ``ParamArena`` block are reduced as ONE contiguous
    message per layer ([out, ld] = W, b and padding) when the block's leader ("W") fires
    - the bucketing the reference's docstring wishes for (pipe.py:309-311)."""
    if not param.requires_grad:
        return
    block = getattr(param, "_block_grad", None)
    if block is not None:
        if getattr(param, "_block_leader", False):
            param._request = comm.iallreduce(block)
        return
    param._request = comm.iallreduce(param.grad)


def backprop_block_for_comms(params):
    """Wait for every outstanding gradient all-reduce (MPI Waitall analogue)."""
    for param in params:
        if param.requires_grad and getattr(param, "_request", None) is not None:
            param._request.wait()
            param._request = None


def tag_arena_blocks(model):
    """Mark W as block leader so the hooks reduce whole arena blocks."""
    for lin in getattr(model, "linears", []):
        blk = lin.arena.block(lin.block_index, grads=True)
        w, b = lin._params["W"], lin._params["b"]
        w._block_grad, w._block_leader = blk, True
        b._block_grad, b._block_leader = blk, False


class Worker:
    """Executes all ticks of a schedule for one batch on one (dp_rank, pp_stage) cell."""

    def __init__(self, dp_comm, pp_comm, model, dataset, optimizer, device=None):
        self.dp_comm = dp_comm if dp_comm is not None else SelfComm()
        self.pp_comm = pp_comm if pp_comm is not None else SelfComm()
        self.stage_id = self.pp_comm.Get_rank()
        self.pipeline_depth = self.pp_comm.Get_size()
        self.model = model
        self.dataset = dataset
        self.optimizer = optimizer
        self.device = torch.device(device) if device is not None else model.arena.weights.device
        self.input_buffers: list = []
        self.output_buffers: list = []
        self.input_grad_buffers: list = []
        self.output_grad_buffers: list = []
        self._buf_key = None
        self.last_losses: list = []
        tag_arena_blocks(model)
        if dp_comm is not None and self.dp_comm.size > 1:
            # arena rebinding (e.g. .to(device)) must refresh the block tags
            model.arena.on_rebind(lambda: tag_arena_blocks(model))

    # -- buffers -------------------------------------------------------------
    def _ensure_buffers(self, n_slots: int):
        mb = self.dataset.mubatch_size
        key = (n_slots, mb, self.model.in_dim, self.model.out_dim)
        if self._buf_key == key:
            return
        mk = lambda d: [torch.empty(mb, d, dtype=torch.float32, device=self.device) for _ in range(n_slots)]
        self.input_buffers, self.output_buffers = mk(self.model.in_dim), mk(self.model.out_dim)
        self.input_grad_buffers, self.output_grad_buffers = mk(self.model.in_dim), mk(self.model.out_dim)
        self._buf_key = key

    # -- instruction handlers ----------------------------------------------------
    def load_micro_batch_input(self, batch_id, mubatch_id, buffer_id):
        data = self.dataset.load_micro_batch_input(batch_id, mubatch_id)
        assert data.shape == self.input_buffers[buffer_id].shape, (
            f"shape is {tuple(data.shape)} but should be {tuple(self.input_buffers[buffer_id].shape)}")
        self.input_buffers[buffer_id] = data.to(self.device, non_blocking=True)

    def load_micro_batch_target(self, batch_id, mubatch_id, buffer_id):
        data = self.dataset.load_micro_batch_target(batch_id, mubatch_id)
        assert data.shape == self.output_grad_buffers[buffer_id].shape
        self.output_grad_buffers[buffer_id] = data.to(self.device, non_blocking=True)

    def _comm_op(self, ins):
        b = ins.buffer_id
        if isinstance(ins, SendActivations):
            return ("send", self.output_buffers[b], self.get_successor())
        if isinstance(ins, RecvActivations):
            # fresh tensor: the previous occupant may still be referenced by a stash
            self.input_buffers[b] = torch.empty_like(self.input_buffers[b])
            return ("recv", self.input_buffers[b], self.get_predecessor())
        if isinstance(ins, SendInputGrad):
            return ("send", self.input_grad_buffers[b], self.get_predecessor())
        if isinstance(ins, RecvOutputGrad):
            self.output_grad_buffers[b] = torch.empty_like(self.output_grad_buffers[b])
            return ("recv", self.output_grad_buffers[b], self.get_successor())
        raise TypeError(ins)

    def send_activations(self, buffer_id):
        self.pp_comm.batch([self._comm_op(SendActivations(buffer_id))])

    def recv_activations(self, buffer_id):
        self.pp_comm.batch([self._comm_op(RecvActivations(buffer_id))])

    def send_grad(self, buffer_id):
        self.pp_comm.batch([self._comm_op(SendInputGrad(buffer_id))])

    def recv_grad(self, buffer_id):
        self.pp_comm.batch([self._comm_op(RecvOutputGrad(buffer_id))])

    def forward(self, buffer_id, mubatch_id):
        if hasattr(self.model, "dropout_shard"):   # dropout masks are drawn per global sample: rank-strided shards
            self.model.dropout_shard = (self.dp_comm.Get_rank(), self.dp_comm.Get_size())
        out = self.model.forward(self.input_buffers[buffer_id], mubatch_id=mubatch_id)
        self.output_buffers[buffer_id] = out if out.is_contiguous() else out.contiguous()

    def backward_accumulate(self, buffer_id, mubatch_id):
        dx = self.model.backward(self.output_grad_buffers[buffer_id], mubatch_id=mubatch_id)
        self.input_grad_buffers[buffer_id] = dx if dx.is_contiguous() else dx.contiguous()
        loss_layer = getattr(self.model, "loss_layer", None)
        if loss_layer is not None and loss_layer.last_loss is not None:
            self.last_losses.append(loss_layer.last_loss)

    def backward_and_reduce(self, buffer_id, mubatch_id):
        self.model.register_grad_hook(lambda param: backprop_allreduce_gradient(self.dp_comm, param))
        self.model.register_post_grad_hook(backprop_block_for_comms)
        self.backward_accumulate(buffer_id, mubatch_id=mubatch_id)
        self.model.reset_grad_hooks()
        self.model.reset_post_grad_hooks()

    def optimizer_step(self):
        self.optimizer.step()

    def zero_grad(self):
        self.model.zero_grad()
        self.last_losses = []

    def get_predecessor(self):
        return self.stage_id - 1

    def get_successor(self):
        return self.stage_id + 1

    _INSTRUCTION_MAP = {
        LoadMuBatchInput: load_micro_batch_input,
        LoadMuBatchTarget: load_micro_batch_target,
        Forward: forward,
        BackwardGradAllReduce: backward_and_reduce,
        BackwardGradAcc: backward_accumulate,
        OptimizerStep: optimizer_step,
        ZeroGrad: zero_grad,
        RecvActivations: recv_activations,
        SendActivations: send_activations,
        RecvOutputGrad: recv_grad,
        SendInputGrad: send_grad,
    }

    def execute(self, sched, batch_id):
        """Run one batch.  Consecutive comm instructions are coalesced into one group."""
        assert sched.num_buffers % 2 == 0
        self._ensure_buffers(sched.num_buffers // 2)
        pending = []
        for commands in sched.steps():
            for command in commands:
                if isinstance(command, COMM_INSTRUCTIONS):
                    pending.append(self._comm_op(command))
                    continue
                if pending:
                    self.pp_comm.batch(pending)
                    pending = []
                fn = self._INSTRUCTION_MAP[type(command)]
                if isinstance(command, LoadInstruction):
                    fn(self, batch_id, **dataclasses.asdict(command))
                else:
                    fn(self, **dataclasses.asdict(command))
        if pending:
            self.pp_comm.batch(pending)

    def batch_loss(self):
        """Sum of the micro-batch losses of the last executed batch (last stage only)."""
        if not self.last_losses:
            return None
        return float(sum(float(l) for l in self.last_losses))
