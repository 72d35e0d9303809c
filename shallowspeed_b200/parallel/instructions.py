"""Pipeline instruction IR (pure data).

Same instruction vocabulary as the reference (``shallowspeed/pipe.py:12-138``), so a
ShallowSpeed user finds every instruction type under the same name.  The IR stays pure
data - no tensors, no communicators - which keeps schedules unit-testable on a laptop
and lets the native runtime (``csrc/runtime/pipe_executor.cpp``) lower a whole step to a
static stream/event plan ONCE instead of re-interpreting Python objects per batch.

Difference to the reference: ``buffer_id`` is a real *slot* id.  The reference always
passes 0 and keeps in-flight micro-batch state inside the modules; here a slot owns the
stage-boundary buffers (activation in/out, gradient in/out) and the activation stash of
one in-flight micro-batch, so sends/receives can run asynchronously on side streams.
"""
from __future__ import annotations

from dataclasses import dataclass


class PipeInstr:
    """Base of the instruction IR."""

    opcode = -1  # stable integer id used by the native plan


@dataclass(frozen=True)
class ZeroGrad(PipeInstr):
    """Open a gradient-accumulation phase (param.grad := 0)."""

    opcode = 0


@dataclass(frozen=True)
class OptimizerStep(PipeInstr):
    """Apply param.grad to the trainable parameters."""

    opcode = 1


@dataclass(frozen=True)
class BufferPipeInstr(PipeInstr):
    buffer_id: int


@dataclass(frozen=True)
class RecvActivations(BufferPipeInstr):
    """Receive the activations of a micro-batch from the previous stage into slot."""

    opcode = 2


@dataclass(frozen=True)
class SendActivations(BufferPipeInstr):
    """Send the local forward result of slot to the next stage."""

    opcode = 3


@dataclass(frozen=True)
class RecvOutputGrad(BufferPipeInstr):
    """Receive d(loss)/d(stage output) of slot from the next stage."""

    opcode = 4


@dataclass(frozen=True)
class SendInputGrad(BufferPipeInstr):
    """Send d(loss)/d(stage input) of slot to the previous stage."""

    opcode = 5


@dataclass(frozen=True)
class MuBatchPipeInstr(PipeInstr):
    buffer_id: int
    mubatch_id: int


@dataclass(frozen=True)
class Forward(MuBatchPipeInstr):
    """Local forward of micro-batch ``mubatch_id`` living in slot ``buffer_id``."""

    opcode = 6


@dataclass(frozen=True)
class BackwardGradAcc(MuBatchPipeInstr):
    """Local backward; param.grad += grad of this micro-batch."""

    opcode = 7


@dataclass(frozen=True)
class BackwardGradAllReduce(MuBatchPipeInstr):
    """Local backward of the LAST-processed micro-batch: every layer's gradient becomes
    final here, so the DP reduction of layer l is started as soon as it is computed and
    overlaps the backward of layer l-1 (on the GPU: fused into the wgrad kernel)."""

    opcode = 8


@dataclass(frozen=True)
class LoadInstruction(MuBatchPipeInstr):
    pass


@dataclass(frozen=True)
class LoadMuBatchInput(LoadInstruction):
    """Load the inputs X of a micro-batch into slot (first stage only)."""

    opcode = 9


@dataclass(frozen=True)
class LoadMuBatchTarget(LoadInstruction):
    """Load the targets y of a micro-batch into slot (last stage only)."""

    opcode = 10


ALL_INSTRUCTIONS = [
    ZeroGrad, OptimizerStep, RecvActivations, SendActivations, RecvOutputGrad, SendInputGrad,
    Forward, BackwardGradAcc, BackwardGradAllReduce, LoadMuBatchInput, LoadMuBatchTarget,
]
OPCODE_TO_CLS = {c.opcode: c for c in ALL_INSTRUCTIONS}
COMM_INSTRUCTIONS = (RecvActivations, SendActivations, RecvOutputGrad, SendInputGrad)
SEND_INSTRUCTIONS = (SendActivations, SendInputGrad)
RECV_INSTRUCTIONS = (RecvActivations, RecvOutputGrad)
BACKWARD_INSTRUCTIONS = (BackwardGradAcc, BackwardGradAllReduce)


def encode(instr: PipeInstr):
    """(opcode, buffer_id, mubatch_id) triple for the native plan (-1 = unused field)."""
    return (instr.opcode, getattr(instr, "buffer_id", -1), getattr(instr, "mubatch_id", -1))


def flatten(steps):
    return [cmd for tick in steps for cmd in tick]
