"""Model layer: Parameter / Module / Linear / ReLU / GELU / SiLU / Tanh / Softmax / MSELoss / CrossEntropyLoss / Sequential.

Capability parity with the reference's ``shallowspeed/layers.py:17-233``: explicit
``forward(inputs, mubatch_id)`` / ``backward(dout, mubatch_id)`` with a per-micro-batch
activation stash (the thing that lets GPipe / 1F1B keep several micro-batches in
flight), gradient *accumulation* into ``param.grad``, and the grad-hook /
post-grad-hook protocol ``Sequential.backward`` drives so that the DP all-reduce of
layer *l* can overlap the backward of layer *l-1* (layers.py:201-213).

The class skeleton is the reference's on purpose: ``Module`` / ``ReLU`` / ``Softmax`` / ``Sequential`` keep its method names,
cache keys (``bitmask_{id}`` / ``input_{id}``) and hook loops, because that API surface IS the parity requirement
(layers.py:31-96, 169-233).  What is new here is everything underneath it:

GPU-first differences (design, not translation):

* storage is ``torch.Tensor``; all parameters of a pipeline stage live in ONE flat
  fp32 arena (``ParamArena``) with a twin arena for gradients.  Each Linear owns an
  ``[out, ld]`` block, ``ld = round_up(in + 1, 8)``: columns ``[0, in)`` are ``W``,
  column ``in`` is the bias.  Row pitch is a multiple of 32 B so a TMA tensor map can
  address the block directly (global strides must be multiples of 16 B - the default
  model's 127/126/125/123-wide layers would otherwise be illegal), and W and b of a
  layer are updated / all-reduced as one tile stream by the fused kernel.
* ``Parameter.data`` / ``.grad`` are *views* into the arenas, so the reference's
  per-parameter API (and the SHA-1 replica check) still works.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Callable, Optional, Sequence

import numpy as np
import torch

from ..ops import functional as F

LD_ALIGN = 8  # floats -> 32-byte row pitch granularity


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def param_ld(in_dims: int) -> int:
    """Row pitch (in floats) of a Linear block: W columns + 1 bias column, padded."""
    return round_up(in_dims + 1, LD_ALIGN)


class ParamArena:
    """One contiguous fp32 buffer for the weights of a stage and one for the grads.

    ``blocks`` is a list of ``(out_dims, in_dims)``.  Block *i* occupies
    ``[offset_i, offset_i + out_i * ld_i)`` in both buffers.  Offsets are aligned to
    128 B so every block base satisfies TMA's 16 B global-address alignment.
    """

    BLOCK_ALIGN = 32  # floats (128 B)

    def __init__(self, blocks: Sequence[tuple], device="cpu"):
        self.blocks = [(int(o), int(i)) for o, i in blocks]
        self.lds = [param_ld(i) for _, i in self.blocks]
        self.offsets = []
        off = 0
        for (o, _), ld in zip(self.blocks, self.lds):
            self.offsets.append(off)
            off = round_up(off + o * ld, self.BLOCK_ALIGN)
        self.numel = max(off, self.BLOCK_ALIGN)
        self.weights = torch.zeros(self.numel, dtype=torch.float32, device=device)
        self.grads = torch.zeros(self.numel, dtype=torch.float32, device=device)
        # SGD momentum buffer, same offsets and row pitches as ``weights``; allocated by ``enable_momentum`` only, so
        # plain SGD costs no memory.  Ordinary device memory even when the weights live in memory shared with peers:
        # only this replica ever reads or writes it.
        self.momentum: Optional[torch.Tensor] = None
        # exponential moving average of the weights, the same layout; allocated by ``enable_ema`` only, and ordinary
        # device memory for the same reason as ``momentum``
        self.ema: Optional[torch.Tensor] = None
        self._listeners: list[Callable[[], None]] = []

    # -- views ---------------------------------------------------------------
    def block(self, i: int, grads: bool = False) -> torch.Tensor:
        """The full ``[out, ld]`` block *i* (weights or grads)."""
        o, _ = self.blocks[i]
        ld = self.lds[i]
        buf = self.grads if grads else self.weights
        return buf[self.offsets[i] : self.offsets[i] + o * ld].view(o, ld)

    def weight_view(self, i, grads=False):
        return self.block(i, grads)[:, : self.blocks[i][1]]

    def bias_view(self, i, grads=False):
        in_dims = self.blocks[i][1]
        return self.block(i, grads)[:, in_dims : in_dims + 1].t()  # [1, out], strides (1, ld)

    def momentum_block(self, i: int) -> torch.Tensor:
        """The ``[out, ld]`` block *i* of the momentum buffer (bias momentum in column ``in``)."""
        o, _ = self.blocks[i]
        return self.momentum[self.offsets[i] : self.offsets[i] + o * self.lds[i]].view(o, self.lds[i])

    # -- storage management ----------------------------------------------------
    def enable_momentum(self):
        """Allocate the (zeroed) momentum buffer on the weights' device; a no-op when it exists."""
        if self.momentum is None:
            self.momentum = torch.zeros(self.numel, dtype=torch.float32, device=self.weights.device)
        return self.momentum

    def ema_block(self, i: int) -> torch.Tensor:
        """The ``[out, ld]`` block *i* of the EMA buffer (bias in column ``in``)."""
        o, _ = self.blocks[i]
        return self.ema[self.offsets[i] : self.offsets[i] + o * self.lds[i]].view(o, self.lds[i])

    def enable_ema(self):
        """Allocate the EMA buffer on the weights' device as a copy of the current weights (padding stays zero); a
        no-op when it exists."""
        if self.ema is None:
            self.ema = torch.zeros(self.numel, dtype=torch.float32, device=self.weights.device)
            for i, (_, k) in enumerate(self.blocks):
                self.ema_block(i)[:, : k + 1].copy_(self.block(i)[:, : k + 1])
        return self.ema

    def on_rebind(self, fn: Callable[[], None]):
        self._listeners.append(fn)

    def rebind(self, weights: torch.Tensor, grads: torch.Tensor, copy: bool = True):
        """Move the arena onto new storage (another device, or a symmetric-memory
        allocation owned by the native runtime).  All Parameter views are refreshed."""
        assert weights.numel() >= self.numel and grads.numel() >= self.numel
        assert weights.dtype == torch.float32 and grads.dtype == torch.float32
        if copy:
            weights[: self.numel].copy_(self.weights)
            grads[: self.numel].copy_(self.grads)
        self.weights, self.grads = weights, grads
        if self.momentum is not None and self.momentum.device != weights.device:
            self.momentum = self.momentum.to(weights.device)
        if self.ema is not None and self.ema.device != weights.device:
            self.ema = self.ema.to(weights.device)
        for fn in self._listeners:
            fn()

    def to(self, device):
        device = torch.device(device)
        if self.weights.device != device:
            self.rebind(
                torch.empty(self.numel, dtype=torch.float32, device=device),
                torch.empty(self.numel, dtype=torch.float32, device=device),
            )
        return self


class Parameter:
    """A tensor plus its gradient accumulator (reference: layers.py:17-28)."""

    def __init__(self, data: torch.Tensor, requires_grad: bool = True, grad: Optional[torch.Tensor] = None):
        self.data = data
        self.grad = grad if grad is not None else torch.zeros_like(data, dtype=torch.float32)
        self.requires_grad = requires_grad
        self._request = None  # in-flight DP all-reduce handle (set by parallel.worker)

    def __repr__(self):
        return f"Parameter(shape={tuple(self.data.shape)}, requires_grad={self.requires_grad})"


class Module(ABC):
    """Stateful op with trainable parameters and a per-micro-batch activation cache
    (reference: layers.py:31-64)."""

    def __init__(self):
        self._params: dict[str, Parameter] = {}
        self._cache: dict[str, torch.Tensor] = {}
        self._training = True

    def __call__(self, inputs, mubatch_id=0):
        return self.forward(inputs, mubatch_id=mubatch_id)

    @abstractmethod
    def forward(self, inputs: torch.Tensor, mubatch_id=0):
        raise NotImplementedError

    @abstractmethod
    def backward(self, dout: torch.Tensor, mubatch_id=0):
        raise NotImplementedError

    def train(self):
        self._training = True

    def eval(self):
        self._training = False

    def zero_grad(self):
        for param in self.parameters():
            param.grad.zero_()

    def parameters(self):
        return list(self._params.values())


class ReLU(Module):
    """Caches the sign mask per micro-batch.  On CUDA the fused Linear kernel hands us
    the *output* y = relu(z); ``y > 0`` is the same mask, so no extra tensor is
    materialised (SURVEY.md K1).

    Under dropout the owning Linear stashes its dropped output a = relu(z) * keep * s instead, so ``a > 0`` is "active
    and kept", and ``dropout_scale`` (s) multiplies the gradient where the mask passes it."""

    dropout_scale = None
    kind = "relu"

    def forward(self, inputs, mubatch_id=0):
        if self._training:
            self._cache[f"bitmask_{mubatch_id}"] = inputs > 0
        return F.relu(inputs)

    def stash_output(self, outputs, mubatch_id=0):
        if self._training:
            self._cache[f"bitmask_{mubatch_id}"] = outputs

    def backward(self, dout, mubatch_id=0):
        assert self._training
        dout = F.relu_grad(dout, self._cache.pop(f"bitmask_{mubatch_id}"))
        if self.dropout_scale is not None:
            dout = dout * self.dropout_scale
        return dout

    def __repr__(self):
        return "ReLU()"


class _Gated(Module):
    """A smooth activation f: ``forward`` returns f(z) and caches the gate gamma = f'(z) per micro-batch; ``backward``
    is dout * gamma.  Under dropout the owning Linear stashes gamma * keep * s instead (``stash_gate``), so the
    backward needs no mask of its own (ops.functional.activation_ref is the math)."""

    kind = None

    def forward(self, inputs, mubatch_id=0):
        a, gamma = F.activation(self.kind, inputs)
        self.stash_gate(gamma, mubatch_id)
        return a

    def stash_gate(self, gamma, mubatch_id=0):
        if self._training:
            self._cache[f"gate_{mubatch_id}"] = gamma

    def backward(self, dout, mubatch_id=0):
        assert self._training
        return F.gate_grad(dout, self._cache.pop(f"gate_{mubatch_id}"))

    def __repr__(self):
        return f"{type(self).__name__}()"


class GELU(_Gated):
    """0.5 z (1 + erf(z / sqrt(2))): torch's ``nn.GELU()`` (the erf form)."""

    kind = "gelu"


class SiLU(_Gated):
    """z sigmoid(z): torch's ``nn.SiLU()``."""

    kind = "silu"


class Tanh(_Gated):
    kind = "tanh"


ACTIVATIONS = {"relu": ReLU, "gelu": GELU, "silu": SiLU, "tanh": Tanh}


class Softmax(Module):
    def forward(self, inputs, mubatch_id=0):
        if self._training:
            self._cache[f"input_{mubatch_id}"] = inputs
        return F.softmax(inputs)

    def backward(self, dout, mubatch_id=0):
        assert self._training
        return F.softmax_grad(dout, self._cache.pop(f"input_{mubatch_id}"))

    def __repr__(self):
        return "Softmax()"


def _init_seed(in_dims: int, out_dims: int, layer_index: Optional[int]):
    # The reference seeds by *shape* only (layers.py:104-106) so that any DP x PP
    # layout builds identical weights without a broadcast.  ``layer_index`` adds the
    # global layer index to the seed (still layout independent) so that equal-shaped
    # layers (hidden=8192 x 16) do not start identical.
    if layer_index is None:
        return in_dims + out_dims * 1337
    return [in_dims + out_dims * 1337, int(layer_index) + 1]


class Linear(Module):
    """y = f?(x @ W^T + b) with hand-written backward (reference: layers.py:99-142); f is ReLU, GELU, SiLU or tanh
    (``activation``: "relu", "gelu", "silu", "tanh" or None).

    ``residual=True`` adds an identity skip around the layer: a = x + drop(f(x W^T + b)).  It needs an activation and
    ``in_dims == out_dims``.  The branch always goes through the gated route (F.activation, ReLU included), since the
    output x + relu(z) is no longer its own mask; the backward is linear_grad(g * gamma) + g."""

    def __init__(self, in_dims, out_dims, activation="relu", arena: Optional[ParamArena] = None,
                 block_index: int = 0, layer_index: Optional[int] = None, device="cpu", residual: bool = False):
        super().__init__()
        if activation is not None:
            F.check_activation(activation)
        if not isinstance(residual, bool):
            raise ValueError(f"residual must be a bool, got {residual!r}")
        if residual and (activation is None or in_dims != out_dims):
            raise ValueError(f"a residual Linear needs an activation and in_dims == out_dims, got {in_dims}->{out_dims}, "
                             f"activation {activation!r}")
        self.residual = residual
        self.in_dims, self.out_dims = in_dims, out_dims
        self.activation = ACTIVATIONS[activation]() if activation is not None else None
        if arena is None:
            arena = ParamArena([(out_dims, in_dims)], device=device)
            block_index = 0
        self.arena, self.block_index = arena, block_index

        from numpy.random import MT19937, RandomState, SeedSequence

        rs = RandomState(MT19937(SeedSequence(_init_seed(in_dims, out_dims, layer_index))))
        w = rs.normal(0.0, 1.0, (out_dims, in_dims)).astype(np.float32) / np.float32(np.sqrt(in_dims))
        arena.weight_view(block_index).copy_(torch.from_numpy(w.astype(np.float32)))
        arena.bias_view(block_index).zero_()
        self._bind()
        arena.on_rebind(self._bind)

    def _bind(self):
        a, i = self.arena, self.block_index
        if "W" in self._params:
            self._params["W"].data, self._params["W"].grad = a.weight_view(i), a.weight_view(i, True)
            self._params["b"].data, self._params["b"].grad = a.bias_view(i), a.bias_view(i, True)
        else:
            self._params["W"] = Parameter(a.weight_view(i), grad=a.weight_view(i, True))
            self._params["b"] = Parameter(a.bias_view(i), grad=a.bias_view(i, True))

    def forward(self, inputs, mubatch_id=0):
        if self._training:
            self._cache[f"input_{mubatch_id}"] = inputs
        W, b = self._params["W"].data, self._params["b"].data
        if self.residual:
            # x + drop(f(z)); the gate (with dropout's keep * s) is the whole backward of the branch
            a, gamma = F.activation(self.activation.kind, F.linear(inputs, W, b))
            if self._training and self.dropout is not None:
                a, gamma = self._dropout(a), self._dropout(gamma)
            if self._training:
                self._cache[f"gate_{mubatch_id}"] = gamma
            return inputs + a
        if isinstance(self.activation, _Gated):
            # z, then (f(z), f'(z)) in one pass; dropout drops both, so the stashed gate is the whole backward
            a, gamma = F.activation(self.activation.kind, F.linear(inputs, W, b))
            if self._training and self.dropout is not None:
                a, gamma = self._dropout(a), self._dropout(gamma)
            self.activation.stash_gate(gamma, mubatch_id)
            return a
        if inputs.is_cuda:
            from ..ops import cuda as K

            out = K.linear_fwd(inputs, W, b, relu=self.activation is not None)
            if self.activation is not None:
                out = self._dropout(out)
                self.activation.stash_output(out, mubatch_id)
            return out
        result = F.linear(inputs, W, b)
        if self.activation:
            out = self.activation(result, mubatch_id)
            if self._training and self.dropout is not None:
                out = self._dropout(out)
                self.activation.stash_output(out > 0, mubatch_id)
            return out
        return result

    # dropout of this Linear's ReLU output (set by models.mlp.MLP): None, or (p, seed, global layer index, scale); the
    # samples and step of the next forward are in dropout_rows = (global sample index of every input row, step)
    dropout = None
    dropout_rows = None

    def _dropout(self, out):
        if not self._training or self.dropout is None:
            return out
        p, seed, layer, scale = self.dropout
        samples, step = self.dropout_rows
        keep = F.dropout_mask(p, seed, layer, step, samples.to(out.device), out.shape[1])
        return F.dropout_ref(out, keep, scale)

    def backward(self, dout, mubatch_id=0):
        assert self._training
        skip = None
        if self.residual:
            skip = dout                                     # the skip's gradient passes through unchanged
            dout = F.gate_grad(dout, self._cache.pop(f"gate_{mubatch_id}"))
        elif self.activation:
            dout = self.activation.backward(dout, mubatch_id)
        x = self._cache.pop(f"input_{mubatch_id}")
        if dout.is_cuda:
            from ..ops import cuda as K

            # dW / db accumulate in place inside the wgrad kernel's epilogue
            dx = K.linear_bwd_accumulate(dout, x, self.arena.block(self.block_index),
                                         self.arena.block(self.block_index, True), self.in_dims)
            return dx if skip is None else dx + skip
        dx, dW, db = F.linear_grad(dout, x, self._params["W"].data)
        self._params["W"].grad += dW
        self._params["b"].grad += db.reshape(1, -1)
        return dx if skip is None else dx + skip

    def __repr__(self):
        return f"Linear({self.in_dims}->{self.out_dims}, act: {self.activation}{', residual' if self.residual else ''})"


class MSELoss(Module):
    """Identity in forward; ``backward(target)`` returns -2 (t - x) / global_batch
    (reference: layers.py:145-166).  ``last_loss`` additionally records the loss value
    of the most recent micro-batch (the reference never computes it)."""

    def __init__(self, batch_size: int):
        super().__init__()
        self.batch_size = batch_size
        self.last_loss = None

    def forward(self, input, mubatch_id=0):
        if self._training:
            self._cache[f"input_{mubatch_id}"] = input
        return input

    def backward(self, target, mubatch_id=0):
        assert self._training
        x = self._cache.pop(f"input_{mubatch_id}")
        self.last_loss = F.mse_loss(x, target, self.batch_size)
        return F.mse_loss_grad(x, target, self.batch_size)

    def __repr__(self):
        return "MSELoss()"


class CrossEntropyLoss(Module):
    """Softmax cross-entropy on logits: torch's ``F.cross_entropy(z, t, reduction="sum") / batch_size`` with
    probability targets.  ``forward`` caches the logits and returns the per-row softmax, so the last stage's output is
    still the class probabilities (argmax / accuracy are unchanged).  ``backward(target)`` records ``last_loss`` of the
    micro-batch and returns dL/dz = (p * sum(t) - t) / batch_size, fused (ops.functional.loss_head_backward)."""

    def __init__(self, batch_size: int):
        super().__init__()
        self.batch_size = batch_size
        self.last_loss = None

    def forward(self, input, mubatch_id=0):
        if self._training:
            self._cache[f"input_{mubatch_id}"] = input
        return F.row_softmax(input)

    def backward(self, target, mubatch_id=0):
        assert self._training
        z = self._cache.pop(f"input_{mubatch_id}")
        dz, _, self.last_loss = F.loss_head_backward(z, target, self.batch_size, loss="cross_entropy")
        return dz

    def __repr__(self):
        return "CrossEntropyLoss()"


class Sequential(Module):
    """Layer list with the backward-hook protocol (reference: layers.py:169-233)."""

    def __init__(self, layers: list):
        super().__init__()
        self.layers = layers
        self._grad_hooks = []
        self._post_grad_hooks = []

    def forward(self, inputs, mubatch_id=0):
        result = inputs
        for layer in self.layers:
            result = layer(result, mubatch_id)
        return result

    def register_grad_hook(self, hook):
        """hook(param) runs as soon as the gradient of ``param`` is final."""
        assert hook not in self._grad_hooks
        self._grad_hooks.append(hook)

    def reset_grad_hooks(self):
        self._grad_hooks = []

    def register_post_grad_hook(self, hook):
        """hook(all_params) runs right before ``backward`` returns."""
        self._post_grad_hooks.append(hook)

    def reset_post_grad_hooks(self):
        self._post_grad_hooks = []

    def backward(self, dout, mubatch_id=0):
        result = dout
        for layer in reversed(self.layers):
            result = layer.backward(result, mubatch_id)
            for hook in self._grad_hooks:
                for param in layer.parameters():
                    hook(param)
        for hook in self._post_grad_hooks:
            hook(self.parameters())
        return result

    def train(self):
        self._training = True
        for l in self.layers:
            l.train()

    def eval(self):
        self._training = False
        for l in self.layers:
            l.eval()

    def zero_grad(self):
        for l in self.layers:
            l.zero_grad()

    def parameters(self):
        result = []
        for l in self.layers:
            result += l.parameters()
        return result
