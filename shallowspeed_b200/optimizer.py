"""Optimizer.  Parity: ``SGD(parameters, lr).step()`` = ``param.data -= lr * param.grad``
for trainable params (reference ``shallowspeed/optimizer.py:4-13``); stateless.

Beyond the reference, ``momentum``, ``weight_decay`` and ``nesterov`` follow ``torch.optim.SGD`` with
``dampening=0`` and one parameter group (biases are decayed too)::

    g' = g + weight_decay * w
    v  = momentum * v + g'            (v starts at 0)
    d  = g' + momentum * v if nesterov else v
    w -= lr * d

The defaults are the reference's stateless rule, bit for bit.

GPU: when all parameters are views into one ``ParamArena`` the update is a single fused
pass over the flat buffers (one multi-tensor kernel on CUDA, ``csrc/kernels/elementwise.cu``)
instead of one axpy per parameter; the momentum buffer is then the arena's flat ``momentum``
buffer.  On the native engine's fused path the update happens inside the wgrad (+all-reduce)
kernel and ``step`` is not called at all.
"""
from __future__ import annotations

import torch


def check_hparams(lr, momentum, weight_decay, nesterov):
    """Raise ``ValueError`` for settings ``torch.optim.SGD`` (dampening 0) would also refuse."""
    if not lr >= 0.0:
        raise ValueError(f"invalid learning rate {lr}")
    if not 0.0 <= momentum < 1.0:
        raise ValueError(f"momentum must be in [0, 1), got {momentum}")
    if not weight_decay >= 0.0:
        raise ValueError(f"weight_decay must be >= 0, got {weight_decay}")
    if nesterov and momentum == 0.0:
        raise ValueError("nesterov needs momentum > 0")


class SGD:
    def __init__(self, parameters, lr: float, momentum: float = 0.0, weight_decay: float = 0.0, nesterov: bool = False,
                 arena=None):
        check_hparams(float(lr), float(momentum), float(weight_decay), bool(nesterov))
        self._params = list(parameters)
        self._lr = float(lr)
        self.momentum, self.weight_decay, self.nesterov = float(momentum), float(weight_decay), bool(nesterov)
        self._arena = arena if arena is not None and all(p.requires_grad for p in self._params) else None
        if self._arena is not None and self.momentum > 0.0:
            self._arena.enable_momentum()
        self._bufs = [None] * len(self._params)   # per-parameter momentum buffers (no arena)

    @property
    def lr(self):
        return self._lr

    @property
    def plain(self):
        """True for the reference's stateless rule (no momentum, no weight decay)."""
        return self.momentum == 0.0 and self.weight_decay == 0.0

    @property
    def arena(self):
        return self._arena

    def _direction(self, w, g, buf):
        """torch.optim.SGD's step direction, same operations in the same order; updates ``buf`` in place."""
        d = g if self.weight_decay == 0.0 else g.add(w, alpha=self.weight_decay)
        if self.momentum == 0.0:
            return d
        buf.mul_(self.momentum).add_(d)           # buf starts at 0: the first step gives buf = d, as torch's clone
        return d.add(buf, alpha=self.momentum) if self.nesterov else buf

    def step(self):
        if self._arena is not None:
            w, g = self._arena.weights, self._arena.grads
            if w.is_cuda:
                from .ops import cuda as K

                if self.plain:
                    K.sgd_step_(w, g, self._lr)
                else:
                    n = self._arena.numel
                    v = self._arena.momentum
                    K.sgd_momentum_step_(w[:n], g[:n], v, self._lr, self.momentum, self.weight_decay, self.nesterov)
            elif self.plain:
                w.add_(g, alpha=-self._lr)
            else:
                w.add_(self._direction(w, g, self._arena.momentum), alpha=-self._lr)
            return
        for i, param in enumerate(self._params):
            if param.requires_grad:
                if self.plain:
                    param.data.sub_(param.grad * self._lr)
                    continue
                if self.momentum > 0.0 and self._bufs[i] is None:
                    self._bufs[i] = torch.zeros_like(param.data)
                param.data.add_(self._direction(param.data, param.grad, self._bufs[i]), alpha=-self._lr)
