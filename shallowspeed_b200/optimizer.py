"""Optimizer.  Parity: ``SGD(parameters, lr).step()`` = ``param.data -= lr * param.grad``
for trainable params (reference ``shallowspeed/optimizer.py:4-13``); stateless.

Beyond the reference, ``momentum``, ``weight_decay`` and ``nesterov`` follow ``torch.optim.SGD`` with
``dampening=0`` and one parameter group (biases are decayed too)::

    g' = g + weight_decay * w
    v  = momentum * v + g'            (v starts at 0)
    d  = g' + momentum * v if nesterov else v
    w -= lr * d

The defaults are the reference's stateless rule, bit for bit.  ``lr`` may change between steps (``SGD.lr`` is
settable); the rule above uses the current value, so the momentum buffer evolves the same way at any ``lr``.

GPU: when all parameters are views into one ``ParamArena`` the update is a single fused
pass over the flat buffers (one multi-tensor kernel on CUDA, ``csrc/kernels/elementwise.cu``)
instead of one axpy per parameter; the momentum buffer is then the arena's flat ``momentum``
buffer.  On the native engine's fused path the update happens inside the wgrad (+all-reduce)
kernel and ``step`` is not called at all.

``ema_decay`` (None: off) keeps an exponential moving average of the weights, torch's
``AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(ema_decay))``: after every step each element moves towards
the new weight, ``e = lerp(e, w, alpha)`` with ``alpha = ops.functional.ema_alpha(ema_decay, ema_updates)`` (1 for
the first update).  The EMA only observes: the weights and the momentum are what they are without it.  It lives in
the arena's ``ema`` buffer (``arena=`` is required), or in ``ema_buffers`` per parameter without an arena.
"""
from __future__ import annotations

import torch

from .ops.functional import check_ema_decay, ema_alpha, ema_lerp_ref


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
                 arena=None, ema_decay=None):
        check_hparams(float(lr), float(momentum), float(weight_decay), bool(nesterov))
        self.ema_decay = check_ema_decay(ema_decay)
        self._params = list(parameters)
        self._lr = float(lr)
        self.momentum, self.weight_decay, self.nesterov = float(momentum), float(weight_decay), bool(nesterov)
        self._arena = arena if arena is not None and all(p.requires_grad for p in self._params) else None
        if self._arena is not None and self.momentum > 0.0:
            self._arena.enable_momentum()
        self._bufs = [None] * len(self._params)   # per-parameter momentum buffers (no arena)
        self._ema_updates = 0
        self.ema_buffers = None                   # per-parameter EMA (no arena), copies of the weights like enable_ema
        if self.ema_decay is not None:
            if self._arena is not None:
                self._arena.enable_ema()
            else:
                self.ema_buffers = [p.data.clone() if p.requires_grad else None for p in self._params]

    @property
    def ema_updates(self):
        """EMA updates so far (torch's ``n_averaged``): every training step adds one, wherever it runs (``step``, or a
        training plan run by the native engine).  Settable, e.g. by a resume."""
        return self._ema_updates

    @ema_updates.setter
    def ema_updates(self, value):
        if isinstance(value, bool) or int(value) != value or value < 0:
            raise ValueError(f"ema_updates must be an int >= 0, got {value!r}")
        self._ema_updates = int(value)

    @property
    def ema_alpha(self):
        """The alpha of the next EMA update (None without an EMA)."""
        return None if self.ema_decay is None else ema_alpha(self.ema_decay, self._ema_updates)

    @property
    def lr(self):
        """Learning rate of the next ``step`` (and of the next native-engine step, which reads it per step).  Settable,
        e.g. by a learning-rate schedule (``lr_schedule.LRSchedule``); validated like the constructor's."""
        return self._lr

    @lr.setter
    def lr(self, value):
        check_hparams(float(value), self.momentum, self.weight_decay, self.nesterov)
        self._lr = float(value)

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
        alpha = self.ema_alpha
        if self.ema_decay is not None:
            self._ema_updates += 1
        if self._arena is not None:
            w, g = self._arena.weights, self._arena.grads
            e = self._arena.ema
            if w.is_cuda:
                from .ops import cuda as K

                if self.plain and e is None:
                    K.sgd_step_(w, g, self._lr)
                else:   # the EMA rides on the stateful pass, which rounds a plain rule like sgd_step_
                    n = self._arena.numel
                    v = self._arena.momentum
                    K.sgd_momentum_step_(w[:n], g[:n], v, self._lr, self.momentum, self.weight_decay, self.nesterov,
                                         ema=e, ema_alpha=alpha)
                return
            if self.plain:
                w.add_(g, alpha=-self._lr)
            else:
                w.add_(self._direction(w, g, self._arena.momentum), alpha=-self._lr)
            if e is not None:
                n = self._arena.numel
                e.copy_(ema_lerp_ref(e, w[:n], alpha))
            return
        for i, param in enumerate(self._params):
            if param.requires_grad:
                if self.plain:
                    param.data.sub_(param.grad * self._lr)
                else:
                    if self.momentum > 0.0 and self._bufs[i] is None:
                        self._bufs[i] = torch.zeros_like(param.data)
                    param.data.add_(self._direction(param.data, param.grad, self._bufs[i]), alpha=-self._lr)
                if self.ema_buffers is not None:
                    self.ema_buffers[i].copy_(ema_lerp_ref(self.ema_buffers[i], param.data, alpha))
