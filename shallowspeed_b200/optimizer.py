"""Optimizer.  Parity: ``SGD(parameters, lr).step()`` = ``param.data -= lr * param.grad``
for trainable params (reference ``shallowspeed/optimizer.py:4-13``); stateless.

GPU: when all parameters are views into one ``ParamArena`` the update is a single fused
pass over the flat buffers (one multi-tensor kernel on CUDA, ``csrc/kernels/elementwise.cu``)
instead of one axpy per parameter.  On the native engine's fused path the update happens
inside the wgrad+all-reduce kernel and ``step`` is not called at all.
"""
from __future__ import annotations


class SGD:
    def __init__(self, parameters, lr: float, arena=None):
        self._params = list(parameters)
        self._lr = float(lr)
        self._arena = arena if arena is not None and all(p.requires_grad for p in self._params) else None

    @property
    def lr(self):
        return self._lr

    def step(self):
        if self._arena is not None:
            w, g = self._arena.weights, self._arena.grads
            if w.is_cuda:
                from .ops import cuda as K

                K.sgd_step_(w, g, self._lr)
            else:
                w.add_(g, alpha=-self._lr)
            return
        for param in self._params:
            if param.requires_grad:
                param.data.sub_(param.grad * self._lr)
