"""Functional ops: forward math + hand-written gradients (no autograd).

Capability parity with the reference's ``shallowspeed/functional.py:4-44``
(relu, relu_grad, linear, linear_grad, softmax, softmax_grad, mse_loss,
mse_loss_grad), re-designed for the GPU:

* tensors are ``torch.Tensor`` (fp32 storage);
* on a CUDA device every op dispatches to a hand-written sm_90a kernel
  (``csrc/kernels``: tensor-core GEMMs fed by TMA for the three Linear GEMMs,
  a fused loss-head kernel for softmax/MSE) through ``shallowspeed_b200.ops.cuda``;
* on CPU the same math runs through plain torch ops - this is the numerics
  oracle the GPU tests compare against, and the "plumbing" path that runs
  without a GPU (the sequential CPU configuration).

Numerical contracts kept from the reference (SURVEY.md section 2.2(4)):
softmax shifts by the *global* max of the whole micro-batch and adds 1e-7 to
the denominator (functional.py:24-27); the 1/global_batch_size factor lives in
the loss gradient so gradients are *summed* over micro-batches and replicas.

Softmax cross-entropy (``loss="cross_entropy"``, beyond the reference) follows
torch's ``F.cross_entropy(z, t, reduction="sum") / batch_size`` with probability
targets instead: the softmax is per row (no global max, no +1e-7) and its gradient
is the fused ``(p * sum(t) - t) / batch_size``.
"""
from __future__ import annotations

import torch

SOFTMAX_EPS = 1e-7
# the losses a model's head can compute, and their codes in the native runtime (csrc/kernels/kernels.h: LossKind)
LOSS_CODES = {"mse": 0, "cross_entropy": 1}


def check_loss(loss: str) -> str:
    if loss not in LOSS_CODES:
        raise ValueError(f"unknown loss {loss!r}: expected one of {sorted(LOSS_CODES)}")
    return loss


def _use_cuda(*tensors) -> bool:
    return any(t is not None and t.is_cuda for t in tensors)


# ----------------------------------------------------------------------------
# reference (pure torch) implementations -- device agnostic, fp32/fp64
# ----------------------------------------------------------------------------
def relu_ref(input: torch.Tensor) -> torch.Tensor:
    return input.clamp_min(0.0)


def relu_grad_ref(grad_output: torch.Tensor, bitmask: torch.Tensor) -> torch.Tensor:
    assert bitmask.dtype == torch.bool
    return grad_output * bitmask


def linear_ref(input, weight, bias):
    """y = x @ W^T + b   (W is [out, in], b is [1, out] or [out])."""
    return input @ weight.T + bias.reshape(1, -1)


def linear_grad_ref(grad_output, input, weight):
    """returns (dX, dW, db) for y = x @ W^T + b."""
    return grad_output @ weight, grad_output.T @ input, grad_output.sum(dim=0)


def softmax_ref(input):
    e = torch.exp(input - input.max())
    return e / (e.sum(dim=1, keepdim=True) + SOFTMAX_EPS)


def softmax_grad_ref(grad_output, input):
    out = softmax_ref(input)
    g = out * grad_output
    return g - out * g.sum(dim=-1, keepdim=True)


def mse_loss_ref(input, target, batch_size: int):
    assert input.shape == target.shape
    return ((target - input) ** 2).sum() / batch_size


def mse_loss_grad_ref(input, target, batch_size: int):
    return -2 * (target - input) / batch_size


def row_softmax_ref(input):
    """softmax of every row on its own: torch.softmax(input, -1)."""
    e = torch.exp(input - input.max(dim=1, keepdim=True).values)
    return e / e.sum(dim=1, keepdim=True)


def cross_entropy_ref(logits, target, batch_size: int):
    """sum over rows and classes of t * (log-sum-exp(z) - z), divided by the global batch size."""
    m = logits.max(dim=1, keepdim=True).values
    log_s = torch.log(torch.exp(logits - m).sum(dim=1, keepdim=True))
    return (target * ((m - logits) + log_s)).sum() / batch_size


def cross_entropy_grad_ref(logits, target, batch_size: int):
    """d cross_entropy / d logits = (softmax(z) * sum(t) - t) / batch_size, per row."""
    p = row_softmax_ref(logits)
    return (p * target.sum(dim=1, keepdim=True) - target) / batch_size


# ----------------------------------------------------------------------------
# public API (dispatching)
# ----------------------------------------------------------------------------
def relu(input):
    if _use_cuda(input):
        from . import cuda as K

        return K.relu(input)
    return relu_ref(input)


def relu_grad(grad_output, bitmask):
    """``bitmask`` is a bool tensor (input > 0) as in the reference
    (functional.py:8-10).  On CUDA any tensor whose sign encodes the mask is
    accepted as well (the engine passes the layer *output*: y > 0 <=> x > 0)."""
    if _use_cuda(grad_output):
        from . import cuda as K

        return K.relu_grad(grad_output, bitmask)
    return relu_grad_ref(grad_output, bitmask)


def linear(input, weight, bias):
    if _use_cuda(input, weight):
        from . import cuda as K

        return K.linear_fwd(input, weight, bias, relu=False)
    return linear_ref(input, weight, bias)


def linear_grad(grad_output, input, weight):
    if _use_cuda(grad_output, input, weight):
        from . import cuda as K

        return K.linear_grad(grad_output, input, weight)
    return linear_grad_ref(grad_output, input, weight)


def softmax(input):
    if _use_cuda(input):
        from . import cuda as K

        return K.softmax(input)
    return softmax_ref(input)


def softmax_grad(grad_output, input):
    if _use_cuda(grad_output, input):
        from . import cuda as K

        return K.softmax_grad(grad_output, input)
    return softmax_grad_ref(grad_output, input)


def mse_loss(input, target, batch_size: int):
    return mse_loss_ref(input, target, batch_size)


def mse_loss_grad(input, target, batch_size: int):
    if _use_cuda(input, target):
        from . import cuda as K

        return K.mse_loss_grad(input, target, batch_size)
    return mse_loss_grad_ref(input, target, batch_size)


def row_softmax(input):
    """Per-row softmax (the probabilities of a cross-entropy model)."""
    if _use_cuda(input):
        from . import cuda as K

        return K.softmax(input, loss="cross_entropy")
    return row_softmax_ref(input)


def cross_entropy(logits, target, batch_size: int):
    if _use_cuda(logits, target):
        from . import cuda as K

        return K.loss_head_backward(logits, target, batch_size, loss="cross_entropy")[2]
    return cross_entropy_ref(logits, target, batch_size)


def cross_entropy_grad(logits, target, batch_size: int):
    if _use_cuda(logits, target):
        from . import cuda as K

        return K.loss_head_backward(logits, target, batch_size, loss="cross_entropy")[0]
    return cross_entropy_grad_ref(logits, target, batch_size)


def loss_head_backward(logits, target, batch_size: int, loss: str = "mse"):
    """Fused loss head: logits -> softmax -> MSE grad -> softmax Jacobian
    product.  Returns (dlogits, probs, loss_sum).  Equivalent to the reference
    chain MSELoss.backward -> Softmax.backward (layers.py:157-163, 89-93) in a
    single pass (SURVEY.md K5).  ``loss="cross_entropy"``: the row softmax and the
    cross-entropy gradient (p * sum(t) - t) / batch_size instead."""
    check_loss(loss)
    if _use_cuda(logits, target):
        from . import cuda as K

        return K.loss_head_backward(logits, target, batch_size, loss=loss)
    if loss == "cross_entropy":
        return (cross_entropy_grad_ref(logits, target, batch_size), row_softmax_ref(logits),
                cross_entropy_ref(logits, target, batch_size))
    p = softmax_ref(logits)
    dp = mse_loss_grad_ref(p, target, batch_size)
    g = p * dp
    dlogits = g - p * g.sum(dim=-1, keepdim=True)
    return dlogits, p, mse_loss_ref(p, target, batch_size)
