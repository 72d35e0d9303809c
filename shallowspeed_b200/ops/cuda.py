"""Python face of the hand-written sm_90a kernels (``csrc/kernels``).

Every function here launches OUR kernels - there is no torch/cuBLAS fallback: if the
native module is missing on a GPU box the import fails loudly (the driver checks which
.so files were loaded).  Matrices handed to the TMA-fed GEMMs must be fp32 with unit inner
stride, a row pitch that is a multiple of 4 floats and a 16-byte aligned base
(``tma_ready``); tensors that are not get one padded staging copy (``as_tma``).
"""
from __future__ import annotations

import torch

try:
    from .. import _C  # built in-tree: python setup.py build_ext --inplace
except ImportError as e:  # pragma: no cover
    raise ImportError(
        "shallowspeed_b200._C (sm_90a kernels + runtime) is not built. Run "
        "`python setup.py build_ext --inplace` (or __graft_entry__.build())."
    ) from e


def _round_up(x, m):
    return (x + m - 1) // m * m


def tma_ready(t: torch.Tensor) -> bool:
    return (t.dim() == 2 and t.dtype == torch.float32 and t.is_cuda and (t.stride(1) == 1 or t.size(1) == 1)
            and t.stride(0) % 4 == 0 and t.stride(0) >= t.size(1) and t.data_ptr() % 16 == 0)


def empty_padded(rows: int, cols: int, device) -> torch.Tensor:
    """[rows, cols] view of a [rows, round_up(cols, 4)] buffer (TMA-legal row pitch)."""
    # zeros: padding columns may be read by 16-byte-granular TMA accesses and must stay finite
    return torch.zeros(rows, _round_up(cols, 4), dtype=torch.float32, device=device)[:, :cols]


def as_tma(t: torch.Tensor) -> torch.Tensor:
    if tma_ready(t):
        return t
    out = empty_padded(t.size(0), t.size(1), t.device)
    out.copy_(t)
    return out


def _bias_arg(bias, out_dims):
    """bias may be [1, out] / [out] with any element stride (arena bias column)."""
    if bias is None:
        return None, 0
    b = bias.reshape(-1) if bias.dim() == 1 else bias
    if b.dim() == 2:
        assert b.size(0) == 1 and b.size(1) == out_dims
        stride = b.stride(1)
    else:
        assert b.numel() == out_dims
        stride = b.stride(0)
    return b, (stride if out_dims > 1 else 1)


# ------------------------------------------------------------------ GEMMs
# precision: "tf32" = one TF32 tensor-core pass (operands truncated to 10 mantissa bits);
#            "fp32" = 3xTF32: lo parts (x - trunc(x)) of both operands, derived in the kernel, three MMAs per k-slice,
#            error ~2^-20;
#            "bf16" = operands rounded to bf16 (nearest even) in registers, one BF16 MMA per 16 k, fp32 accumulation.
# Other names raise ValueError (functional.precision_code).
PRECISION = "fp32"


def _prec(precision):
    from .functional import precision_code

    return precision_code(precision or PRECISION)


def _act_code(activation):
    from .functional import ACTIVATION_CODES, check_activation

    return ACTIVATION_CODES[check_activation(activation)]


def _drop_arg(dropout):
    """None, or the dropout of the launch as (p, seed, layer, step, row_base, dp, rank): row n of the launch draws the mask
    of sample (row_base + n) * dp + rank (``functional.dropout_mask``)."""
    if dropout is None:
        return None
    p, seed, layer, step, row_base, dp, rank = dropout
    return float(p), int(seed), int(layer), int(step), int(row_base), int(dp), int(rank)


def linear_fwd(x, weight, bias=None, relu=False, out=None, precision=None, k_splits=0, activation="relu", gate=None,
               dropout=None):
    """k_splits: 0 = plain kernel, -1 = planner decides, k >= 2 = force k k-splits (experimental wide-layer variant).
    With ``relu`` the layer is activated by ``activation``; a smooth one stores f'(z) into ``gate`` (a view with ``out``'s
    row pitch) when one is given.  ``dropout`` (see ``_drop_arg``) drops the activated output and its gate."""
    x, weight = as_tma(x), as_tma(weight)
    rows, out_dims = x.size(0), weight.size(0)
    y = out if out is not None else empty_padded(rows, out_dims, x.device)
    b, bstride = _bias_arg(bias, out_dims)
    _C.linear_fwd(x, weight, b, bstride, bool(relu), y, _prec(precision), int(k_splits), _act_code(activation), gate,
                  _drop_arg(dropout))
    return y


def linear_dgrad(dz, weight, mask=None, out=None, precision=None, k_splits=0, activation="relu", dropout=None):
    """dX = dz @ W, masked where ``mask <= 0`` (ReLU; times the dropout scale where it passes when ``dropout`` is given), or
    times ``mask`` for a smooth ``activation``, whose mask is the previous layer's gate."""
    dz, weight = as_tma(dz), as_tma(weight)
    dx = out if out is not None else empty_padded(dz.size(0), weight.size(1), dz.device)
    m = None if mask is None else as_tma(mask)
    _C.linear_dgrad(dz, weight, m, dx, _prec(precision), int(k_splits), _act_code(activation), _drop_arg(dropout))
    return dx


def linear_wgrad(dz, x, grad_w, accumulate=False, grad_b=None, weight=None, lr=0.0, fuse_sgd=False, precision=None,
                 velocity=None, momentum=0.0, weight_decay=0.0, nesterov=False, ema=None, ema_alpha=None):
    """grad_w[out, in] (+)= dz^T @ x ; grad_b (+)= colsum(dz).  With ``fuse_sgd`` the update goes straight into
    ``weight`` (TMA reduce-add of -lr * dW).  ``momentum`` / ``weight_decay`` / ``nesterov`` select the stateful rule
    in that epilogue; ``velocity`` is then the momentum buffer laid out like ``weight`` (same row pitch).  ``lr`` is a
    number or a one-element fp32 CUDA tensor (see ``_lr_arg``).  ``ema`` (laid out like ``weight``, bias in column
    ``in`` with ``grad_b``) moves towards the new weights by ``ema_alpha`` (a number or a device scalar, like ``lr``):
    ``ops.functional.ema_lerp_ref``."""
    dz, x = as_tma(dz), as_tma(x)
    b, bstride = _bias_arg(grad_b, dz.size(1))
    _C.linear_wgrad(dz, x, grad_w, bool(accumulate), b, bstride, weight, _lr_arg(lr), bool(fuse_sgd), _prec(precision),
                    velocity, float(momentum), float(weight_decay), bool(nesterov), ema,
                    None if ema_alpha is None else _lr_arg(ema_alpha))
    return grad_w


def linear_grad(grad_output, input, weight):
    """functional API: returns fresh (dX, dW, db)."""
    dx = linear_dgrad(grad_output, weight)
    out_dims, in_dims = weight.shape
    dW = empty_padded(out_dims, in_dims, weight.device)
    db = torch.empty(out_dims, dtype=torch.float32, device=weight.device)
    linear_wgrad(grad_output, input, dW, accumulate=False, grad_b=db)
    return dx, dW, db


def linear_bwd_accumulate(dout, x, w_block, g_block, in_dims):
    """Module path: dX = dout @ W ; G_block[:, :in] += dout^T x ; G_block[:, in] += colsum(dout)."""
    W = w_block[:, :in_dims]
    dx = linear_dgrad(dout, W)
    linear_wgrad(dout, x, g_block[:, :in_dims], accumulate=True, grad_b=g_block[:, in_dims])
    return dx


# ------------------------------------------------------------------ loss head / softmax
def _loss_code(loss):
    from .functional import LOSS_CODES, check_loss

    return LOSS_CODES[check_loss(loss)]


def softmax(logits, loss="mse"):
    """The probabilities of a model with this loss: the reference's global-max softmax (``"mse"``) or the per-row
    softmax (``"cross_entropy"``)."""
    logits = as_tma(logits)
    p = empty_padded(logits.size(0), logits.size(1), logits.device)
    _C.loss_head(logits, None, p, None, None, 0.0, _loss_code(loss))
    return p


def softmax_grad(grad_output, logits):
    logits, up = as_tma(logits), as_tma(grad_output)
    dz = empty_padded(logits.size(0), logits.size(1), logits.device)
    _C.softmax_grad(logits, up, dz)
    return dz


def loss_head_backward(logits, target, batch_size, loss="mse"):
    """(dlogits, probs, loss) of the whole ``logits`` as one micro-batch, for an MSE or a cross-entropy head."""
    code = _loss_code(loss)
    logits, target = as_tma(logits), as_tma(target)
    r, c = logits.shape
    p, dz = empty_padded(r, c, logits.device), empty_padded(r, c, logits.device)
    out = torch.zeros(1, dtype=torch.float32, device=logits.device)
    _C.loss_head(logits, target, p, dz, out, 1.0 / batch_size, code)
    return dz, p, out[0]


def mse_loss_grad(input, target, batch_size):
    x, t = input.contiguous(), target.contiguous()
    y = torch.empty_like(x)
    _C.axpby(x, t, y, 2.0 / batch_size, -2.0 / batch_size)
    return y


# ------------------------------------------------------------------ elementwise
def relu(x):
    xc = x.contiguous()
    y = torch.empty_like(xc)
    _C.relu_fwd(xc, y)
    return y


def relu_grad(grad_output, mask_or_output):
    """mask_or_output: bool mask, or any fp32 tensor whose sign encodes it (layer output)."""
    g = empty_padded(grad_output.size(0), grad_output.size(1), grad_output.device)
    g.copy_(grad_output)
    m = mask_or_output
    if m.dtype != torch.float32:
        m = m.to(torch.float32)
    _C.relu_mask_(g, as_tma(m))
    return g


def act_fwd(kind, z):
    """(f(z), f'(z)) of a smooth activation ("gelu", "silu" or "tanh") in one pass of the stand-alone kernel."""
    from .functional import ACTIVATION_CODES, check_activation

    code = ACTIVATION_CODES[check_activation(kind)]
    zc = z.contiguous()
    a, g = torch.empty_like(zc), torch.empty_like(zc)
    _C.act_fwd(code, zc, a, g)
    return a, g


def gate_grad(grad_output, gamma):
    """grad_output * gamma (the backward of a smooth activation)."""
    g = empty_padded(grad_output.size(0), grad_output.size(1), grad_output.device)
    g.copy_(grad_output)
    _C.gate_mul_(g, as_tma(gamma))
    return g


def _lr_arg(lr):
    """The update kernels read the learning rate from device memory when they run: a number is written into a device
    scalar on the current stream; a one-element fp32 CUDA tensor is passed through, so its value may still change
    (stream-ordered) after the call."""
    return lr if isinstance(lr, torch.Tensor) else float(lr)


def sgd_step_(weights_flat, grads_flat, lr):
    _C.sgd_(weights_flat, grads_flat, _lr_arg(lr))


def sgd_momentum_step_(weights_flat, grads_flat, momentum_flat, lr, momentum, weight_decay=0.0, nesterov=False, ema=None,
                       ema_alpha=None):
    """torch.optim.SGD's rule (dampening 0) over flat buffers in one pass; ``momentum_flat`` (None when
    ``momentum == 0``) is updated in place.  ``ema`` (flat, like the weights) moves towards the new weights by
    ``ema_alpha`` (``ops.functional.ema_lerp_ref``); with a plain rule the weights round as in ``sgd_step_``."""
    _C.sgd_momentum_(weights_flat, grads_flat, momentum_flat, _lr_arg(lr), float(momentum), float(weight_decay),
                     bool(nesterov), ema, None if ema_alpha is None else _lr_arg(ema_alpha))


def count_correct(pred, target):
    correct = torch.zeros(1, dtype=torch.int32, device=pred.device)
    _C.argmax_correct(as_tma(pred), as_tma(target), correct)
    return correct


def gemm_kernel_count() -> int:
    return _C.gemm_kernel_count()
