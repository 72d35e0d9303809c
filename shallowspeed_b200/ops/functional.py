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
    """The mask selects, as in every kernel and torch's own ReLU backward: a masked-off gradient is +0 even when it is
    NaN or +-Inf (a product would make NaN * 0 = NaN)."""
    assert bitmask.dtype == torch.bool
    return torch.where(bitmask, grad_output, 0.0)


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
# dropout: masks drawn from a counter-based generator (Philox4x32-10), the same bits as csrc/kernels/ptx.cuh
# ----------------------------------------------------------------------------
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def _mulhilo32(a: torch.Tensor, m: int):
    """(hi, lo) 32-bit words of a * m for int64 tensors a in [0, 2^32): the 64-bit product is formed from 16-bit halves of
    m so that no intermediate leaves int64."""
    p_lo = a * (m & 0xFFFF)                       # < 2^48
    p_hi = a * (m >> 16)                          # < 2^48, weighs 2^16
    low = p_lo + ((p_hi & 0xFFFF) << 16)          # < 2^49
    return (p_hi >> 16) + (low >> 32), low & _U32


def philox4x32_10(counter, key):
    """Philox4x32-10 (Random123) over broadcastable int64 tensors or ints holding 32-bit words.  ``counter`` is a 4-tuple,
    ``key`` a 2-tuple; returns the 4 output words as int64 tensors."""
    like = next((t for t in (*counter, *key) if isinstance(t, torch.Tensor)), None)
    dev = like.device if like is not None else None
    c0, c1, c2, c3 = (torch.as_tensor(c, dtype=torch.int64, device=dev) & _U32 for c in counter)
    k0, k1 = (torch.as_tensor(k, dtype=torch.int64, device=dev) & _U32 for k in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + PHILOX_W0) & _U32, (k1 + PHILOX_W1) & _U32
        hi0, lo0 = _mulhilo32(c0, PHILOX_M0)
        hi1, lo1 = _mulhilo32(c2, PHILOX_M1)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return c0, c1, c2, c3


def check_dropout(p, seed):
    """Validated (p, seed): 0 <= p < 1 and 0 <= seed < 2**64, else ValueError."""
    if isinstance(p, bool) or not isinstance(p, (int, float)) or not (0.0 <= float(p) < 1.0):
        raise ValueError(f"dropout must be a number in [0, 1), got {p!r}")
    if isinstance(seed, bool) or not isinstance(seed, int) or not (0 <= seed < 2 ** 64):
        raise ValueError(f"dropout_seed must be an integer in [0, 2**64), got {seed!r}")
    return float(p), int(seed)


def dropout_threshold(p: float) -> int:
    """floor(p * 2^32) in fp64: a unit is dropped iff Philox word 0 < threshold."""
    return int(float(p) * 4294967296.0)


def dropout_scale(p: float) -> float:
    """float32(1 / (1 - p)): 1 / (1 - p) in fp64, rounded to fp32 once."""
    import numpy as np

    return float(np.float32(1.0 / (1.0 - float(p))))


def dropout_mask(p: float, seed: int, layer: int, step: int, samples, n_features: int, device=None) -> torch.Tensor:
    """Keep mask [len(samples), n_features] (bool) of the output of global Linear ``layer`` in optimizer step ``step``.
    ``samples``: the rows' positions in the global batch (row n of DP rank r of dp is n * dp + r).  Element (s, f) is
    kept iff word 0 of Philox4x32-10 with counter (f, s, layer, step mod 2^32) and key (seed lo, seed hi) is at least
    ``dropout_threshold(p)``: a pure function of the sample, the layer, the feature and the step."""
    samples = torch.as_tensor(samples, dtype=torch.int64, device=device)
    f = torch.arange(n_features, dtype=torch.int64, device=samples.device).view(1, -1)
    u, _, _, _ = philox4x32_10((f, samples.view(-1, 1), int(layer), int(step) & _U32), (seed & _U32, seed >> 32))
    return u >= dropout_threshold(p)


def dropout_ref(a: torch.Tensor, keep: torch.Tensor, scale: float) -> torch.Tensor:
    """Inverted dropout of ReLU outputs: keep ? a * scale : 0 (one multiply in a's dtype)."""
    return torch.where(keep, a * scale, torch.zeros_like(a))


# ----------------------------------------------------------------------------
# exponential moving average of the weights (torch.optim.swa_utils.get_ema_multi_avg_fn), the same math as
# csrc/kernels/ptx.cuh: ema_lerp
# ----------------------------------------------------------------------------
def check_ema_decay(decay):
    """``decay`` itself, or ValueError unless it is None or a float with 0 < decay < 1."""
    if decay is None:
        return None
    if isinstance(decay, bool) or not isinstance(decay, (int, float)) or not 0.0 < float(decay) < 1.0:
        raise ValueError(f"ema_decay must be None or a float in (0, 1), got {decay!r}")
    return float(decay)


def ema_alpha(decay: float, n: int) -> float:
    """Weight of the new weights in EMA update ``n`` (0-based): 1 for the first update (the EMA becomes the weights),
    else 1 - decay, computed in fp64 and rounded to fp32 once."""
    if n == 0:
        return 1.0
    return float(torch.tensor(1.0 - float(decay), dtype=torch.float64).to(torch.float32))


def ema_lerp_ref(e: torch.Tensor, w: torch.Tensor, alpha: float) -> torch.Tensor:
    """torch.lerp(e, w, alpha)'s formula in fp32, one tensor op per rounding, so nothing can be contracted:
    ``e + alpha * (w - e)`` for alpha < 0.5, else ``w - (w - e) * (1 - alpha)``.  The native kernels match it bit for bit."""
    a = torch.tensor(alpha, dtype=torch.float32, device=e.device)
    diff = w - e
    if alpha < 0.5:
        return e + a * diff
    return w - diff * (torch.ones((), dtype=torch.float32, device=e.device) - a)


# ----------------------------------------------------------------------------
# tensor-core precision of the native GEMMs: the names a user passes and their codes in the native runtime
# (csrc/kernels/precision.h: Precision).  fp32 (the default) = 3xTF32, fp32-equivalent products; tf32 = one TF32 pass;
# bf16 = operands rounded to bf16 (nearest even) in registers, fp32 accumulation.  Storage is fp32 in every mode.
# ----------------------------------------------------------------------------
PRECISION_CODES = {"fp32": 1, "fp32x3": 1, "3xtf32": 1, "tf32": 0, "bf16": 2}


def precision_code(precision) -> int:
    """The native code of a precision name, or ValueError for a name that is not in ``PRECISION_CODES``."""
    if not isinstance(precision, str) or precision not in PRECISION_CODES:
        raise ValueError(f"unknown precision {precision!r}: expected one of {sorted(PRECISION_CODES)}")
    return PRECISION_CODES[precision]


# ----------------------------------------------------------------------------
# hidden-layer activations: f and the gate f' in one pass, the same math as csrc/kernels/ptx.cuh: act_fwd
# ----------------------------------------------------------------------------
# the activations of the hidden Linears and their codes in the native runtime (csrc/kernels/activation.h: ActKind)
ACTIVATION_CODES = {"relu": 0, "gelu": 1, "silu": 2, "tanh": 3}


def check_activation(activation) -> str:
    """The activation name, or ValueError for anything else than relu, gelu, silu or tanh."""
    if not isinstance(activation, str) or activation not in ACTIVATION_CODES:
        raise ValueError(f"unknown activation {activation!r}: expected one of {sorted(ACTIVATION_CODES)}")
    return activation


def activation_ref(kind: str, z: torch.Tensor):
    """(a, gamma) = (f(z), f'(z)) in z's dtype.  gelu: the erf form, torch's ``F.gelu(approximate="none")``; silu:
    ``F.silu``; tanh: ``torch.tanh``; relu: clamp and the 0 / 1 step (its derivative at 0 taken as 0)."""
    check_activation(kind)
    if kind == "gelu":
        c = 0.5 * (1.0 + torch.erf(z * 0.7071067811865476))
        return z * c, c + z * (torch.exp(-0.5 * z * z) * 0.3989422804014327)
    if kind == "silu":
        s = torch.sigmoid(z)
        return z * s, s * (1.0 + z * (1.0 - s))
    if kind == "tanh":
        t = torch.tanh(z)
        return t, 1.0 - t * t
    return z.clamp_min(0.0), (z > 0).to(z.dtype)


def activation(kind: str, z: torch.Tensor):
    """(f(z), f'(z)) of a smooth activation: the stand-alone kernel on CUDA, activation_ref elsewhere."""
    if _use_cuda(z) and kind != "relu":
        from . import cuda as K

        return K.act_fwd(kind, z)
    return activation_ref(kind, z)


def gate_grad(grad_output, gamma):
    """The backward of a smooth activation: grad_output * gamma (gamma already holds dropout's keep * s)."""
    if _use_cuda(grad_output):
        from . import cuda as K

        return K.gate_grad(grad_output, gamma)
    return grad_output * gamma


# ----------------------------------------------------------------------------
# training-set shuffling: a keyed permutation of the dataset rows per epoch, the same map as csrc/kernels/ptx.cuh
# ----------------------------------------------------------------------------
SHUFFLE_WORD = 0x53485546   # "SHUF": the fourth counter word, which keeps these draws apart from dropout's
SHUFFLE_ROUNDS = 6


def check_shuffle_seed(seed):
    """Validated shuffle seed: None (no shuffling) or an integer in [0, 2**64), else ValueError."""
    if seed is None:
        return None
    if isinstance(seed, bool) or not isinstance(seed, int) or not (0 <= seed < 2 ** 64):
        raise ValueError(f"shuffle_seed must be None or an integer in [0, 2**64), got {seed!r}")
    return int(seed)


def shuffle_width(n: int) -> int:
    """w: the smallest even integer >= 2 with 2^w >= n (the Feistel network permutes w-bit values)."""
    w = 2
    while (1 << w) < n:
        w += 2
    return w


def shuffle_index(n: int, seed: int, epoch: int, positions) -> torch.Tensor:
    """Dataset row held by each global position q in [0, n) in epoch ``epoch`` (used mod 2^32): a 6-round balanced
    Feistel network on w = shuffle_width(n) bits, halves of h = w / 2 bits, round i mapping (L, R) to
    (R, L ^ (philox4x32_10((R, i, epoch, SHUFFLE_WORD), (seed lo, seed hi)).x & (2^h - 1))), applied once and then again
    while the value is >= n (cycle walking).  A bijection on [0, n); int64 tensor of positions' shape."""
    if not (1 <= int(n) < 2 ** 32):
        raise ValueError(f"the dataset must hold between 1 and 2**32 - 1 rows, got {n}")
    q = torch.as_tensor(positions, dtype=torch.int64)
    if q.numel() and (int(q.min()) < 0 or int(q.max()) >= n):
        raise ValueError(f"positions must lie in [0, {n})")
    h = shuffle_width(int(n)) // 2
    mask = (1 << h) - 1
    key, e = (seed & _U32, seed >> 32), int(epoch) & _U32

    def network(x):
        L, R = x >> h, x & mask
        for i in range(SHUFFLE_ROUNDS):
            f = philox4x32_10((R, i, e, SHUFFLE_WORD), key)[0] & mask
            L, R = R, L ^ f
        return (L << h) | R

    x = network(q.clone())
    walk = x >= n
    while bool(walk.any()):   # masked cycle walk: only the values still outside [0, n) take another pass
        x[walk] = network(x[walk])
        walk = x >= n
    return x


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
