// Small fused kernels around the GEMMs (SURVEY.md K4, K5, K6, K8 and the stage-boundary
// ReLU backward).  None of these is FLOP-heavy; they exist to keep the number of launches
// and the number of passes over memory minimal.
#include "kernels.h"
#include "ptx.cuh"

#include <cfloat>
#include <climits>

namespace ssb {

// ---------------------------------------------------------------- block reductions
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max_nan(float v) {   // the MSE head's global max: NaN propagates (softmax_ref)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <bool IS_MAX>
__device__ float block_reduce(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = IS_MAX ? warp_max_nan(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = IS_MAX ? -FLT_MAX : 0.f;
    for (int i = 0; i < nw; ++i) r = IS_MAX ? max_nan(r, scratch[i]) : r + scratch[i];   // fixed order: deterministic
    return r;
}

// ---------------------------------------------------------------- loss head
// One CTA handles the whole micro-batch (rows x cols is tiny: 4..128 x 10).  Keeps the
// reference's softmax contract: shift by the GLOBAL max of the micro-batch, +1e-7 in the
// denominator (functional.py:24-27).
//   MODE 0: probs only (inference / functional.softmax)
//   MODE 1: loss backward: dz = J_softmax^T * (-2 (t - p) * inv_batch), loss = sum (t-p)^2 * inv_batch
//   MODE 2: generic softmax backward with a given upstream gradient
// Softmax cross-entropy (per-row softmax, no global max, no +1e-7; the formulas are ptx.cuh's ce_*):
//   MODE 3: loss backward: probs, dz = (p * sum(t) - t) * inv_batch, loss = sum t ((m - z) + log s) * inv_batch
//   MODE 4: probs only (inference)
template <int MODE>
__global__ void __launch_bounds__(256) loss_head_kernel(const float* __restrict__ logits, int ldl,
                                                        const float* __restrict__ aux, int lda,   // target | upstream
                                                        float* __restrict__ probs, int ldp,
                                                        float* __restrict__ dlogits, int ldd,
                                                        float* __restrict__ loss_out, int rows_total, int cols, float inv_batch,
                                                        int rows_per_block) {
    // one CTA per micro-batch: the global-max / loss contract is per micro-batch
    __shared__ float scratch[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int row0 = blockIdx.x * rows_per_block;
    const int rows = min(rows_per_block, rows_total - row0);
    logits += (size_t)row0 * ldl;
    if (aux != nullptr) aux += (size_t)row0 * lda;
    if (probs != nullptr) probs += (size_t)row0 * ldp;
    if (dlogits != nullptr) dlogits += (size_t)row0 * ldd;
    if (loss_out != nullptr) loss_out += blockIdx.x;

    if constexpr (MODE >= 3) {
        // one warp per row; every reduction is the warp's butterfly (fixed order), the loss then block_reduce's
        float loss = 0.f;
        for (int r = warp; r < rows; r += nw) {
            const float* x = logits + (size_t)r * ldl;
            const float* t = (MODE == 3) ? aux + (size_t)r * lda : nullptr;
            float m = -FLT_MAX;
            for (int c = lane; c < cols; c += 32) m = fmaxf(m, x[c]);
            m = warp_max(m);
            float s = 0.f, T = 0.f;
            for (int c = lane; c < cols; c += 32) {
                s += ce_exp(x[c], m);
                if (MODE == 3) T += t[c];
            }
            s = warp_sum(s);
            if (MODE == 3) T = warp_sum(T);
            const float log_s = logf(s);
            for (int c = lane; c < cols; c += 32) {
                const float pc = ce_prob(ce_exp(x[c], m), s);
                if (probs != nullptr) probs[(size_t)r * ldp + c] = pc;
                if (MODE == 3) {
                    loss += ce_loss_term(t[c], x[c], m, log_s);
                    dlogits[(size_t)r * ldd + c] = ce_dlogit(pc, T, t[c], inv_batch);
                }
            }
        }
        if (MODE == 3 && loss_out != nullptr) {
            const float total = block_reduce<false>(loss, scratch);
            if (threadIdx.x == 0) loss_out[0] = total * inv_batch;
        }
        return;
    }

    float mx = -FLT_MAX;
    for (int i = threadIdx.x; i < rows * cols; i += blockDim.x) mx = max_nan(mx, logits[(size_t)(i / cols) * ldl + (i % cols)]);
    const float gmax = block_reduce<true>(mx, scratch);

    float loss = 0.f;
    for (int r = warp; r < rows; r += nw) {
        const float* x = logits + (size_t)r * ldl;
        float s = 0.f;
        for (int c = lane; c < cols; c += 32) s += expf(x[c] - gmax);
        s = warp_sum(s);
        const float inv = 1.f / (s + 1e-7f);
        float gsum = 0.f;
        for (int c = lane; c < cols; c += 32) {
            const float pc = expf(x[c] - gmax) * inv;
            if (probs != nullptr) probs[(size_t)r * ldp + c] = pc;
            if (MODE == 1) {
                const float d = aux[(size_t)r * lda + c] - pc;
                loss += d * d;
                gsum += pc * (-2.f * d * inv_batch);
            } else if (MODE == 2) {
                gsum += pc * aux[(size_t)r * lda + c];
            }
        }
        if (MODE != 0) {
            gsum = warp_sum(gsum);
            for (int c = lane; c < cols; c += 32) {
                const float pc = expf(x[c] - gmax) * inv;
                const float up = (MODE == 1) ? (-2.f * (aux[(size_t)r * lda + c] - pc) * inv_batch) : aux[(size_t)r * lda + c];
                const float dzv = pc * up - pc * gsum;
                dlogits[(size_t)r * ldd + c] = dzv;
            }
        }
    }
    if (MODE == 1 && loss_out != nullptr) {
        const float total = block_reduce<false>(loss, scratch);
        if (threadIdx.x == 0) loss_out[0] = total * inv_batch;
    }
}

cudaError_t launch_loss_head(const float* logits, int ldl, const float* target, int ldt, float* probs, int ldp,
                             float* dlogits, int ldd, float* loss_out, int rows, int cols, float inv_batch,
                             cudaStream_t stream, int rows_per_mubatch, int loss) {
    if (loss != LOSS_MSE && loss != LOSS_CROSS_ENTROPY) return cudaErrorInvalidValue;
    const int rpb = rows_per_mubatch > 0 ? rows_per_mubatch : rows;
    const int blocks = (rows + rpb - 1) / rpb;
    const bool ce = loss == LOSS_CROSS_ENTROPY;
    if (target != nullptr) {
        if (ce)
            loss_head_kernel<3><<<blocks, 256, 0, stream>>>(logits, ldl, target, ldt, probs, ldp, dlogits, ldd, loss_out, rows, cols, inv_batch, rpb);
        else
            loss_head_kernel<1><<<blocks, 256, 0, stream>>>(logits, ldl, target, ldt, probs, ldp, dlogits, ldd, loss_out, rows, cols, inv_batch, rpb);
    } else {
        if (ce)
            loss_head_kernel<4><<<blocks, 256, 0, stream>>>(logits, ldl, nullptr, 0, probs, ldp, nullptr, 0, nullptr, rows, cols, 0.f, rpb);
        else
            loss_head_kernel<0><<<blocks, 256, 0, stream>>>(logits, ldl, nullptr, 0, probs, ldp, nullptr, 0, nullptr, rows, cols, 0.f, rpb);
    }
    return cudaGetLastError();
}

cudaError_t launch_softmax_grad(const float* logits, int ldl, const float* upstream, int ldu, float* dlogits, int ldd,
                                int rows, int cols, cudaStream_t stream) {
    loss_head_kernel<2><<<1, 256, 0, stream>>>(logits, ldl, upstream, ldu, nullptr, 0, dlogits, ldd, nullptr, rows, cols, 0.f, rows);
    return cudaGetLastError();
}

// ---------------------------------------------------------------- elementwise
__global__ void relu_mask_kernel(float* __restrict__ g, int ldg, const float* __restrict__ y, int ldy, int rows, int cols) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        if (!(y[(size_t)r * ldy + c] > 0.f)) g[(size_t)r * ldg + c] = 0.f;
    }
}
cudaError_t launch_relu_mask(float* g, int ldg, const float* y, int ldy, int rows, int cols, cudaStream_t stream) {
    const long total = (long)rows * cols;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    relu_mask_kernel<<<blocks, 256, 0, stream>>>(g, ldg, y, ldy, rows, cols);
    return cudaGetLastError();
}
__global__ void relu_mask_scaled_kernel(float* __restrict__ g, int ldg, const float* __restrict__ y, int ldy, int rows,
                                        int cols, float scale) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        float* gp = g + (size_t)r * ldg + c;
        *gp = (y[(size_t)r * ldy + c] > 0.f) ? *gp * scale : 0.f;
    }
}
cudaError_t launch_relu_mask_scaled(float* g, int ldg, const float* y, int ldy, int rows, int cols, float scale,
                                    cudaStream_t stream) {
    const long total = (long)rows * cols;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    relu_mask_scaled_kernel<<<blocks, 256, 0, stream>>>(g, ldg, y, ldy, rows, cols, scale);
    return cudaGetLastError();
}

DropoutSpec dropout_spec(double p, uint64_t seed) {
    DropoutSpec d{};
    d.threshold = (uint32_t)(p * 4294967296.0);   // floor: p >= 0
    d.scale = (float)(1.0 / (1.0 - p));
    d.seed = seed;
    d.dp = 1;
    return d;
}

__global__ void relu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = relu_f(x[i]);
}
cudaError_t launch_relu_fwd(const float* x, float* y, long n, cudaStream_t stream) {
    int blocks = (int)((n + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    relu_fwd_kernel<<<blocks, 256, 0, stream>>>(x, y, n);
    return cudaGetLastError();
}

// stage-boundary backward of a smooth activation: the gate replaces the ReLU mask (and its dropout scale)
__global__ void gate_mul_kernel(float* __restrict__ g, int ldg, const float* __restrict__ gamma, int ldgam, int rows,
                                int cols) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        g[(size_t)r * ldg + c] *= gamma[(size_t)r * ldgam + c];
    }
}
cudaError_t launch_gate_mul(float* g, int ldg, const float* gamma, int ldgam, int rows, int cols, cudaStream_t stream) {
    const long total = (long)rows * cols;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    gate_mul_kernel<<<blocks, 256, 0, stream>>>(g, ldg, gamma, ldgam, rows, cols);
    return cudaGetLastError();
}

__global__ void gate_mul_to_kernel(float* __restrict__ out, int ldo, const float* __restrict__ g, int ldg,
                                   const float* __restrict__ gamma, int ldgam, int rows, int cols) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        out[(size_t)r * ldo + c] = g[(size_t)r * ldg + c] * gamma[(size_t)r * ldgam + c];
    }
}
cudaError_t launch_gate_mul_to(float* out, int ldo, const float* g, int ldg, const float* gamma, int ldgam, int rows, int cols,
                               cudaStream_t stream) {
    const long total = (long)rows * cols;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    gate_mul_to_kernel<<<blocks, 256, 0, stream>>>(out, ldo, g, ldg, gamma, ldgam, rows, cols);
    return cudaGetLastError();
}

__global__ void act_fwd_kernel(int kind, const float* __restrict__ z, float* __restrict__ y, float* __restrict__ gamma,
                               long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float a, g;
        act_fwd(kind, z[i], a, g);
        y[i] = a;
        gamma[i] = g;
    }
}
cudaError_t launch_act_fwd(int kind, const float* z, float* y, float* gamma, long n, cudaStream_t stream) {
    if (!act_smooth(kind)) return cudaErrorInvalidValue;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    act_fwd_kernel<<<blocks, 256, 0, stream>>>(kind, z, y, gamma, n);
    return cudaGetLastError();
}

__global__ void axpby_kernel(const float* __restrict__ x, const float* __restrict__ t, float* __restrict__ y, float a, float b, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = a * x[i] + b * t[i];
}
cudaError_t launch_axpby(const float* x, const float* t, float* y, float a, float b, long n, cudaStream_t stream) {
    int blocks = (int)((n + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    axpby_kernel<<<blocks, 256, 0, stream>>>(x, t, y, a, b, n);
    return cudaGetLastError();
}

// flat-arena SGD: one launch for every parameter of the stage (n is a multiple of 4: the
// arena is padded to 128 B); 2 x 16-byte loads in flight per thread per iteration.
__global__ void __launch_bounds__(256) sgd_kernel(float4* __restrict__ w, const float4* __restrict__ g, const float* __restrict__ lr_ptr,
                                                  long n4) {
    const float lr = *lr_ptr;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 a = w[i];
        const float4 b = g[i];
        a.x -= lr * b.x; a.y -= lr * b.y; a.z -= lr * b.z; a.w -= lr * b.w;
        w[i] = a;
    }
}
__global__ void sgd_tail_kernel(float* w, const float* g, const float* lr, long start, long n) {
    const long i = start + blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (i < n) w[i] -= *lr * g[i];
}
cudaError_t launch_sgd(float* w, const float* g, const float* lr, long n, cudaStream_t stream) {
    if (lr == nullptr) return cudaErrorInvalidValue;
    const bool aligned = ((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(g)) & 15) == 0;
    const long n4 = aligned ? n / 4 : 0;
    if (n4 > 0) {
        long blocks = (n4 + 255) / 256;
        if (blocks > 132 * 8) blocks = 132 * 8;
        sgd_kernel<<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<float4*>(w), reinterpret_cast<const float4*>(g), lr, n4);
    }
    const long done = n4 * 4;
    if (done < n) sgd_tail_kernel<<<(int)((n - done + 255) / 256), 256, 0, stream>>>(w, g, lr, done, n);
    return cudaGetLastError();
}

// flat-arena SGD with the stateful rule (sgd_direction): same float4 body and scalar tail as sgd_kernel, plus the
// momentum buffer v (nullptr when momentum == 0: weight decay alone keeps no state).
// EMA: the EMA buffer e moves towards each new weight (ema_lerp, alpha read from the device); without a rule (plain SGD
// with an EMA) the weight update is sgd_kernel's own expression, so the weights do not depend on the EMA.
template <bool EMA>
__device__ __forceinline__ float sgd_momentum_elem(float w, float g, float* v, long i, float lr, float mu, float wd,
                                                   bool nesterov, bool rule) {
    if (EMA && !rule) return w - lr * g;
    float vi = v != nullptr ? v[i] : 0.f;
    const float d = sgd_direction<false>(g, w, vi, mu, wd, nesterov);
    if (v != nullptr) v[i] = vi;
    return w - lr * d;
}
template <bool EMA = false>
__global__ void __launch_bounds__(256) sgd_momentum_kernel(float4* __restrict__ w, const float4* __restrict__ g,
                                                           float4* __restrict__ v, const float* __restrict__ lr_ptr,
                                                           float mu, float wd, int nesterov, long n4,
                                                           float4* __restrict__ e, const float* __restrict__ alpha_ptr) {
    const float lr = *lr_ptr;
    const float alpha = EMA ? *alpha_ptr : 0.f;
    const bool rule = !EMA || mu != 0.f || wd != 0.f;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 a = w[i];
        const float4 b = g[i];
        if (rule) {
            float4 m = v != nullptr ? v[i] : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool nv = nesterov != 0;
            a.x -= lr * sgd_direction<false>(b.x, a.x, m.x, mu, wd, nv);
            a.y -= lr * sgd_direction<false>(b.y, a.y, m.y, mu, wd, nv);
            a.z -= lr * sgd_direction<false>(b.z, a.z, m.z, mu, wd, nv);
            a.w -= lr * sgd_direction<false>(b.w, a.w, m.w, mu, wd, nv);
            if (v != nullptr) v[i] = m;
        } else {
            a.x -= lr * b.x; a.y -= lr * b.y; a.z -= lr * b.z; a.w -= lr * b.w;
        }
        w[i] = a;
        if constexpr (EMA) {
            float4 t = e[i];
            t.x = ema_lerp(t.x, a.x, alpha); t.y = ema_lerp(t.y, a.y, alpha);
            t.z = ema_lerp(t.z, a.z, alpha); t.w = ema_lerp(t.w, a.w, alpha);
            e[i] = t;
        }
    }
}
template <bool EMA = false>
__global__ void sgd_momentum_tail_kernel(float* w, const float* g, float* v, const float* lr, float mu, float wd,
                                         int nesterov, long start, long n, float* e, const float* alpha) {
    const long i = start + blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (i < n) {
        const float nw = sgd_momentum_elem<EMA>(w[i], g[i], v, i, *lr, mu, wd, nesterov != 0, mu != 0.f || wd != 0.f);
        w[i] = nw;
        if constexpr (EMA) e[i] = ema_lerp(e[i], nw, *alpha);
    }
}
cudaError_t launch_sgd_momentum(float* w, const float* g, const float* lr, const SgdState& opt, long n,
                                cudaStream_t stream) {
    if (lr == nullptr || sgd_state_check(opt) != nullptr) return cudaErrorInvalidValue;
    float* v = opt.V;
    float* e = opt.E;
    const bool aligned = ((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(v) |
                           reinterpret_cast<uintptr_t>(e)) & 15) == 0;
    const long n4 = aligned ? n / 4 : 0;
    if (n4 > 0) {
        long blocks = (n4 + 255) / 256;
        if (blocks > 132 * 8) blocks = 132 * 8;
        if (e != nullptr)
            sgd_momentum_kernel<true><<<(int)blocks, 256, 0, stream>>>(
                reinterpret_cast<float4*>(w), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(v), lr, opt.momentum,
                opt.weight_decay, opt.nesterov, n4, reinterpret_cast<float4*>(e), opt.ema_alpha);
        else
            sgd_momentum_kernel<<<(int)blocks, 256, 0, stream>>>(
                reinterpret_cast<float4*>(w), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(v), lr, opt.momentum,
                opt.weight_decay, opt.nesterov, n4, nullptr, nullptr);
    }
    const long done = n4 * 4;
    if (done < n) {
        const int blocks = (int)((n - done + 255) / 256);
        if (e != nullptr)
            sgd_momentum_tail_kernel<true><<<blocks, 256, 0, stream>>>(w, g, v, lr, opt.momentum, opt.weight_decay, opt.nesterov,
                                                                     done, n, e, opt.ema_alpha);
        else
            sgd_momentum_tail_kernel<<<blocks, 256, 0, stream>>>(w, g, v, lr, opt.momentum, opt.weight_decay, opt.nesterov, done,
                                                                 n, nullptr, nullptr);
    }
    return cudaGetLastError();
}

// does (a, ia) come before (b, ib) in argmax order?  NaN is the maximum and the lower index wins a tie, as in
// torch.argmax / numpy.argmax; ib == INT_MAX is the empty candidate.
__device__ __forceinline__ bool argmax_before(float a, int ia, float b, int ib) {
    if (ia == INT_MAX) return false;
    if (ib == INT_MAX) return true;
    if (b != b) return a != a && ia < ib;
    return a != a || a > b || (a == b && ia < ib);
}
// one warp per row: argmax(pred) == argmax(target) (first maximum wins, NaN the largest, like numpy.argmax)
__global__ void argmax_correct_kernel(const float* __restrict__ pred, int ldp, const float* __restrict__ target, int ldt,
                                      int rows, int cols, int* correct) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    float bp = 0.f, bt = 0.f;
    int ip = INT_MAX, it = INT_MAX;
    for (int c = lane; c < cols; c += 32) {
        const float a = pred[(size_t)row * ldp + c], b = target[(size_t)row * ldt + c];
        if (argmax_before(a, c, bp, ip)) { bp = a; ip = c; }
        if (argmax_before(b, c, bt, it)) { bt = b; it = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float op = __shfl_xor_sync(0xffffffffu, bp, o); const int oip = __shfl_xor_sync(0xffffffffu, ip, o);
        const float ot = __shfl_xor_sync(0xffffffffu, bt, o); const int oit = __shfl_xor_sync(0xffffffffu, it, o);
        if (argmax_before(op, oip, bp, ip)) { bp = op; ip = oip; }
        if (argmax_before(ot, oit, bt, it)) { bt = ot; it = oit; }
    }
    if (lane == 0 && ip == it) atomicAdd(correct, 1);
}
cudaError_t launch_argmax_correct(const float* pred, int ldp, const float* target, int ldt, int rows, int cols,
                                  int* correct, cudaStream_t stream) {
    argmax_correct_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(pred, ldp, target, ldt, rows, cols, correct);
    return cudaGetLastError();
}

// ---------------------------------------------------------------- shuffled input staging
// one warp per destination row: lane 0 walks the permutation, the warp copies the sample's x and y rows
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ x_src, const float* __restrict__ y_src,
                                                          ShuffleSpec spec, int batch, float* __restrict__ x_dst, int ldx,
                                                          float* __restrict__ y_dst, int ldy, int rows, int in_dim,
                                                          int out_dim, int vec) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    uint32_t s = 0;
    if (lane == 0) {
        const int64_t q = (int64_t)batch * spec.gbs + (int64_t)row * spec.dp + spec.rank;
        s = shuffle_index(spec.n, spec.seed, spec.epoch, (uint32_t)q);
    }
    s = __shfl_sync(0xffffffffu, s, 0);
    if (x_src != nullptr) {
        const float* src = x_src + (size_t)s * in_dim;
        float* dst = x_dst + (size_t)row * ldx;
        if (vec) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll 4
            for (int c = lane; c < (in_dim >> 2); c += 32) d4[c] = __ldg(s4 + c);
        } else {
            for (int c = lane; c < in_dim; c += 32) dst[c] = __ldg(src + c);
        }
    }
    if (y_src != nullptr) {
        const float* src = y_src + (size_t)s * out_dim;
        float* dst = y_dst + (size_t)row * ldy;
        for (int c = lane; c < out_dim; c += 32) dst[c] = __ldg(src + c);
    }
}
const char* shuffle_spec_check(const ShuffleSpec& spec, int batch, int rows) {
    if (spec.n == 0u) return "the dataset is empty";
    if (spec.dp < 1 || spec.rank < 0 || spec.rank >= spec.dp) return "the DP rank must lie in [0, dp)";
    if (spec.gbs < 1 || rows < 0 || (int64_t)rows * spec.dp > spec.gbs) return "the rows of a rank exceed its share of the global batch";
    if (batch < 0 || (int64_t)(batch + 1) * spec.gbs > (int64_t)spec.n) return "the batch lies past the last full global batch";
    return nullptr;
}

cudaError_t launch_gather_rows(const float* x_src, const float* y_src, const ShuffleSpec& spec, int batch, float* x_dst,
                               int ldx, float* y_dst, int ldy, int rows, int in_dim, int out_dim, cudaStream_t stream) {
    if (shuffle_spec_check(spec, batch, rows) != nullptr) return cudaErrorInvalidValue;
    if ((x_src != nullptr && (x_dst == nullptr || ldx < in_dim)) || (y_src != nullptr && (y_dst == nullptr || ldy < out_dim)))
        return cudaErrorInvalidValue;
    if (rows == 0 || (x_src == nullptr && y_src == nullptr)) return cudaSuccess;
    const int vec = x_src != nullptr && in_dim % 4 == 0 && ldx % 4 == 0 &&
                    ((reinterpret_cast<uintptr_t>(x_src) | reinterpret_cast<uintptr_t>(x_dst)) & 15) == 0;
    gather_rows_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(x_src, y_src, spec, batch, x_dst, ldx, y_dst, ldy, rows, in_dim,
                                                          out_dim, vec);
    return cudaGetLastError();
}

__global__ void shuffle_index_kernel(uint32_t n, uint64_t seed, uint32_t epoch, const int64_t* __restrict__ q,
                                     int64_t* __restrict__ out, long count) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < count; i += (long)gridDim.x * blockDim.x)
        out[i] = (int64_t)shuffle_index(n, seed, epoch, (uint32_t)q[i]);
}
cudaError_t launch_shuffle_index(uint32_t n, uint64_t seed, uint32_t epoch, const int64_t* q, int64_t* out, long count,
                                 cudaStream_t stream) {
    if (n == 0u) return cudaErrorInvalidValue;
    if (count <= 0) return cudaSuccess;
    long blocks = (count + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    shuffle_index_kernel<<<(int)blocks, 256, 0, stream>>>(n, seed, epoch, q, out, count);
    return cudaGetLastError();
}

}  // namespace ssb
