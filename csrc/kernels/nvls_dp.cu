// NVLS data-parallel kernels: the NVSwitch does the reduction and the broadcast.
//
//   nvls_reduce_sgd : W <- W - lr * sum_r G_r   for the whole parameter arena of a stage, ONE launch.
//                     Replica r owns the float4 chunks c with c % dp == r:  g = multimem.ld_reduce(G_mc[c])  (the
//                     switch pulls and sums the dp copies), w = W[c] - lr * g, multimem.st(W_mc[c], w) (the switch
//                     writes every replica, the owner included).  Each element is reduced exactly once and the RESULT
//                     is multicast, so replicas stay bit-identical (SHA-1 assert_sync contract).
//   nvls_allreduce  : G <- sum_r G_r in place (stand-alone collective for the link-roofline benchmark).
//
// Cross-replica ordering uses two flags that live in the multicast allocation:
//   flag_in  += 1 per replica (multimem.red.release) once its gradients are final  -> everyone waits for dp * epoch
//   flag_out += 1 per replica once ALL its CTAs have written their share           -> nobody leaves the kernel before
//                                                                                     dp * epoch (next reader of W / G)
// A replica's CTAs never wait for each other (the last CTA to finish signals and is the only one that waits for
// the peers), the peers' kernels run on other GPUs; the grid is kept <= #SMs so CTA 0 (which announces flag_in) is
// always resident.  Spins are bounded (ptx.cuh: trap, no hang).
#include "kernels/ptx.cuh"
#include "runtime/nvls_context.h"

namespace ssb {

__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float* mc_addr) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc_addr)
                 : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st_f4(float* mc_addr, const float4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void multimem_red_release_add(uint32_t* mc_addr, uint32_t v) {
    asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_addr), "r"(v) : "memory");
}

// STATEFUL (SGD only): momentum / weight decay through sgd_direction; the owner of chunk c reads and writes its unicast
// momentum V[c] (never multicast: no other replica touches chunk c's state).
template <bool SGD, bool STATEFUL = false>
__global__ void __launch_bounds__(256) nvls_reduce_kernel(const NvlsParams p) {
    const uint32_t epoch = *p.epoch + 1u;                     // same value on every replica (one bump per launch)
    const uint32_t target = epoch * (uint32_t)p.dp;
    const float lr = SGD ? *p.lr : 0.f;                      // learning rate of this step (device slot)

    // ---- my gradients are final (stream order: the wgrad kernels of this step precede this launch)
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        __threadfence_system();
        multimem_red_release_add(p.flag_in_mc, 1u);
    }
    if (threadIdx.x == 0) wait_flag_ge(p.flag_in_uc, target);  // every replica's gradients are final
    __syncthreads();

    // ---- my share: float4 chunks c with c % dp == rank
    const int64_t n4 = p.numel / 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i * p.dp + p.rank < n4; i += stride) {
        const int64_t c = i * p.dp + p.rank;
        const float4 g = multimem_ld_reduce_f4(p.G_mc + 4 * c);
        if (SGD) {
            float4 w = *reinterpret_cast<const float4*>(p.W_uc + 4 * c);
            if constexpr (STATEFUL) {
                float4* vp = p.opt.V != nullptr ? reinterpret_cast<float4*>(p.opt.V + 4 * c) : nullptr;
                float4 v = vp != nullptr ? *vp : make_float4(0.f, 0.f, 0.f, 0.f);
                const float mu = p.opt.momentum, wd = p.opt.weight_decay;
                const bool nv = p.opt.nesterov != 0;
                w.x -= lr * sgd_direction<false>(g.x, w.x, v.x, mu, wd, nv);
                w.y -= lr * sgd_direction<false>(g.y, w.y, v.y, mu, wd, nv);
                w.z -= lr * sgd_direction<false>(g.z, w.z, v.z, mu, wd, nv);
                w.w -= lr * sgd_direction<false>(g.w, w.w, v.w, mu, wd, nv);
                if (vp != nullptr) *vp = v;
            } else {
                w.x -= lr * g.x; w.y -= lr * g.y; w.z -= lr * g.z; w.w -= lr * g.w;
            }
            multimem_st_f4(p.W_mc + 4 * c, w);
        } else {
            multimem_st_f4(p.G_mc + 4 * c, g);
        }
    }

    // ---- last CTA of this replica announces "my share is written everywhere"
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int old = atomicAdd(p.cta_done, 1u);
        if (old == gridDim.x - 1u) {
            *p.cta_done = 0u;                                  // re-arm for the next launch (graph replay)
            *p.epoch = epoch;
            __threadfence_system();
            multimem_red_release_add(p.flag_out_mc, 1u);
            // the kernel (= the stream) does not complete before every replica's share has landed in MY memory;
            // only this CTA waits, the others have exited, so a large grid can never starve itself
            wait_flag_ge(p.flag_out_uc, target);
        }
    }
}

static int nvls_grid(const NvlsParams& p, int max_ctas) {
    const int64_t my_chunks = (p.numel / 4 + p.dp - 1) / p.dp;
    int64_t ctas = (my_chunks + 256 * 4 - 1) / (256 * 4);      // ~4 chunks per thread
    if (ctas < 1) ctas = 1;
    if (ctas > max_ctas) ctas = max_ctas;
    return (int)ctas;
}

cudaError_t launch_nvls_reduce_sgd(const NvlsParams& p, int max_ctas, cudaStream_t stream) {
    if (p.lr == nullptr) return cudaErrorInvalidValue;
    if (p.opt.momentum != 0.f || p.opt.weight_decay != 0.f)
        nvls_reduce_kernel<true, true><<<nvls_grid(p, max_ctas), 256, 0, stream>>>(p);
    else
        nvls_reduce_kernel<true><<<nvls_grid(p, max_ctas), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_nvls_allreduce(const NvlsParams& p, int max_ctas, cudaStream_t stream) {
    nvls_reduce_kernel<false><<<nvls_grid(p, max_ctas), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace ssb
