// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), warp-level TF32
// tensor-core tiles fed from swizzled shared memory, and system-scope flag ops for peer-memory
// protocols.  Nothing here is generic CUDA C++ - this file only compiles for sm_90a.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "activation.h"
#include "dropout.h"
#include "precision.h"
#include "shuffle.h"

namespace ssb {

// ------------------------------------------------------------------ misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// A spin that cannot hang the GPU forever: ~4 s at 2 GHz, then trap (the host sees a
// launch failure instead of a dead box).
#ifndef SSB_SPIN_LIMIT_CYCLES
#define SSB_SPIN_LIMIT_CYCLES (8000000000ll)
#endif

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > SSB_SPIN_LIMIT_CYCLES) __trap();
    }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
// 2-D tiled store shared -> global (bulk group completion).
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_src), "r"(c0), "r"(c1)
                 : "memory");
}
// 2-D tiled reduce-add shared -> global (fp32 add performed in L2).
__device__ __forceinline__ void tma_reduce_add_2d(const void* tmap, uint32_t smem_src, int c0, int c1) {
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_src), "r"(c0), "r"(c1)
                 : "memory");
}
// contiguous bulk copy shared -> global (the destination may be peer memory mapped over NVLink)
__device__ __forceinline__ void bulk_copy_s2g(void* gdst, uint32_t smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// make generic-proxy smem writes visible to the async proxy (TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ thread-block clusters (distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// the shared::cluster address of the same offset in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t smem_addr, uint32_t rank) {
    uint32_t d;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(d) : "r"(smem_addr), "r"(rank));
    return d;
}
// every thread of every CTA of the cluster: release what it wrote before, acquire what the others wrote
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// 16 bytes from registers into a peer's shared memory (dst and bar: shared::cluster addresses from mapa_shared); the
// store counts as 16 bytes of transaction on the peer's mbarrier, and a peer thread that observes that barrier's phase
// complete also observes the data
__device__ __forceinline__ void st_async_v4(uint32_t dst, uint4 v, uint32_t bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(bar) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}

// ------------------------------------------------------------------ warp-level TF32 tensor-core tiles
// Every operand tile in shared memory is made of 128-byte rows (32 fp32) in the TMA SWIZZLE_128B layout: the 16-byte
// chunk index of an element is XOR-ed with (row & 7), rows 128 B apart, tile base 1024 B aligned.
//   K-major  tile [mn rows x 32 k]                     : element (mn, k) in row mn
//   MN-major tile = panels of [32 k-rows x 32 mn] (4 KB): element (mn, k) in row k of panel mn / 32
__device__ __forceinline__ uint32_t sw128_off(uint32_t row, uint32_t col) {
    return row * 128u + ((((col >> 2) ^ row) & 7u) << 4) + ((col & 3u) << 2);
}
template <bool MN>
__device__ __forceinline__ uint32_t operand_off(uint32_t mn, uint32_t k) {
    return MN ? (mn >> 5) * 4096u + sw128_off(k, mn & 31u) : sw128_off(mn, k);
}
// not volatile: the loads may be scheduled across the (register-only) mma.sync; the memory clobber keeps them behind
// the mbarrier waits that make the tiles valid
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// bf16 products: the m16n8k16 BF16 MMA, fp32 accumulate.  Operands are packed two per register, the lower k in the
// lower half.
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// (bf16(lo), bf16(hi)) rounded to nearest even; cvt's first source operand goes to the upper half
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// 3xTF32: x = hi + lo with hi = trunc_tf32(x) (the top 19 bits) and lo = x - hi exact in fp32, so
// a*b ~= lo_a*hi_b + hi_a*lo_b + hi_a*hi_b  (error ~2^-20 relative).  The hi operand is truncated explicitly, so the
// split does not depend on how the tensor core treats the low 13 mantissa bits of its inputs.
__device__ __forceinline__ uint32_t tf32_hi_bits(float x) { return __float_as_uint(x) & 0xFFFFE000u; }

// Tensor-core precision of a product (kernels.h: PREC_TF32 / PREC_3XTF32 / PREC_BF16).
// One warp: D[32 x 8*nt] += A[m_base .. m_base+31, one 32-wide k-block] * B[n_base .. n_base+8*nt-1, same k-block]^T,
// both operands read from swizzled tiles (operand_off).  The k-block's products are summed into a fresh tensor-core
// accumulator and then added to `acc` with an fp32 add, so the accumulated rounding error grows with the number of
// 32-wide k-blocks, not with the number of MMA steps.  PREC_3XTF32: 3xTF32 products, the lo parts derived from the tile.
// PREC_BF16: two m16n8k16 BF16 MMAs per k-block, operands rounded to bf16 in registers (see below).
// acc[i][j][r]: m16 tile i, n8 tile j, mma.sync C fragment register r (rows lane/4 (+8), columns 2*(lane%4) (+1)).
// MI: m16 tiles of the block (2: 32 rows of A, 1: the 16 rows m_base .. m_base+15).  Each (i, j) tile sees the same
// instructions on the same operands whatever MI and NT are, so its sums do not depend on the block shape.
template <int NT, bool A_MN, bool B_MN, int PREC, int MI = 2>
__device__ __forceinline__ void warp_mma_kblock(float (&acc)[MI][NT][4], uint32_t a_tile, uint32_t m_base, uint32_t b_tile,
                                                uint32_t n_base, int nt, int lane) {
    const uint32_t g = (uint32_t)lane >> 2, t = (uint32_t)lane & 3u;
    float part[MI][NT][4];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) part[i][j][r] = 0.f;
    if constexpr (PREC == PREC_BF16) {
        // The loads are the TF32 fragments' at k0 and k0 + 8.  Thread (g, t) holds logical k {2t, 2t+1, 2t+8, 2t+9} of
        // the k16 fragment; they are fed physical k {k0+t, k0+t+4, k0+8+t, k0+12+t}, the same map for A and B, which
        // covers k0 .. k0+15 once over t = 0..3.  A sum over k does not depend on how its terms are numbered, so the
        // shared-memory layout is the TF32 one.
#pragma unroll
        for (uint32_t k0 = 0; k0 < 32u; k0 += 16u) {
            uint32_t a[MI][4];
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const uint32_t r0 = m_base + 16u * i + g;
                a[i][0] = pack_bf16x2(lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t)), lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t + 4u)));
                a[i][1] = pack_bf16x2(lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t)),
                                      lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t + 4u)));
                a[i][2] = pack_bf16x2(lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t + 8u)),
                                      lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t + 12u)));
                a[i][3] = pack_bf16x2(lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t + 8u)),
                                      lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t + 12u)));
            }
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                if (j < nt) {
                    const uint32_t n = n_base + 8u * j + g;
                    const uint32_t b0 = pack_bf16x2(lds_f32(b_tile + operand_off<B_MN>(n, k0 + t)),
                                                    lds_f32(b_tile + operand_off<B_MN>(n, k0 + t + 4u)));
                    const uint32_t b1 = pack_bf16x2(lds_f32(b_tile + operand_off<B_MN>(n, k0 + t + 8u)),
                                                    lds_f32(b_tile + operand_off<B_MN>(n, k0 + t + 12u)));
#pragma unroll
                    for (int i = 0; i < MI; ++i) mma_bf16(part[i][j], a[i], b0, b1);
                }
            }
        }
    } else {
#pragma unroll
        for (uint32_t k0 = 0; k0 < 32u; k0 += 8u) {
            uint32_t ah[MI][4], al[MI][4];
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const uint32_t r0 = m_base + 16u * i + g;
                const float x[4] = {lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t)), lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t)),
                                    lds_f32(a_tile + operand_off<A_MN>(r0, k0 + t + 4u)),
                                    lds_f32(a_tile + operand_off<A_MN>(r0 + 8u, k0 + t + 4u))};
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    ah[i][r] = tf32_hi_bits(x[r]);
                    al[i][r] = __float_as_uint(x[r] - __uint_as_float(ah[i][r]));
                }
            }
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                if (j < nt) {
                    const uint32_t n = n_base + 8u * j + g;
                    const float y0 = lds_f32(b_tile + operand_off<B_MN>(n, k0 + t));
                    const float y1 = lds_f32(b_tile + operand_off<B_MN>(n, k0 + t + 4u));
                    const uint32_t bh0 = tf32_hi_bits(y0), bh1 = tf32_hi_bits(y1);
                    const uint32_t bl0 = __float_as_uint(y0 - __uint_as_float(bh0)), bl1 = __float_as_uint(y1 - __uint_as_float(bh1));
#pragma unroll
                    for (int i = 0; i < MI; ++i) {
                        if (PREC == PREC_3XTF32) {
                            mma_tf32(part[i][j], al[i], bh0, bh1);
                            mma_tf32(part[i][j], ah[i], bl0, bl1);
                        }
                        mma_tf32(part[i][j], ah[i], bh0, bh1);
                    }
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[i][j][r] += part[i][j][r];
}

template <int NT, int MI>
__device__ __forceinline__ void warp_acc_zero(float (&acc)[MI][NT][4]) {
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;
}

// Lane r receives row r of the warp's 32-row block, columns 16*ch .. 16*ch+15, straight from the accumulator fragments
// (warp shuffles, no shared memory).  Every lane of the warp must call it; ch must be a compile-time constant after
// unrolling, so that the fragments stay in registers.
template <int NT>
__device__ __forceinline__ void warp_acc_row16(const float (&acc)[2][NT][4], int ch, float (&v)[16], int lane) {
    const int src_g = lane & 7, hi_tile = lane >> 4, hi_row = (lane >> 3) & 1;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        const int j = 2 * ch + (c >> 3), src = src_g * 4 + ((c & 7) >> 1), e = c & 1;
        const float a0 = __shfl_sync(0xffffffffu, acc[0][j][e], src);
        const float a1 = __shfl_sync(0xffffffffu, acc[0][j][2 + e], src);
        const float a2 = __shfl_sync(0xffffffffu, acc[1][j][e], src);
        const float a3 = __shfl_sync(0xffffffffu, acc[1][j][2 + e], src);
        v[c] = hi_tile ? (hi_row ? a3 : a2) : (hi_row ? a1 : a0);
    }
}

// Accumulator fragments -> a per-warp row-major scratch [32 rows][ld] (ld odd: conflict-free row-per-lane reads), so that
// afterwards lane r reads row r of the warp's block: scratch[lane * ld + column].
template <int NT>
__device__ __forceinline__ void warp_acc_to_rows(const float (&acc)[2][NT][4], float* scratch, int ld, int nt, int lane) {
    const int g = lane >> 2, t = lane & 3;
    __syncwarp();   // the previous readers of the scratch are done
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            if (j < nt) {
                float* r0 = scratch + (16 * i + g) * ld + 8 * j + 2 * t;
                r0[0] = acc[i][j][0];
                r0[1] = acc[i][j][1];
                r0[8 * ld] = acc[i][j][2];
                r0[8 * ld + 1] = acc[i][j][3];
            }
        }
    __syncwarp();
}

// ------------------------------------------------------------------ system-scope flags (peer memory)
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// flag store AFTER an explicit system-scope fence (fence + relaxed store = release pattern; a
// st.release.sys per flag would pay one more ~3 us NVLink-draining fence each)
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void wait_flag_ge(const uint32_t* p, uint32_t target) {
    if (static_cast<int32_t>(ld_acquire_sys(p) - target) >= 0) return;
    const long long t0 = clock64();
    while (static_cast<int32_t>(ld_acquire_sys(p) - target) < 0) {
        if (clock64() - t0 > SSB_SPIN_LIMIT_CYCLES) __trap();
    }
}
// ---- gpu-scope counters: producer kernel -> concurrently running consumer kernel on the same device
__device__ __forceinline__ void red_add_release_gpu(uint32_t* p, uint32_t v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void wait_counter_ge_gpu(const uint32_t* p, uint32_t target) {
    if (static_cast<int32_t>(ld_acquire_gpu(p) - target) >= 0) return;
    const long long t0 = clock64();
    while (static_cast<int32_t>(ld_acquire_gpu(p) - target) < 0) {
        __nanosleep(64);
        if (clock64() - t0 > SSB_SPIN_LIMIT_CYCLES) __trap();
    }
}
// generic-proxy global writes (of another kernel, observed through an acquire) -> this thread's TMA (async proxy) reads
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

__device__ __forceinline__ float4 ld_nc_f4(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}

// ------------------------------------------------------------------ optimizer update rule
// torch.optim.SGD with dampening 0, for one element: returns the step direction d (the caller applies w -= lr * d) and
// updates the momentum buffer v in place.  Every fused update site calls this, so all of them round alike:
//     g' = g + wd * w ;  v = mu * v + g' ;  d = nesterov ? g' + mu * v : v
// With mu == 0 the result is d = g' whatever v holds, so a site without a momentum buffer passes v = 0 and skips the
// store.  The explicitly rounded operations keep the compiler from contracting differently at different sites.
// PLAIN (no momentum, no weight decay) is today's d = g and compiles to exactly the stateless code.
template <bool PLAIN>
__device__ __forceinline__ float sgd_direction(float g, float w, float& v, float mu, float wd, bool nesterov) {
    if constexpr (PLAIN) {
        return g;
    } else {
        const float gp = __fadd_rn(g, __fmul_rn(wd, w));
        v = __fadd_rn(__fmul_rn(mu, v), gp);
        return nesterov ? __fadd_rn(gp, __fmul_rn(mu, v)) : v;
    }
}

// Exponential moving average of one weight: e moves towards the new weight w by alpha, with torch.lerp's formula
//     alpha < 0.5 :  e + alpha * (w - e)          else :  w - (w - e) * (1 - alpha)
// so alpha = 1 gives e = w exactly.  Every update site calls this, and the explicitly rounded operations keep the
// compiler from contracting differently at different sites (ops.functional.ema_lerp_ref is the same formula in torch).
__device__ __forceinline__ float ema_lerp(float e, float w, float alpha) {
    const float diff = __fsub_rn(w, e);
    return alpha < 0.5f ? __fadd_rn(e, __fmul_rn(alpha, diff)) : __fsub_rn(w, __fmul_rn(diff, __fsub_rn(1.f, alpha)));
}

// ------------------------------------------------------------------ softmax cross-entropy, per element of one row
// torch's F.cross_entropy(z, t, reduction="sum") / B with probability targets, for one row of logits z and target t:
//     m = max_k z_k ;  s = sum_k exp(z_k - m) ;  p_k = exp(z_k - m) / s ;  T = sum_k t_k
//     loss = sum_k t_k ((m - z_k) + log s) / B ;   dz_k = (p_k T - t_k) / B
// The shift is the ROW's max, so s >= 1 and log s is exact to an ulp for every row, however far its logits lie below
// the other rows' (the MSE head's reference contract shifts by the micro-batch's max and adds 1e-7).  The gradient is
// the fused form: no division by p, which underflows for confidently wrong rows.  The chain kernel's loss head and
// loss_head_kernel both call these, and the explicitly rounded operations keep the compiler from contracting them
// differently in the two, so each element is formed alike from s, T and log s.  The sums themselves (s, T and the loss)
// run in different orders: the chain head adds a row's classes in order in one lane, loss_head_kernel adds them per lane
// and then across the warp.  The two paths' results can therefore differ in the last bits.
__device__ __forceinline__ float ce_exp(float z, float m) { return expf(__fsub_rn(z, m)); }
__device__ __forceinline__ float ce_prob(float e, float s) { return __fdiv_rn(e, s); }
__device__ __forceinline__ float ce_loss_term(float t, float z, float m, float log_s) {
    return __fmul_rn(t, __fadd_rn(__fsub_rn(m, z), log_s));
}
__device__ __forceinline__ float ce_dlogit(float p, float T, float t, float inv_batch) {
    return __fmul_rn(__fmaf_rn(p, T, -t), inv_batch);
}

// ------------------------------------------------------------------ dropout masks
// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants): 10 rounds of two 32x32 -> 64-bit products, the key bumped
// by the Weyl constants between rounds.  ops/functional.py: philox4x32_10 is the same generator on torch tensors.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}
// Inverted dropout (DropoutSpec): element (feature f, global sample s) of global Linear `layer`'s output in optimizer step
// `step` is kept iff word 0 of Philox4x32-10 with counter (f, s, layer, step) and key (seed lo, seed hi) is >= threshold.
// Every site that drops or scales calls this, so the kernels and the torch oracle draw the same bits.
__device__ __forceinline__ bool dropout_keep(const DropoutSpec& d, uint32_t layer, uint32_t step, uint32_t f, uint32_t s) {
    return philox4x32_10(make_uint4(f, s, layer, step), (uint32_t)d.seed, (uint32_t)(d.seed >> 32)).x >= d.threshold;
}

// ------------------------------------------------------------------ smooth hidden activations (activation.h)
// a = f(z) and the gate g = f'(z) of one pre-activation, for kind GELU (erf form), SiLU or tanh; every kernel that applies
// a smooth activation calls this, and ops/functional.py: activation_ref is the same math in torch.  Precise erff /
// expf / tanhf (no fast-math).  Dropout multiplies both by keep * s afterwards, so the backward is g * dout alone.
__device__ __forceinline__ void act_fwd(int kind, float z, float& a, float& g) {
    if (kind == ACT_GELU) {
        const float c = 0.5f * (1.f + erff(z * 0.70710678118654752f));       // Phi(z)
        a = z * c;
        g = c + z * (expf(-0.5f * z * z) * 0.39894228040143268f);          // Phi(z) + z phi(z)
    } else if (kind == ACT_SILU) {
        const float s = 1.f / (1.f + expf(-z));                            // sigma(z); 0 once expf overflows
        a = z * s;
        g = s * (1.f + z * (1.f - s));
    } else {
        const float t = tanhf(z);
        a = t;
        g = 1.f - t * t;
    }
}
// ReLU of every kernel: max(z, 0) that keeps NaN, as torch's clamp_min and numpy's maximum do (fmaxf alone returns 0
// for a NaN, which would turn a diverged unit into a dead one).  Every other z keeps fmaxf's bits: z <= 0 (-0 included)
// gives +0.
__device__ __forceinline__ float relu_f(float z) { return z != z ? z : fmaxf(z, 0.f); }
// max that propagates NaN (torch's and numpy's max); fmaxf's bits for every other pair.
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }

// act_fwd for every ActKind, ReLU included: a = max(z, 0) and g = 1[z > 0].  The residual kernels store the gate of a
// ReLU layer too (its output x + relu(z) is no longer its own mask); the smooth-only act_fwd stays as the gated kernels
// compile it.
__device__ __forceinline__ void act_fwd_any(int kind, float z, float& a, float& g) {
    if (kind == ACT_RELU) {
        a = relu_f(z);
        g = z > 0.f ? 1.f : 0.f;
    } else {
        act_fwd(kind, z, a, g);
    }
}

// ------------------------------------------------------------------ training-set shuffling
// Dataset row held by position q < n in epoch `epoch` (ShuffleSpec): a 6-round balanced Feistel network on w bits (w the
// smallest even integer >= 2 with 2^w >= n, halves of h = w / 2 bits), whose round function is word 0 of Philox4x32-10
// with counter (R, round, epoch, "SHUF") and key (seed lo, seed hi), masked to h bits.  Cycle walking (apply the network
// again while the value is >= n) turns the permutation of [0, 2^w) into one of [0, n); 2^w <= 4n bounds the expected
// number of passes by 4.  ops/functional.py: shuffle_index is the same map on torch tensors.
__device__ __forceinline__ uint32_t shuffle_index(uint32_t n, uint64_t seed, uint32_t epoch, uint32_t q) {
    int w = 2;
    while ((1ull << w) < (uint64_t)n) w += 2;
    const int h = w >> 1;
    const uint32_t mask = (1u << h) - 1u;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t x = q;
    do {
        uint32_t L = x >> h, R = x & mask;
#pragma unroll 1
        for (uint32_t i = 0; i < 6; ++i) {
            const uint32_t f = philox4x32_10(make_uint4(R, i, epoch, 0x53485546u), k0, k1).x & mask;
            const uint32_t t = L ^ f;
            L = R;
            R = t;
        }
        x = (L << h) | R;
    } while (x >= n);
    return x;
}

}  // namespace ssb
