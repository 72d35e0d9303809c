// THE fused data-parallel path (SURVEY.md K3 + C3 + K6):
//
//     dW tile = dZ^T X   (mma.sync TF32 / 3xTF32, accumulator in registers)
//       -> pushed from a shared-memory staging tile into the OWNER replica's staging memory over
//          NVLink (P2P st.global), tile by tile while the next tile's operands stream in
//       -> the owner sums the DP partials in fixed rank order (bitwise deterministic, and
//          bit-identical on every replica because only the owner computes the result)
//       -> W_tile -= lr * sum, and the NEW WEIGHTS are written to every replica's W (P2P)
//       -> device-side flags (st.release.sys / ld.acquire.sys, epoch valued) gate each phase.
//
// No NCCL call, no separate optimizer pass, no gradient buffer round trip: per layer ONE
// kernel replaces { wgrad GEMM, grad accumulate, all-reduce, SGD }.  The same protocol is
// also available without the GEMM (dp_reduce_sgd: reduce an already accumulated G), used
// when micro-batches had to accumulate through memory (pipeline stages).
//
// Deadlock freedom: every CTA first pushes ALL its partial tiles (never waits on a peer),
// only then reduces the tiles it owns (waits only on pushes), only then waits for the
// owners of its other tiles.  grid <= #SMs with one CTA per SM, so every CTA of every rank
// is resident; all spins are bounded (trap after ~4 s instead of hanging the GPU).
#include "kernels.h"
#include "ptx.cuh"

#include <algorithm>

namespace ssb {

static constexpr int kThreads = 160;                   // warp 0 TMA, warps 1..4 MMA + push / reduce
static constexpr int kMaxBlockN = 64;                  // a math warp holds a 32 x block_n fp32 accumulator in registers
static constexpr uint32_t kBlockM = 128;
static constexpr uint32_t kBlockK = 32;
static constexpr uint32_t kABytes = kBlockM * 128;
static constexpr uint32_t kPanelBytes = 32 * 128;

__device__ __forceinline__ float4 ld_cg_f4(const float* p) {   // bypass L1: data written by a peer GPU
    float4 v;
    asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_cg_f(const float* p) {
    float v;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ unsigned long long gtime_dp() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define DPDBG(idx) do { if (p.dbg != nullptr && blockIdx.x == 0) p.dbg[idx] = gtime_dp(); } while (0)

struct TileCoord {
    int t, mt, nt, owner, slot;
};
__device__ __forceinline__ TileCoord tile_coord(const DpLayerParams& p, int t) {
    TileCoord c;
    c.t = t; c.mt = t / p.n_tiles_n; c.nt = t % p.n_tiles_n; c.owner = t % p.dp;
    c.slot = p.one_shot ? t : t / p.dp;
    return c;
}
__device__ __forceinline__ int64_t slot_floats(const DpLayerParams& p) { return (int64_t)kBlockM * p.block_n + kBlockM; }
__device__ __forceinline__ float* stage_slot(const DpPeers& peers, const DpLayerParams& p, int owner, int src, int slot,
                                             uint32_t epoch) {
    return peers.stage[owner] + (int64_t)src * p.stage_src_stride + p.stage_offset + (int64_t)slot * slot_floats(p) +
           (p.one_shot ? (int64_t)(epoch & 1u) * p.stage_parity_stride : 0);
}

// one element of the stateful rule: reads and writes the local momentum at arena offset `off`
__device__ __forceinline__ float elem_direction(const DpLayerParams& p, int64_t off, float g, float w) {
    float v = p.opt.V != nullptr ? p.opt.V[off] : 0.f;
    const float d = sgd_direction<false>(g, w, v, p.opt.momentum, p.opt.weight_decay, p.opt.nesterov != 0);
    if (p.opt.V != nullptr) p.opt.V[off] = v;
    return d;
}

// ---- phase B: the owner reduces one tile in rank order, applies SGD, publishes the weights
// Executed by `nthreads` threads (tid in [0, nthreads)), all of which must call it.
// STATEFUL: momentum / weight decay through sgd_direction; the momentum of the tile lives in the reducing replica's
// LOCAL arena p.opt.V (the owner's, or every replica's own with one_shot) and is never published.
template <bool STATEFUL>
__device__ void dp_owner_reduce_tile(const DpPeers& peers, const DpLayerParams& p, const TileCoord& tc, uint32_t epoch,
                                     int tid, int nthreads, int bar_id, int part = 0, int nparts = 1, bool publish = true) {
    const int me = p.rank;
    const float lr = *p.lr;                               // written before the launch: load it under the wait below
    // wait until every replica's partial of this tile has landed in my staging memory
    if (tid < p.dp) wait_flag_ge(peers.arrive[me] + (int64_t)tid * p.slots_per_src + p.slot_flag_base + tc.slot, epoch);
    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthreads) : "memory");
    if (tid == 0) DPDBG(5);

    const int m0 = tc.mt * (int)kBlockM, n0 = tc.nt * p.block_n;
    const int f4_per_row = p.block_n / 4;
    const float* st0 = stage_slot(peers, p, me, 0, tc.slot, epoch);
    const int n_pub = p.one_shot ? 1 : p.dp;              // one-shot: every replica updates only its own W
    const bool vec_ok = (p.ldw % 4) == 0;
    // batches of kU float4 per thread: issue every staging / weight load of the batch first, then
    // reduce in fixed rank order - otherwise each iteration pays a full L2 round trip
    constexpr int kU = 4;
    const int rows_valid = min((int)kBlockM, p.m_total - m0);
    // this CTA's share of the tile rows (helper CTAs split the reduce)
    const int rows_per = (rows_valid + nparts - 1) / nparts;
    const int r_begin = min(rows_valid, part * rows_per), r_end = min(rows_valid, r_begin + rows_per);
    const int limit_f4 = r_end * f4_per_row;                // rows beyond m_total never need work
    for (int f0 = r_begin * f4_per_row + tid; f0 < limit_f4; f0 += nthreads * kU) {
        float4 part[kMaxDp > 4 ? 4 : kMaxDp][kU];           // up to 4 replicas buffered; more are streamed below
        float4 wv[kU];
        const int nbuf = p.dp < 4 ? p.dp : 4;
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int f = f0 + u * nthreads;
            const int r = f / f4_per_row, c4 = f % f4_per_row;
            const int n = n0 + 4 * c4;
            const bool ok = f < limit_f4 && n < p.n_total;
#pragma unroll
            for (int s = 0; s < 4; ++s)
                part[s][u] = (ok && s < nbuf) ? ld_cg_f4(st0 + (int64_t)s * p.stage_src_stride + (int64_t)r * p.block_n + 4 * c4)
                                              : make_float4(0.f, 0.f, 0.f, 0.f);
            const int64_t woff = p.w_offset + (int64_t)(m0 + r) * p.ldw + n;
            wv[u] = (ok && vec_ok && n + 3 < p.n_total) ? *reinterpret_cast<const float4*>(peers.W[me] + woff)
                                                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int f = f0 + u * nthreads;
            const int r = f / f4_per_row, c4 = f % f4_per_row;
            const int m = m0 + r, n = n0 + 4 * c4;
            if (f >= limit_f4 || n >= p.n_total) continue;
            float4 sum = part[0][u];
#pragma unroll
            for (int s = 1; s < 4; ++s)
                if (s < nbuf) { sum.x += part[s][u].x; sum.y += part[s][u].y; sum.z += part[s][u].z; sum.w += part[s][u].w; }
            for (int s = 4; s < p.dp; ++s) {                  // fixed order 0,1,..,dp-1 => deterministic, replica-independent
                const float4 v = ld_cg_f4(st0 + (int64_t)s * p.stage_src_stride + (int64_t)r * p.block_n + 4 * c4);
                sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
            }
            const int64_t woff = p.w_offset + (int64_t)m * p.ldw + n;
            if (vec_ok && n + 3 < p.n_total) {
                float4 w = wv[u];
                if constexpr (STATEFUL) {                      // sum becomes the step direction
                    float4* vp = p.opt.V != nullptr ? reinterpret_cast<float4*>(p.opt.V + woff) : nullptr;
                    float4 v = vp != nullptr ? *vp : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float mu = p.opt.momentum, wd = p.opt.weight_decay;
                    const bool nv = p.opt.nesterov != 0;
                    sum.x = sgd_direction<false>(sum.x, w.x, v.x, mu, wd, nv);
                    sum.y = sgd_direction<false>(sum.y, w.y, v.y, mu, wd, nv);
                    sum.z = sgd_direction<false>(sum.z, w.z, v.z, mu, wd, nv);
                    sum.w = sgd_direction<false>(sum.w, w.w, v.w, mu, wd, nv);
                    if (vp != nullptr) *vp = v;
                }
                w.x -= lr * sum.x; w.y -= lr * sum.y; w.z -= lr * sum.z; w.w -= lr * sum.w;
                if (n_pub == 1) *reinterpret_cast<float4*>(peers.W[me] + woff) = w;
                else for (int r2 = 0; r2 < p.dp; ++r2) *reinterpret_cast<float4*>(peers.W[r2] + woff) = w;   // publish to all replicas
            } else {
                const float sv[4] = {sum.x, sum.y, sum.z, sum.w};
                for (int e = 0; e < 4 && n + e < p.n_total; ++e) {
                    float d = sv[e];
                    if constexpr (STATEFUL) d = elem_direction(p, woff + e, d, peers.W[me][woff + e]);
                    const float w = peers.W[me][woff + e] - lr * d;
                    if (n_pub == 1) peers.W[me][woff + e] = w;
                    else for (int r2 = 0; r2 < p.dp; ++r2) peers.W[r2][woff + e] = w;
                }
            }
        }
    }
    if (tc.nt == 0 && part == 0) {   // bias gradient rides at the end of the slot
        for (int r = tid; r < (int)kBlockM; r += nthreads) {
            const int m = m0 + r;
            if (m >= p.m_total) continue;
            float sum = 0.f;
            for (int s = 0; s < p.dp; ++s)
                sum += ld_cg_f(st0 + (int64_t)s * p.stage_src_stride + (int64_t)kBlockM * p.block_n + r);
            const int64_t boff = p.w_offset + (int64_t)m * p.ldw + p.n_total;
            if constexpr (STATEFUL) sum = elem_direction(p, boff, sum, peers.W[me][boff]);
            const float b = peers.W[me][boff] - lr * sum;
            if (n_pub == 1) peers.W[me][boff] = b;
            else for (int r2 = 0; r2 < p.dp; ++r2) peers.W[r2][boff] = b;
        }
    }
    if (p.one_shot || !publish) return;                   // nothing to publish / the caller publishes all its tiles at once
    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthreads) : "memory");
    if (tid == 0) {
        __threadfence_system();                            // one cumulative fence after the CTA barrier
        for (int r2 = 0; r2 < p.dp; ++r2) st_relaxed_sys(peers.done[r2] + p.tile_flag_base + tc.t, epoch);
    }
}

__device__ __forceinline__ void dp_wait_tile_done(const DpPeers& peers, const DpLayerParams& p, const TileCoord& tc, uint32_t epoch) {
    wait_flag_ge(peers.done[p.rank] + p.tile_flag_base + tc.t, epoch);
}

// =============================================================================================
// Kernel 1: WGRAD GEMM fused with the DP reduction + SGD + weight broadcast (persistent tiles)
// =============================================================================================
template <bool STATEFUL = false>
__global__ void __launch_bounds__(kThreads, 1)
fused_wgrad_dp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const DpLayerParams p, const DpPeers peers) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t smem_base = (raw + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - raw);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = (p.k_total + kBlockK - 1) / kBlockK;
    const int num_tiles = p.n_tiles_m * p.n_tiles_n;
    if (p.helpers > 1 && (blockIdx.x % p.helpers) != 0) {
        // helper CTA (one-shot layers, one tile per CTA group): no GEMM - just its share of the reduce
        const uint32_t epoch_h = *reinterpret_cast<const volatile uint32_t*>(p.epoch_ptr);
        const TileCoord tc = tile_coord(p, blockIdx.x / p.helpers);
        dp_owner_reduce_tile<STATEFUL>(peers, p, tc, epoch_h, threadIdx.x, kThreads, 1, blockIdx.x % p.helpers, p.helpers);
        return;
    }
    const int cta = p.helpers > 1 ? blockIdx.x / p.helpers : blockIdx.x;      // tile-group index
    const int n_cta = p.helpers > 1 ? gridDim.x / p.helpers : gridDim.x;
    const uint32_t b_bytes = p.block_n * 128u;
    const uint32_t stage_bytes = kABytes + b_bytes;
    const uint32_t tile_bytes_k = kBlockM * ((uint32_t)p.block_n * 4u + 16u);
    const uint32_t bar_base = smem_base + p.stages * stage_bytes + tile_bytes_k;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);          // one arrive per math warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    const uint32_t epoch = *reinterpret_cast<const volatile uint32_t*>(p.epoch_ptr);

    if (warp == 0) {
        {   // converged warp, elect.sync-chosen issuing lane
            int it = 0;
            for (int t = cta; t < num_tiles; t += n_cta) {
                const int m0 = (t / p.n_tiles_n) * kBlockM, n0 = (t % p.n_tiles_n) * p.block_n;
                for (int kb = 0; kb < num_kb; ++kb, ++it) {
                    const int s = it % p.stages;
                    const uint32_t ph = (it / p.stages) & 1;
                    mbar_wait(empty_bar(s), ph ^ 1);
                    if (elect_one()) {
                        mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                        const uint32_t a_dst = smem_base + s * stage_bytes, b_dst = a_dst + kABytes;
                        const int k0 = kb * kBlockK;
#pragma unroll
                        for (int i = 0; i < 4; ++i) tma_load_2d(a_dst + i * kPanelBytes, &tmA, full_bar(s), m0 + 32 * i, k0);
                        for (int j = 0; j < p.block_n / 32; ++j)
                            tma_load_2d(b_dst + j * kPanelBytes, &tmB, full_bar(s), n0 + 32 * j, k0);
                    }
                    __syncwarp();
                }
            }
        }
    } else {
        const int q = warp & 3;
        const int m_local = q * 32 + lane;
        const int etid = (warp - 1) * 32 + lane;                 // 0..127 among the math threads
        const int nt = p.block_n / 8;
        // ---------------- phase A: compute every tile, push the partial to its owner
        const bool batch_flags = (num_tiles > (int)gridDim.x) && p.helpers <= 1;   // more than one tile per CTA
        if (etid == 0) DPDBG(0);
        int it = 0, tile_i = 0;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++tile_i) {
            const TileCoord tc = tile_coord(p, t);
            float acc[2][kMaxBlockN / 8][4];
            warp_acc_zero(acc);
            float dbsum = 0.f;
            for (int kb = 0; kb < num_kb; ++kb, ++it) {
                const int s = it % p.stages;
                const uint32_t ph = (it / p.stages) & 1;
                mbar_wait(full_bar(s), ph);
                const uint32_t a_src = smem_base + s * stage_bytes;
                if (p.split) warp_mma_kblock<kMaxBlockN / 8, true, true, true>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, nt, lane);
                else warp_mma_kblock<kMaxBlockN / 8, true, true, false>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, nt, lane);
                if (tc.nt == 0) {
#pragma unroll 8
                    for (int r = 0; r < 32; ++r) dbsum += lds_f32(a_src + operand_off<true>((uint32_t)m_local, (uint32_t)r));
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));
            }
            if (etid == 0 && tile_i == 0) DPDBG(1);
            const int n_dst = p.one_shot ? p.dp : 1;
            // registers -> padded smem tile (one row per thread) -> row-contiguous 512-byte warp stores: each P2P store
            // instruction carries one full contiguous row segment over NVLink instead of 32 scattered 16-byte pieces
            const uint32_t pitch = (uint32_t)p.block_n * 4u + 16u;
            uint8_t* tile = smem_gen + p.stages * stage_bytes;
            warp_acc_to_rows(acc, reinterpret_cast<float*>(tile) + q * 32 * (int)(pitch / 4u), (int)(pitch / 4u), nt, lane);
            if (p.bulk_push) fence_proxy_async_smem();            // every writer, before the barrier: rows are read by the TMA engine
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (p.bulk_push) {
                // one TMA bulk copy per row and destination (the row's writers fenced before the barrier above)
                for (int d = 0; d < n_dst; ++d) {
                    const int dst_rank = p.one_shot ? d : tc.owner;
                    float* dst = stage_slot(peers, p, dst_rank, p.rank, tc.slot, epoch);
                    bulk_copy_s2g(dst + (int64_t)m_local * p.block_n, smem_base + p.stages * stage_bytes + (uint32_t)m_local * pitch,
                                  (uint32_t)p.block_n * 4u);
                }
                tma_store_commit();
                tma_store_wait_all();
                asm volatile("fence.proxy.async;" ::: "memory");
            } else {
                const int ew = warp - 1;                          // 0..3
                const int f4_per_row = p.block_n / 4;
                for (int d = 0; d < n_dst; ++d) {
                    const int dst_rank = p.one_shot ? d : tc.owner;
                    float* dst = stage_slot(peers, p, dst_rank, p.rank, tc.slot, epoch);
                    for (int r = ew; r < (int)kBlockM; r += 4)
                        for (int c4 = lane; c4 < f4_per_row; c4 += 32)
                            *reinterpret_cast<float4*>(dst + (int64_t)r * p.block_n + 4 * c4) =
                                *reinterpret_cast<const float4*>(tile + (size_t)r * pitch + (size_t)c4 * 16);
                }
            }
            if (tc.nt == 0)
                for (int d = 0; d < n_dst; ++d) {
                    const int dst_rank = p.one_shot ? d : tc.owner;
                    stage_slot(peers, p, dst_rank, p.rank, tc.slot, epoch)[(int64_t)kBlockM * p.block_n + m_local] = dbsum;
                }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (etid == 0 && !batch_flags) {
                if (tile_i == 0) DPDBG(2);
                __threadfence_system();                           // partial visible system-wide before the flag(s)
                if (tile_i == 0) DPDBG(3);
                for (int d = 0; d < n_dst; ++d) {
                    const int dst_rank = p.one_shot ? d : tc.owner;
                    st_relaxed_sys(peers.arrive[dst_rank] + (int64_t)p.rank * p.slots_per_src + p.slot_flag_base + tc.slot, epoch);
                }
            }
        }
        if (batch_flags && etid == 0) {
            // several tiles per CTA (wide layers): ONE system fence for all pushes of this CTA, then all arrival flags -
            // a fence per tile costs 4.4 us each and stalls the epilogue warps between tiles
            __threadfence_system();
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const TileCoord tc = tile_coord(p, t);
                const int n_dst = p.one_shot ? p.dp : 1;
                for (int d = 0; d < n_dst; ++d) {
                    const int dst_rank = p.one_shot ? d : tc.owner;
                    st_relaxed_sys(peers.arrive[dst_rank] + (int64_t)p.rank * p.slots_per_src + p.slot_flag_base + tc.slot, epoch);
                }
            }
        }
        // ---------------- phase B: reduce + SGD + publish the tiles this replica owns
        if (etid == 0) DPDBG(4);
        for (int t = cta; t < num_tiles; t += n_cta) {
            const TileCoord tc = tile_coord(p, t);
            if (p.one_shot || tc.owner == p.rank)
                dp_owner_reduce_tile<STATEFUL>(peers, p, tc, epoch, etid, 128, 1, 0, p.helpers > 1 ? p.helpers : 1, /*publish=*/!batch_flags);
        }
        if (batch_flags && !p.one_shot) {
            // all owned tiles of this CTA are reduced and their new weights stored into every replica: one fence, all flags
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (etid == 0) {
                __threadfence_system();
                for (int t = cta; t < num_tiles; t += n_cta) {
                    const TileCoord tc = tile_coord(p, t);
                    if (tc.owner != p.rank) continue;
                    for (int r2 = 0; r2 < p.dp; ++r2) st_relaxed_sys(peers.done[r2] + p.tile_flag_base + tc.t, epoch);
                }
            }
        }
        // ---------------- phase C: wait for the owners of my other tiles
        if (etid == 0) DPDBG(6);
        if (etid == 0 && !p.one_shot) {
            for (int t = cta; t < num_tiles; t += n_cta) {
                const TileCoord tc = tile_coord(p, t);
                if (tc.owner != p.rank) dp_wait_tile_done(peers, p, tc, epoch);
            }
        }
    }
}

// =============================================================================================
// Kernel 2: the same protocol on an already accumulated gradient block G (no GEMM)
// =============================================================================================
template <bool STATEFUL = false>
__global__ void __launch_bounds__(128, 1) dp_reduce_sgd_kernel(const DpLayerParams p, const DpPeers peers) {
    const uint32_t epoch = *reinterpret_cast<const volatile uint32_t*>(p.epoch_ptr);
    const int num_tiles = p.n_tiles_m * p.n_tiles_n;
    const int tid = threadIdx.x;
    const int f4_per_row = p.block_n / 4;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileCoord tc = tile_coord(p, t);
        const int m0 = tc.mt * (int)kBlockM, n0 = tc.nt * p.block_n;
        const int n_dst = p.one_shot ? p.dp : 1;
        for (int f = tid; f < (int)kBlockM * f4_per_row; f += blockDim.x) {
            const int r = f / f4_per_row, c4 = f % f4_per_row;
            const int m = m0 + r, n = n0 + 4 * c4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < p.m_total) {
                const float* g = p.G + (int64_t)m * p.ldg + n;
                if (n + 3 < p.n_total && (p.ldg % 4) == 0) v = *reinterpret_cast<const float4*>(g);
                else {
                    if (n < p.n_total) v.x = g[0];
                    if (n + 1 < p.n_total) v.y = g[1];
                    if (n + 2 < p.n_total) v.z = g[2];
                    if (n + 3 < p.n_total) v.w = g[3];
                }
            }
            for (int d = 0; d < n_dst; ++d) {
                float* dst = stage_slot(peers, p, p.one_shot ? d : tc.owner, p.rank, tc.slot, epoch);
                *reinterpret_cast<float4*>(dst + (int64_t)r * p.block_n + 4 * c4) = v;
            }
        }
        if (tc.nt == 0)
            for (int r = tid; r < (int)kBlockM; r += blockDim.x) {
                const float v = (m0 + r < p.m_total) ? p.G[(int64_t)(m0 + r) * p.ldg + p.n_total] : 0.f;
                for (int d = 0; d < n_dst; ++d)
                    stage_slot(peers, p, p.one_shot ? d : tc.owner, p.rank, tc.slot, epoch)[(int64_t)kBlockM * p.block_n + r] = v;
            }
        __syncthreads();
        if (tid == 0) {
            __threadfence_system();
            for (int d = 0; d < n_dst; ++d)
                st_relaxed_sys(peers.arrive[p.one_shot ? d : tc.owner] + (int64_t)p.rank * p.slots_per_src + p.slot_flag_base + tc.slot, epoch);
        }
    }
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileCoord tc = tile_coord(p, t);
        if (p.one_shot || tc.owner == p.rank) dp_owner_reduce_tile<STATEFUL>(peers, p, tc, epoch, tid, 128, 1);
    }
    if (tid == 0 && !p.one_shot) {
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const TileCoord tc = tile_coord(p, t);
            if (tc.owner != p.rank) dp_wait_tile_done(peers, p, tc, epoch);
        }
    }
}

__global__ void bump_epoch_kernel(uint32_t* epoch) { *epoch = *epoch + 1; }

// =========================================================================== host side
const char* make_tmap_mn(CUtensorMap* map, const float* base, int inner, int outer, int ld);   // tc_gemm.cu

void dp_layer_geometry(int in, int out, int dp, int* block_n, int* n_tiles_m, int* n_tiles_n, int64_t* slots, int64_t* slot_floats_out,
                       int one_shot) {
    *block_n = in >= kMaxBlockN ? kMaxBlockN : (in + 31) / 32 * 32;
    // latency-bound one-shot layers: narrow tiles => 4x more CTAs share the push and the reduce
    if (one_shot && !getenv("SSB_DP_WIDE_TILES")) *block_n = 32;
    *n_tiles_m = (out + (int)kBlockM - 1) / (int)kBlockM;
    *n_tiles_n = (in + *block_n - 1) / *block_n;
    const int64_t tiles = (int64_t)*n_tiles_m * *n_tiles_n;
    *slots = one_shot ? tiles : (tiles + dp - 1) / dp;
    *slot_floats_out = (int64_t)kBlockM * *block_n + kBlockM;
}

const char* fused_dp_plan(FusedDpPlan* plan, const float* dZ, int lddz, const float* X, int ldx, int rows, const DpLayerParams& lp,
                          const DpPeers& peers, int max_ctas, bool split) {
    *plan = FusedDpPlan{};
    if (lp.lr == nullptr) return "fused_dp_plan: lr (the device learning-rate slot) is not set";
    plan->p = lp;
    plan->peers = peers;
    DpLayerParams& p = plan->p;
    p.k_total = rows;
    if (dZ != nullptr) {
        if (const char* e = make_tmap_mn(&plan->tmA, dZ, p.m_total, rows, lddz)) return e;
        if (const char* e = make_tmap_mn(&plan->tmB, X, p.n_total, rows, ldx)) return e;
        p.split = split ? 1 : 0;                  // 3xTF32: the kernel derives the lo parts from the tiles
    }
    const int num_kb = (rows + (int)kBlockK - 1) / (int)kBlockK;
    const int stage_bytes = (int)kABytes + p.block_n * 128;
    const int tile_bytes = (int)kBlockM * (p.block_n * 4 + 16);   // padded transpose tile for coalesced P2P stores
    int stages = (200 * 1024 - tile_bytes) / stage_bytes;
    if (stages > 6) stages = 6;
    if (stages > std::max(num_kb, 2)) stages = std::max(num_kb, 2);
    p.stages = stages;
    plan->smem_bytes = stages * stage_bytes + tile_bytes + 1024 + 8 * (2 * stages) + 16;
    const int tiles = p.n_tiles_m * p.n_tiles_n;
    plan->grid = tiles < max_ctas ? tiles : max_ctas;
    // small one-shot layers: spend idle SMs on the reduce (helper CTAs split the tile rows)
    p.helpers = 1;
    if (dZ != nullptr && p.one_shot && tiles <= 16 && getenv("SSB_DP_HELPERS")) {   // experimental, off by default
        p.helpers = 4;
        plan->grid = tiles * p.helpers;
    }
    return nullptr;
}

static bool stateful(const DpLayerParams& p) { return p.opt.momentum != 0.f || p.opt.weight_decay != 0.f; }

int dp_element_owner(int proto, int in, int out, int ld, int64_t offset, int dp, int m, int n) {
    if (dp <= 1) return -1;
    switch (proto) {
        case DP_PROTO_LL: return (m % (int)kBlockM) / ((int)kBlockM / dp);          // rows per owner = 128 / dp (dp_ll.cu)
        case DP_PROTO_TWO_SHOT: {
            int block_n = 0, tm = 0, tn = 0;
            int64_t slots = 0, slot_floats = 0;
            dp_layer_geometry(in, out, dp, &block_n, &tm, &tn, &slots, &slot_floats, 0);
            const int t = (m / (int)kBlockM) * tn + (n >= in ? 0 : n / block_n);      // the bias rides with tile column 0
            return t % dp;
        }
        case DP_PROTO_NVLS: return (int)(((offset + (int64_t)m * ld + n) / 4) % dp);
        default: return -1;
    }
}

cudaError_t fused_dp_configure() {
    cudaError_t e = cudaFuncSetAttribute(fused_wgrad_dp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(fused_wgrad_dp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
}
cudaError_t launch_fused_wgrad_dp(const FusedDpPlan& plan, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = fused_dp_configure();
        if (e != cudaSuccess) return e;
        configured = true;
    }
    if (stateful(plan.p))
        fused_wgrad_dp_kernel<true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.tmA, plan.tmB, plan.p, plan.peers);
    else
        fused_wgrad_dp_kernel<false><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.tmA, plan.tmB, plan.p, plan.peers);
    return cudaGetLastError();
}
cudaError_t launch_dp_reduce_sgd(const FusedDpPlan& plan, cudaStream_t stream) {
    if (stateful(plan.p)) dp_reduce_sgd_kernel<true><<<plan.grid, 128, 0, stream>>>(plan.p, plan.peers);
    else dp_reduce_sgd_kernel<false><<<plan.grid, 128, 0, stream>>>(plan.p, plan.peers);
    return cudaGetLastError();
}
cudaError_t launch_bump_epoch(uint32_t* epoch, cudaStream_t stream) {
    bump_epoch_kernel<<<1, 1, 0, stream>>>(epoch);
    return cudaGetLastError();
}

}  // namespace ssb
