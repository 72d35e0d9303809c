// Layer-chain kernel for narrow MLPs (every layer width <= 128, any first-layer fan-in).
//
// One CTA owns one micro-batch (<= 128 rows) and walks it through the WHOLE stage in a
// single launch:   forward L layers -> loss head -> backward (dgrad) L-1 layers.
//
//   * activations never leave the SM between layers: the epilogue writes the layer output
//     into shared memory directly in the swizzled K-major layout the next layer's MMAs read
//     as their B operand (and a copy to global for the weight-gradient GEMMs / pipeline);
//   * weights are streamed by a producer thread that runs AHEAD of the math through a deep
//     TMA ring - weight tiles do not depend on activations, so layer l+1's weights are in
//     flight while layer l is being computed;
//   * accumulators live in the registers of the warp whose epilogue consumes them (mma.sync
//     TF32, 3xTF32 for fp32-equivalent products, or BF16); fused epilogues: bias + ReLU (forward),
//     softmax + MSE gradient + softmax Jacobian, or softmax cross-entropy (loss head), ReLU mask (backward).
//
// This removes ~14 dependent kernel launches (and their prologues / cold starts) from the
// critical path of the reference workload; the per-layer kernels in tc_gemm.cu remain the
// general path (wide layers) and compute the weight gradients afterwards.
//
// Cluster form (CLUSTER, C = ChainParams::cluster CTAs per feature slice): CTA rank c < C of the micro-batch's
// thread-block cluster owns output features [32c, 32c + 32) of every GEMM and streams only that slice of each weight
// matrix.  Each of its eight math warps owns m16n8 tiles of that output (chain_tile_lo), runs them over all k-blocks and
// runs their epilogue on its own fragments.  A first layer of more than 4 k-blocks (more than 128 inputs) is spread over
// P = ChainParams::ksplit = 2 CTAs per slice: rank C + c, the helper of slice c, streams the k-blocks kb with kb % 4 in
// {2, 3} of W_1's 32 rows and of X (chain_ksplit_kblock), the owner those with kb % 4 in {0, 1}.  Every warp sums its
// tiles per k-phase kb % 4; the helper's warps store their two phase sums into the owner (st.async), which adds the four
// in phase order, runs the epilogue and goes on alone - the helper is done after layer 1.  The 32-feature output is
// exactly one K-major panel of the next GEMM's B operand: it is written locally, and each warp stores its block of it
// into the same offset of every other owner (st.async, completion counted on the peer's per-buffer mbarrier; see
// exchange).
#pragma once
#include "kernels.h"
#include "ptx.cuh"

#include <algorithm>

namespace ssb {

static constexpr int kThreads = 288;                      // 1 producer warp + 8 math / epilogue warps
static constexpr uint32_t kBlockM = 128;
static constexpr uint32_t kBlockK = 32;
static constexpr uint32_t kABytes = kBlockM * 128;
static constexpr uint32_t kPanelBytes = 32 * 128;
static constexpr int kScratchLd = 33;                     // odd pitch: conflict-free row-per-lane access
// columns (micro-batch rows) of one math warp: 16 * ceil(N / 32) <= 64
static constexpr int chain_warp_cols(int n_pad) { return 16 * ((n_pad / 16 + 1) / 2); }

// CLUSTER, full-K form: the CTA's 32 x N output is 2 x N/8 m16n8 tiles.  Math warp w (0..7) owns the m16 slab w & 1
// (features 16 (w & 1) .. +15 of the CTA's 32) and the n8 tiles [chain_tile_lo(N/8, w >> 1), chain_tile_lo(N/8, (w >> 1) + 1))
// of it: a quarter of the rows, contiguous, so that the tiles are one warp_mma_kblock block.
__host__ __device__ constexpr int chain_tile_lo(int nj, int quarter) { return nj * quarter / 4; }
// Every byte of a CTA's panel (N rows x 128 B) is in exactly one warp's tiles, so the bytes a peer receives from this
// CTA's senders in one exchange are the N * 128 it armed its recv_bar with for this CTA; and no warp owns more n8
// tiles than the NTW / 2 its accumulator holds.
constexpr bool chain_tiles_cover_panel() {
    for (int n_pad = 16; n_pad <= 128; n_pad += 16) {
        const int cols = chain_warp_cols(n_pad), ntw = cols <= 16 ? 2 : cols <= 32 ? 4 : 8, nj = n_pad / 8;
        int bytes = 0;
        for (int w = 0; w < 8; ++w) {
            const int tiles = chain_tile_lo(nj, (w >> 1) + 1) - chain_tile_lo(nj, w >> 1);
            if (tiles > ntw / 2) return false;
            bytes += tiles * 8 * 64;                      // 8 rows x 16 features x 4 B
        }
        if (bytes != n_pad * 128) return false;
    }
    return true;
}
static_assert(chain_tiles_cover_panel(), "the full-K tiles of the 8 math warps must cover the CTA's panel exactly once");

// CLUSTER, k-split first layer: the i-th k-block that part h (0: the owner, 1: the helper) of a feature slice streams and
// multiplies, and how many of a GEMM's nkb k-blocks that part has.  Part h takes the k-phases kb % 4 in {2h, 2h + 1}, in
// increasing kb, so its i-th k-block is in phase 2h + (i & 1) and each phase's k-blocks come in k-block order.
__host__ __device__ constexpr int chain_ksplit_kblock(int i, int part) { return 4 * (i >> 1) + 2 * part + (i & 1); }
__host__ __device__ constexpr int chain_ksplit_count(int nkb, int part) {
    const int tail = nkb % 4 - 2 * part;                  // k-blocks of the last, partial group of 4 in this part's phases
    return 2 * (nkb / 4) + (tail < 0 ? 0 : tail > 2 ? 2 : tail);
}

// CLUSTER: the cnt (= CNT when it is a template argument) k-blocks of one ring stage on this warp's tiles.  The k-block
// products are independent, so the unrolled CNT forms overlap them; the k-block sums are added into acc in k-block order
// either way.  a: K-major / MN-major 32-feature weight panels, kPanelBytes apart; b: activation panels.
template <int NT, bool A_MN, int PREC, int CNT>
__device__ __forceinline__ void tile_kblocks(float (&acc)[1][NT][4], int cnt, uint32_t a_src, uint32_t b_src, uint32_t b_step,
                                             uint32_t m_base, uint32_t n_base, int nt, int lane) {
#pragma unroll
    for (int j = 0; j < (CNT > 0 ? CNT : 4); ++j)
        if (CNT > 0 || j < cnt)
            warp_mma_kblock<NT, A_MN, false, PREC, 1>(acc, a_src + j * kPanelBytes, m_base, b_src + j * b_step, n_base, nt, lane);
}
template <int NT, bool A_MN, int PREC>
__device__ __forceinline__ void tile_stage(float (&acc)[1][NT][4], int cnt, uint32_t a_src, uint32_t b_src, uint32_t b_step,
                                           uint32_t m_base, uint32_t n_base, int nt, int lane) {
    if (nt == NT) {                                       // every tile of the accumulator: constant bounds throughout
        switch (cnt) {
            case 4: tile_kblocks<NT, A_MN, PREC, 4>(acc, 4, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            case 3: tile_kblocks<NT, A_MN, PREC, 3>(acc, 3, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            case 2: tile_kblocks<NT, A_MN, PREC, 2>(acc, 2, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            default: tile_kblocks<NT, A_MN, PREC, 1>(acc, 1, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
        }
    } else if (nt > 0) {
        tile_kblocks<NT, A_MN, PREC, 0>(acc, cnt, a_src, b_src, b_step, m_base, n_base, nt, lane);
    }
}
// CLUSTER, k-split layer 1: the cnt (= CNT when it is a template argument) k-blocks of one ring stage, slot j into acc0
// for even j and into acc1 for odd j, so that the products of both k-phases overlap; each accumulator still receives
// its k-blocks in k-block order.  a: K-major 32-feature weight panels; b: the X panels of the stage.
template <int NT, int PREC, int CNT>
__device__ __forceinline__ void ksplit_kblocks(float (&acc0)[1][NT][4], float (&acc1)[1][NT][4], int cnt, uint32_t a_src,
                                               uint32_t b_src, uint32_t b_step, uint32_t m_base, uint32_t n_base, int nt, int lane) {
#pragma unroll
    for (int j = 0; j < (CNT > 0 ? CNT : 4); ++j)
        if (CNT > 0 || j < cnt)
            warp_mma_kblock<NT, false, false, PREC, 1>((j & 1) ? acc1 : acc0, a_src + j * kPanelBytes, m_base, b_src + j * b_step,
                                                        n_base, nt, lane);
}
template <int NT, int PREC>
__device__ __forceinline__ void ksplit_stage(float (&acc0)[1][NT][4], float (&acc1)[1][NT][4], int cnt, uint32_t a_src,
                                             uint32_t b_src, uint32_t b_step, uint32_t m_base, uint32_t n_base, int nt, int lane) {
    if (nt == NT) {                                       // every tile of the accumulators: constant bounds throughout
        switch (cnt) {
            case 4: ksplit_kblocks<NT, PREC, 4>(acc0, acc1, 4, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            case 3: ksplit_kblocks<NT, PREC, 3>(acc0, acc1, 3, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            case 2: ksplit_kblocks<NT, PREC, 2>(acc0, acc1, 2, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
            default: ksplit_kblocks<NT, PREC, 1>(acc0, acc1, 1, a_src, b_src, b_step, m_base, n_base, NT, lane); break;
        }
    } else if (nt > 0) {
        ksplit_kblocks<NT, PREC, 0>(acc0, acc1, cnt, a_src, b_src, b_step, m_base, n_base, nt, lane);
    }
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max_f(float v) {   // NaN-propagating: the MSE head's global max
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// byte offset of element (row n, feature m) inside a K-major SWIZZLE_128B operand tile made of
// 32-feature panels of [n_pad rows x 128 B]
__device__ __forceinline__ uint32_t act_smem_off(int n, int m, uint32_t panel_bytes) {
    const uint32_t c = (uint32_t)(m & 31);
    return (uint32_t)(m >> 5) * panel_bytes + (uint32_t)n * 128u + ((((c >> 2) ^ ((uint32_t)n & 7u))) << 4) + ((c & 3u) << 2);
}

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define DBG(role, idx) do { if (p.dbg != nullptr && blockIdx.x == 0 && (idx) < 256) p.dbg[(role) * 256 + (idx)] = gtime(); } while (0)

// PREC (precision.h) is a compile-time switch: the single-pass TF32 instantiation carries none of the extra products, and
// each precision's instantiations are compiled in a translation unit of their own (see chain_kernel below).
// FOLD (pipeline boundaries inside the kernel, see ChainParams) is a compile-time switch as well: launches without a
// folded boundary use the instantiation without its prologue and its predicated peer stores.
// NTW: n8 tiles of a math warp's accumulator (chain_warp_cols / 8, rounded up to 2, 4 or 8) - sized at compile time
// so that small micro-batches keep their accumulators in a few registers.
// CLUSTER: the cluster form (see the top of the file); never combined with FOLD.
// CE: the loss head computes softmax cross-entropy (ChainParams::loss_kind); a compile-time switch, so the MSE
// instantiations carry none of its code.
// DROP: inverted dropout on every ReLU'd layer (ChainParams::drop); the same kind of switch.  The forward epilogues drop
// and scale before any copy of the activation leaves the registers (operand tile, peer panels, act[l], the folded
// out_peer slot); the dgrad epilogues scale where the mask of a dropped layer passes.
// GATE: a smooth activation (ChainParams::act_kind) on every layer with relu set; the same kind of switch.  The forward
// epilogues apply f (ptx.cuh: act_fwd) instead of the ReLU and store the gate f'(z) (* keep * s under DROP) to
// gate[l] next to the global copy of act[l] (not in inference plans: gate[l] == nullptr); the dZ_L staging and the dgrad
// epilogues multiply by the gate where they test the stored activation, which leaves nothing for DROP to scale there.
// RES: a residual model (ChainParams::res), only together with GATE: every activated layer is gated, ReLU included
// (ptx.cuh: act_fwd_any), and the layers in res_mask carry an identity skip.  Because such a layer has in == out, the
// math warp that owns a fragment (feature, row) of its output owns the same fragment of its input tile and of the
// gradients on either side of it, in both forms (chain_tile_lo; warp (q, half)):
//   * forward: a = x + f(z), x read back from the resident input tile (abuf) in shared memory - the stage's first layer
//     reads it from act[0] (the staged or received input) instead, since its input tile may be in ring slots already
//     reused.  See exchange for why the input tile is still intact when the epilogue reads it;
//   * dgrad of layer l: W_l^T dz_l + g_l before the gate of layer l - 1, where g_l (the pre-gate sum of the dgrad of layer
//     l + 1) stayed in the registers of the warp that produced it; a backward-only launch reads g_L from gout.
template <int PREC, bool FOLD, int NTW, bool CLUSTER, bool CE, bool DROP, bool GATE, bool RES>
__global__ void __launch_bounds__(kThreads, 1) mlp_chain_kernel(const ChainParams p) {
    static_assert(!(FOLD && CLUSTER), "folded pipeline launches run one CTA per micro-batch");
    static_assert(!RES || GATE, "residual models run gated");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t smem_base = (raw + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - raw);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int L = p.n_layers;
    const int N = p.n_pad;                                   // tile N (rows of this micro-batch, padded to 16)
    const int crank = CLUSTER ? (int)cluster_ctarank() : 0;
    // CLUSTER: ranks >= C are the helpers of a k-split layer 1 (p.ksplit == 2); rank: the feature slice
    // [32 rank, 32 rank + 32) of every GEMM, which the helper shares with its owner, rank crank - C
    const bool helper = CLUSTER && crank >= p.cluster;
    const int rank = helper ? crank - p.cluster : crank;
    const int mb = CLUSTER ? (int)blockIdx.x / (p.cluster * p.ksplit) : (int)blockIdx.x;   // micro-batch of this CTA (in the launch)
    const int row0 = (p.mu_base + mb) * p.mb_rows;           // first global row of this micro-batch
    const uint32_t a_bytes = CLUSTER ? kPanelBytes : kABytes;   // one k-block of the weight operand: 32 or 128 features
    const uint32_t b_bytes = (uint32_t)N * 128u;             // one 32-feature panel of an activation tile
    const uint32_t stage_bytes = (uint32_t)p.kps * (a_bytes + b_bytes);   // kps A tiles, then kps X tiles (layer 1)
    const uint32_t stage_b_off = (uint32_t)p.kps * a_bytes;
    const uint32_t abuf_bytes = 4u * b_bytes;
    const uint32_t abuf0 = smem_base + p.stages * stage_bytes;            // activation ping-pong
    const uint32_t bar_base = abuf0 + 2u * abuf_bytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
    auto recv_bar = [&](int b) { return bar_base + 8u * (2 * p.stages + b); };   // CLUSTER: peer panels of abuf b landed
    const uint32_t land_bar = bar_base + 8u * (2 * p.stages + 2);   // CLUSTER, k-split: the helper's phase sums landed
    const uint32_t bars_end = p.stages * stage_bytes + 2u * abuf_bytes + 8u * (2 * p.stages + (CLUSTER ? 3 : 0));
    // CLUSTER, k-split: the helper's phase sums, [2 phases][2 slabs][N / 8 n8 tiles][32 lanes][4] floats = 256 N bytes
    const uint32_t land_off = (bars_end + 15u) & ~15u;
    // loss-head transpose scratch [N][kScratchLd] floats behind the barriers (and the landing area)
    const uint32_t scratch_off = (CLUSTER ? land_off + 256u * (uint32_t)N : bars_end) + 128u;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 8);                      // one arrive per math warp
        }
        if constexpr (CLUSTER) {
            mbar_init(recv_bar(0), 1);                       // the local arm; the peers' bytes are transaction counts
            mbar_init(recv_bar(1), 1);
            mbar_init(land_bar, 1);
        }
        fence_barrier_init();
    }
    if constexpr (CLUSTER) cluster_sync();                   // the peers' barriers are initialised before any copy targets them
    else __syncthreads();

    // number of backward GEMMs: layers L..lo (layer 1's dgrad is skipped on the first stage)
    const int bwd_lo = p.first_stage ? 2 : 1;
    // CLUSTER: a CTA whose feature slice starts at or beyond a GEMM's output width has nothing to compute in it (the
    // 10-class logits on ranks >= 1); producer and math warps skip it alike
    auto idle = [&](int width) { return CLUSTER && 32 * rank >= width; };

    if (warp == 0) {
        // ============================================================ weight (and X) producer
        // The whole warp walks the loop (converged); one elect.sync-chosen lane issues.  Weight tiles do not depend on
        // activations, so the ring runs ahead of the math into the next layer.
        {
            int it = 0;
            auto acquire = [&]() {
                const int s = it % p.stages;
                mbar_wait(empty_bar(s), ((it / p.stages) & 1) ^ 1);
                return s;
            };
            if (p.do_fwd) {
                for (int l = 1; l <= L; ++l) {
                    if (helper && l > 1) break;              // the helper streams layer 1 only
                    if (idle(p.layers[l - 1].out)) continue;
                    const int nkb = (p.layers[l - 1].in + (int)kBlockK - 1) / (int)kBlockK;
                    const bool with_x = (l == 1) && !(FOLD && p.x_from_global);   // folded pipeline input: staged by the epilogue warps
                    // CLUSTER, k-split layer 1: this part's k-blocks (chain_ksplit_kblock), i-th in ring slot i % kps
                    const bool ks = CLUSTER && l == 1 && p.ksplit > 1;
                    const int n_kb = ks ? chain_ksplit_count(nkb, helper ? 1 : 0) : nkb;
                    for (int kb0 = 0; kb0 < n_kb; kb0 += p.kps, ++it) {
                        const int cnt = min(p.kps, n_kb - kb0);
                        const int s = acquire();
                        const uint32_t a_dst = smem_base + s * stage_bytes;
                        if (elect_one()) {
                            DBG(0, it);
                            mbar_arrive_expect_tx(full_bar(s), (uint32_t)cnt * (a_bytes + (with_x ? b_bytes : 0u)));
                            for (int j = 0; j < cnt; ++j) {
                                const int kb = ks ? chain_ksplit_kblock(kb0 + j, helper ? 1 : 0) : kb0 + j;
                                // CLUSTER: the 32 rows of W_l this CTA's features need (32-row box)
                                tma_load_2d(a_dst + j * a_bytes, p.maps + 2 * (l - 1), full_bar(s), kb * kBlockK, 32 * rank);
                                if (with_x)
                                    tma_load_2d(a_dst + stage_b_off + j * b_bytes, p.maps + 2 * L, full_bar(s), kb * kBlockK, row0);
                            }
                        }
                        __syncwarp();
                    }
                }
            }
            if (p.do_bwd && !helper) {
                for (int l = L; l >= bwd_lo; --l) {
                    if (idle(p.layers[l - 1].in)) continue;
                    const int nkb = (p.layers[l - 1].out + (int)kBlockK - 1) / (int)kBlockK;
                    for (int kb0 = 0; kb0 < nkb; kb0 += p.kps, ++it) {
                        const int cnt = min(p.kps, nkb - kb0);
                        const int s = acquire();
                        const uint32_t a_dst = smem_base + s * stage_bytes;
                        if (elect_one()) {
                            DBG(0, it);
                            mbar_arrive_expect_tx(full_bar(s), (uint32_t)cnt * a_bytes);
                            for (int j = 0; j < cnt; ++j) {
                                if constexpr (CLUSTER) {
                                    // MN-major panel `rank` of the k-block: this CTA's 32 output features
                                    tma_load_2d(a_dst + j * a_bytes, p.maps + 2 * (l - 1) + 1, full_bar(s), 32 * rank, (kb0 + j) * kBlockK);
                                } else {
#pragma unroll
                                    for (int i = 0; i < 4; ++i)
                                        tma_load_2d(a_dst + j * kABytes + i * kPanelBytes, p.maps + 2 * (l - 1) + 1, full_bar(s), 32 * i,
                                                    (kb0 + j) * kBlockK);
                                }
                            }
                        }
                        __syncwarp();
                    }
                }
            }
        }
    } else {
        // ============================================================ math + epilogue warps
        // Warp (q, half) owns output features q*32 .. q*32+31 and micro-batch rows [c_lo, c_hi): it runs the tensor-core
        // MMAs of exactly the block its epilogue consumes, so accumulators never leave the warp's registers (lane r reads
        // feature row r through warp_acc_row16).  The activation tile of the next GEMM is written by all 8 warps and
        // published with one named barrier among them.
        // CLUSTER: every GEMM runs in the full-K form: each warp owns its tiles (chain_tile_lo) over all k-blocks and
        // runs their epilogue on its own fragments (a k-split layer 1: over the k-blocks of the owner and the helper).
        // The (q == 0) warps stage a dZ_L read from global memory, feature lane by feature lane.
        const int q = warp & 3;
        const int half = (warp - 1) >> 2;
        const int m = (CLUSTER ? 32 * rank : q * 32) + lane;   // feature handled by this thread in the epilogue
        const bool epi = !CLUSTER || q == 0;                 // this warp runs the row-wise epilogues
        // column (= row of the micro-batch) range of this warp, in chunks of 16
        const int n_chunks = N / 16;
        const int c_lo = 16 * ((n_chunks * half) / 2), c_hi = 16 * ((n_chunks * (half + 1)) / 2);
        const int nt = (c_hi - c_lo) / 8;
        float acc[2][NTW][4];                                // this warp's block of the current layer's product
        // CLUSTER, full-K form: this warp's tiles (features t_f0 + g (+8) of fragment register r >> 1, rows
        // t_n0 + 8 j + 2 (lane & 3) + (r & 1)) and their accumulators (tacc2: the second k-phase of a k-split layer 1)
        const int t_m0 = 16 * ((warp - 1) & 1);              // first feature of the slab, of the CTA's 32
        const int t_f0 = 32 * rank + t_m0 + (lane >> 2);     // feature of fragment registers 0, 1 (2, 3: +8)
        const int t_j0 = chain_tile_lo(N / 8, (warp - 1) >> 1);
        const int t_n0 = 8 * t_j0, tnt = chain_tile_lo(N / 8, ((warp - 1) >> 1) + 1) - t_j0;
        float tacc[1][NTW / 2][4], tacc2[1][NTW / 2][4];
        int it = 0, gemm_i = 0;
        // DROP: keep ? x * scale : 0 for feature f of row n of this micro-batch in local layer l (ptx.cuh: dropout_keep)
        uint32_t drop_step = 0u;
        if constexpr (DROP) drop_step = *p.drop.step;
        auto drop_fwd = [&](float x, int l, int f, int n) {
            const uint32_t sample = (uint32_t)((row0 + n) * p.drop.dp + p.drop.rank);
            return dropout_keep(p.drop, (uint32_t)(p.drop.layer + l - 1), drop_step, (uint32_t)f, sample) ? x * p.drop.scale : 0.f;
        };
        // GATE: a = f(z) and its gate g for feature f of row n in local layer l, both dropped like drop_fwd under DROP
        auto gate_fwd = [&](float z, int l, int f, int n, float& g) {
            float a;
            if constexpr (RES) act_fwd_any(p.act_kind, z, a, g);
            else act_fwd(p.act_kind, z, a, g);
            if constexpr (DROP) {
                const uint32_t sample = (uint32_t)((row0 + n) * p.drop.dp + p.drop.rank);
                const bool keep = dropout_keep(p.drop, (uint32_t)(p.drop.layer + l - 1), drop_step, (uint32_t)f, sample);
                a = keep ? a * p.drop.scale : 0.f;
                g = keep ? g * p.drop.scale : 0.f;
            }
            return a;
        };
        // RES: layer l carries a skip; the skip input x of element (row n, feature f) of layer l, read from the input tile
        // `src` (l >= 2) or from act[0] (l == 1, rows of this micro-batch only); the received g_L of element (n, f)
        auto is_res = [&](int l) { return RES && l >= 1 && l <= L && ((p.res_mask >> (l - 1)) & 1u) != 0u; };
        auto skip_in = [&](int l, uint32_t src, int n, int f) {
            float x = 0.f;
            if (l == 1) {
                if (n < p.mb_rows)
                    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(x) : "l"(p.act[0] + (int64_t)(row0 + n) * p.act_ld[0] + f));
            } else {
                x = *reinterpret_cast<const float*>(smem_gen + (src - smem_base) + act_smem_off(n, f, b_bytes));
            }
            return x;
        };
        auto g_recv = [&](int n, int f) {
            float x = 0.f;
            if (n < p.mb_rows)
                asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(x) : "l"(p.gout + (int64_t)(row0 + n) * p.act_ld[L] + f));
            return x;
        };
        int wbuf = 0;                                        // activation buffer the NEXT epilogue writes
        uint32_t recv_phase = 0u;                            // CLUSTER: parity of recv_bar(b) in bit b
        // CLUSTER: the tile in abuf b is complete once the peers' panels landed (see exchange below)
        auto wait_recv = [&](int b) {
            mbar_wait(recv_bar(b), (recv_phase >> b) & 1u);
            recv_phase ^= 1u << b;
        };
        // D[features, rows] of one layer: A = weights from the ring (K-major forward, MN-major backward), B = the
        // activation tile (layer 1: X from the ring slots) -> acc.  One CTA per micro-batch only.
        auto run_gemm = [&](int nkb, bool a_mn, bool b_from_stage, uint32_t bsrc, bool skip) {
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i);
            warp_acc_zero(acc);
            for (int kb0 = 0; kb0 < nkb && !skip; kb0 += p.kps, ++it) {
                const int cnt = min(p.kps, nkb - kb0);
                const int s = it % p.stages;
                mbar_wait(full_bar(s), (it / p.stages) & 1);
                const uint32_t a_src = smem_base + s * stage_bytes;
                for (int j = 0; j < cnt; ++j) {
                    const uint32_t a_j = a_src + j * a_bytes;
                    const uint32_t b_j = b_from_stage ? a_src + stage_b_off + j * b_bytes : bsrc + (kb0 + j) * b_bytes;
                    const uint32_t m_base = (uint32_t)q * 32u;
                    if (a_mn)
                        warp_mma_kblock<NTW, true, false, PREC>(acc, a_j, m_base, b_j, (uint32_t)c_lo, nt, lane);
                    else
                        warp_mma_kblock<NTW, false, false, PREC>(acc, a_j, m_base, b_j, (uint32_t)c_lo, nt, lane);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));
            }
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i + 1);
            ++gemm_i;
        };
        // CLUSTER, full-K form of run_gemm -> tacc: every k-block of this warp's tiles, summed in k-block order.
        auto run_gemm_tiles = [&](int nkb, bool a_mn, bool b_from_stage, uint32_t bsrc, bool skip) {
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i);
            warp_acc_zero(tacc);
            if (!b_from_stage) wait_recv((int)((bsrc - abuf0) / abuf_bytes));
            for (int kb0 = 0; kb0 < nkb && !skip; kb0 += p.kps, ++it) {
                const int cnt = min(p.kps, nkb - kb0);
                const int s = it % p.stages;
                mbar_wait(full_bar(s), (it / p.stages) & 1);
                const uint32_t a_src = smem_base + s * stage_bytes;
                const uint32_t b_src = b_from_stage ? a_src + stage_b_off : bsrc + kb0 * b_bytes;
                if (a_mn)
                    tile_stage<NTW / 2, true, PREC>(tacc, cnt, a_src, b_src, b_bytes, (uint32_t)t_m0, (uint32_t)t_n0, tnt, lane);
                else
                    tile_stage<NTW / 2, false, PREC>(tacc, cnt, a_src, b_src, b_bytes, (uint32_t)t_m0, (uint32_t)t_n0, tnt, lane);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));
            }
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i + 1);
            ++gemm_i;
        };
        // CLUSTER, k-split layer 1 (p.ksplit == 2) -> tacc of the owner: the CTA's k-blocks of this warp's tiles
        // (chain_ksplit_kblock: ring slot j of a stage holds the CTA's k-block kb0 + j, in k-phase 2 part + ((kb0 + j) & 1)),
        // the CTA's first k-phase summed into tacc and its second into tacc2, each in k-block order.  The helper's warp
        // stores its two phase sums into the owner's landing area (st.async, counted on the owner's land_bar); the
        // owner's warp adds them as ((phase 0 + phase 1) + phase 2) + phase 3.  That is the order in which the four
        // k-phase partial sums were added when four warps of one CTA split the k-blocks, so the results are unchanged.
        // Every warp stores and adds, with or without tiles or features (see idle), so the owner's land_bar always
        // receives the 256 N bytes it is armed with.
        auto run_gemm_ksplit = [&](int nkb, bool skip) {
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i);
            warp_acc_zero(tacc);
            warp_acc_zero(tacc2);
            const int n_kb = chain_ksplit_count(nkb, helper ? 1 : 0);
            for (int kb0 = 0; kb0 < n_kb && !skip; kb0 += p.kps, ++it) {
                const int cnt = min(p.kps, n_kb - kb0);
                const int s = it % p.stages;
                mbar_wait(full_bar(s), (it / p.stages) & 1);
                const uint32_t a_src = smem_base + s * stage_bytes, b_src = a_src + stage_b_off;
                // kb0 is a multiple of kps, so an odd kb0 means one slot per stage (kps == 1), of the second k-phase
                if ((kb0 & 1) == 0)
                    ksplit_stage<NTW / 2, PREC>(tacc, tacc2, cnt, a_src, b_src, b_bytes, (uint32_t)t_m0, (uint32_t)t_n0, tnt, lane);
                else
                    ksplit_stage<NTW / 2, PREC>(tacc2, tacc, 1, a_src, b_src, b_bytes, (uint32_t)t_m0, (uint32_t)t_n0, tnt, lane);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));
            }
            if (threadIdx.x == 32) DBG(1, 2 * gemm_i + 1);
            ++gemm_i;
            // this lane's 16 bytes of tile j, phase 2 + h: land + h * 128 N + j * 512 (tiles numbered slab-major)
            const uint32_t land = smem_base + land_off + (uint32_t)(((((warp - 1) & 1) * (N / 8) + t_j0) * 512) + 16 * lane);
            const uint32_t phase_bytes = 128u * (uint32_t)N;
            if (helper) {
#pragma unroll
                for (int j = 0; j < NTW / 2; ++j) {
                    if (j < tnt) {
                        const uint32_t bar = mapa_shared(land_bar, (uint32_t)rank);
                        const uint4 v2 = make_uint4(__float_as_uint(tacc[0][j][0]), __float_as_uint(tacc[0][j][1]),
                                                    __float_as_uint(tacc[0][j][2]), __float_as_uint(tacc[0][j][3]));
                        const uint4 v3 = make_uint4(__float_as_uint(tacc2[0][j][0]), __float_as_uint(tacc2[0][j][1]),
                                                    __float_as_uint(tacc2[0][j][2]), __float_as_uint(tacc2[0][j][3]));
                        st_async_v4(mapa_shared(land + j * 512u, (uint32_t)rank), v2, bar);
                        st_async_v4(mapa_shared(land + phase_bytes + j * 512u, (uint32_t)rank), v3, bar);
                    }
                }
                return;
            }
            if (threadIdx.x == 32) mbar_arrive_expect_tx(land_bar, 2u * phase_bytes);
            mbar_wait(land_bar, 0);
#pragma unroll
            for (int j = 0; j < NTW / 2; ++j) {
                if (j < tnt) {
                    const uint4 v2 = lds_v4(land + j * 512u), v3 = lds_v4(land + phase_bytes + j * 512u);
                    const float h2[4] = {__uint_as_float(v2.x), __uint_as_float(v2.y), __uint_as_float(v2.z), __uint_as_float(v2.w)};
                    const float h3[4] = {__uint_as_float(v3.x), __uint_as_float(v3.y), __uint_as_float(v3.z), __uint_as_float(v3.w)};
#pragma unroll
                    for (int r = 0; r < 4; ++r) tacc[0][j][r] = ((tacc[0][j][r] + tacc2[0][j][r]) + h2[r]) + h3[r];
                }
            }
        };
        // CLUSTER, full-K form: element r of this warp's tile j
        auto t_row = [&](int j, int r) { return t_n0 + 8 * j + 2 * (lane & 3) + (r & 1); };
        auto t_feat = [&](int r) { return t_f0 + 8 * (r >> 1); };
        auto st_tile = [&](uint32_t dst, int n, int feat, float x) {   // operand tile for the next GEMM
            *reinterpret_cast<float*>(smem_gen + (dst - smem_base) + act_smem_off(n, feat, b_bytes)) = x;
        };
        // dz[l] (and every global store this warp issued before) is complete: one release-add per warp on ready[l]
        // (consumers: the gated weight-gradient / data-parallel kernels running next to this one)
        auto signal_ready = [&](int l) {
            if (p.ready == nullptr) return;
            __syncwarp();
            if (lane == 0) red_add_release_gpu(p.ready + l, 1u);
        };
        auto publish = [&]() {                               // smem tile complete -> every math warp may read it
            if (threadIdx.x == 32) DBG(2, gemm_i);
            asm volatile("bar.sync 2, 256;" ::: "memory");
        };
        // CLUSTER, instead of publish() for a tile another GEMM consumes: this CTA's panel of abuf b goes to the same
        // offset in every peer, sent by the warps that wrote it.  A sending warp's block is rows [n0, n0 + rows) x the
        // 16-byte chunks [ch0, ch0 + 2^lcpr) of each row; it reads the block back (each lane a chunk at a time) and
        // stores it into every peer with st.async, each store counted as 16 bytes on the peer's recv_bar(b).  The
        // blocks of one exchange cover the panel exactly once (chain_tiles_cover_panel), so every peer receives the
        // (C - 1) * N * 128 bytes that one thread of it arms its recv_bar(b) with; run_gemm waits on that.
        // Every CTA sends its whole panel, features or not, so that every CTA takes part in every exchange.  That is
        // what makes the ping-pong reuse safe without a cluster barrier per tile.  A peer writes the tile after next
        // into my abuf b in its epilogue after next, which follows its GEMM on the next tile (abuf b^1), which waited
        // for all of my bytes of the next tile - those of every one of my warps.  Each of my warps sends its part of
        // the next tile only after its own GEMM on this tile finished reading abuf b, so all of my warps are done
        // with abuf b before any peer writes into it.  The same chain puts every byte of a tile on recv_bar(b) in the
        // phase that is awaited for it, and every store into this CTA has landed before it reaches the cluster barrier
        // at the end of the kernel.  The stores read registers, so my buffers carry no outgoing copy to wait for.
        // RES: the forward epilogue of a residual layer reads its skip input from the tile it consumed (abuf b ^ 1 when
        // it writes abuf b).  Nothing overwrites that tile before every warp of every CTA has read it: my warps write it
        // again only in the epilogue after next, behind the publish of this tile, which each of them reaches after its
        // reads; a peer writes it only after its next GEMM, which waits for all my bytes of this tile, and each of my
        // warps sends its part only after its own reads.
        auto exchange = [&](int b, bool sender, int n0, int rows, int ch0, int lcpr) {
            if (sender) {
                __syncwarp();                                // the warp's st.shared of its block -> its lanes' reads
                const uint32_t panel = abuf0 + (uint32_t)b * abuf_bytes + (uint32_t)rank * b_bytes;   // act_smem_off panel
                const uint32_t bar = recv_bar(b);
                for (int k = lane; k < (rows << lcpr); k += 32) {
                    const int n = n0 + (k >> lcpr), c = ch0 + (k & ((1 << lcpr) - 1));
                    const uint32_t src = panel + (uint32_t)n * 128u + ((uint32_t)(c ^ (n & 7)) << 4);
                    const uint4 v = lds_v4(src);
                    for (int r = 0; r < p.cluster; ++r)
                        if (r != rank) st_async_v4(mapa_shared(src, (uint32_t)r), v, mapa_shared(bar, (uint32_t)r));
                }
            }
            publish();
            if (threadIdx.x == 32) mbar_arrive_expect_tx(recv_bar(b), (uint32_t)(p.cluster - 1) * b_bytes);
        };
        // end of a tile the next GEMM reads; CLUSTER: sender / n0 / rows / ch0 / lcpr describe this warp's block of it
        // (see exchange)
        auto hand_over = [&](int b, bool sender, int n0, int rows, int ch0, int lcpr) {
            if constexpr (CLUSTER) exchange(b, sender, n0, rows, ch0, lcpr);
            else publish();
        };
        int buf = 0;                                         // activation buffer the NEXT gemm reads
        // ---------------- folded pipeline boundaries (see ChainParams): credit of the slots we will write, arrival of
        // the tile we consume.  One thread spins (bounded), a named barrier among the 8 math warps publishes the result.
        uint32_t pp_epoch = 0u;
        if constexpr (FOLD) {
        if (p.in_flag != nullptr || p.out_peer != nullptr) {
            pp_epoch = *reinterpret_cast<const volatile uint32_t*>(p.pp_epoch);
            if (threadIdx.x == 32) {
                if (p.out_peer != nullptr) wait_flag_ge(p.out_credit, pp_epoch - 1u);
                if (p.in_flag != nullptr) wait_flag_ge(p.in_flag, pp_epoch);
            }
            asm volatile("bar.sync 2, 256;" ::: "memory");
        }
        if (p.do_fwd && p.x_from_global) {
            // stage the input tile [rows x in] (written into act[0] by the previous stage over NVLink) as layer 1's B operand
            // in abuf 1
            const int in0 = p.layers[0].in;
            const uint32_t dstx = abuf0 + 1u * abuf_bytes;
            const float* __restrict__ xin = p.act[0] + (int64_t)row0 * p.act_ld[0];
            for (int n = c_lo; n < c_hi; ++n) {
                float x = 0.f;
                if (m < in0 && n < p.mb_rows)
                    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(x) : "l"(xin + (int64_t)n * p.act_ld[0] + m));
                st_tile(dstx, n, m, x);
            }
            publish();
        }
        }   // FOLD
        if (p.do_fwd) {
            for (int l = 1; l <= L; ++l) {
                const ChainLayer& ly = p.layers[l - 1];
                const bool m_ok = m < ly.out;
                const float bias = m_ok ? __ldg(p.W + ly.w_off + (int64_t)m * ly.ldw + ly.in) : 0.f;
                const bool is_logits = (l == L) && p.do_loss;
                const int nkb_f = (ly.in + (int)kBlockK - 1) / (int)kBlockK;
                const bool tile = CLUSTER;                   // full-K form
                float t_bias[2] = {0.f, 0.f};                // full-K form: the biases of features t_feat(0), t_feat(2)
                if (tile && !helper) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (t_feat(2 * h) < ly.out) t_bias[h] = __ldg(p.W + ly.w_off + (int64_t)t_feat(2 * h) * ly.ldw + ly.in);
                }
                // layer 1 reads X from its ring slots (TMA), or - folded pipeline input - from abuf 1 (staged above)
                const bool x_glob = FOLD && (l == 1) && p.x_from_global;
                if (tile && l == 1 && p.ksplit > 1) run_gemm_ksplit(nkb_f, idle(ly.out));
                else if (tile) run_gemm_tiles(nkb_f, false, l == 1, abuf0 + buf * abuf_bytes, idle(ly.out));
                else run_gemm(nkb_f, false, l == 1 && !x_glob, abuf0 + (x_glob ? 1 : buf) * abuf_bytes, idle(ly.out));
                if (helper) break;                           // its phase sums are in the owner: the helper is done
                if (l > 1) buf ^= 1;                         // layer l read buf, wrote buf^1
                else buf = 0;                                // layer 1 writes abuf 0
                if (p.sync_debug) asm volatile("bar.sync 2, 256;" ::: "memory");   // racecheck aid, see kernels.h
                const uint32_t dst = abuf0 + wbuf * abuf_bytes;
                const uint32_t src = abuf0 + (wbuf ^ 1) * abuf_bytes;   // RES, l >= 2: the tile this layer consumed
                const bool res_l = is_res(l);
                float* __restrict__ gout = p.act[l] + (int64_t)row0 * p.act_ld[l];
                float* __restrict__ ggout = nullptr;         // GATE: where this layer's gates go (none: inference)
                if constexpr (GATE) { if (ly.relu && p.gate[l] != nullptr) ggout = p.gate[l] + (int64_t)row0 * p.act_ld[l]; }
                if (!is_logits && tile) {
                    // full-K form: bias, ReLU and the feature mask on this warp's fragments, 4 st.shared per tile into
                    // the operand tile, this warp's block of it to the peers, then the global copy
                    float tgam[NTW / 2][4];                  // GATE: the gates of this warp's fragments
#pragma unroll
                    for (int j = 0; j < NTW / 2; ++j) {
                        if (j < tnt) {
#pragma unroll
                            for (int r = 0; r < 4; ++r) {
                                float x = tacc[0][j][r] + t_bias[r >> 1];
                                if constexpr (GATE) {
                                    tgam[j][r] = 0.f;
                                    if (ly.relu) x = gate_fwd(x, l, t_feat(r), t_row(j, r), tgam[j][r]);
                                } else {
                                    if (ly.relu) x = relu_f(x);
                                    if constexpr (DROP) { if (ly.relu) x = drop_fwd(x, l, t_feat(r), t_row(j, r)); }
                                }
                                if constexpr (RES) { if (res_l && t_feat(r) < ly.out) x += skip_in(l, src, t_row(j, r), t_feat(r)); }
                                x = t_feat(r) < ly.out ? x : 0.f;
                                tacc[0][j][r] = x;
                                st_tile(dst, t_row(j, r), t_feat(r), x);
                            }
                        }
                    }
                    if (l < L) hand_over(wbuf, true, t_n0, 8 * tnt, t_m0 / 4, 2);
                    else publish();
#pragma unroll
                    for (int j = 0; j < NTW / 2; ++j)
#pragma unroll
                        for (int r = 0; r < 4; ++r)
                            if (j < tnt && t_feat(r) < ly.out && t_row(j, r) < p.mb_rows)
                                gout[(int64_t)t_row(j, r) * p.act_ld[l] + t_feat(r)] = tacc[0][j][r];
                    if constexpr (GATE) {
                        if (ggout != nullptr) {
#pragma unroll
                            for (int j = 0; j < NTW / 2; ++j)
#pragma unroll
                                for (int r = 0; r < 4; ++r)
                                    if (j < tnt && t_feat(r) < ly.out && t_row(j, r) < p.mb_rows)
                                        ggout[(int64_t)t_row(j, r) * p.act_ld[l] + t_feat(r)] = tgam[j][r];
                        }
                    }
                    wbuf ^= 1;
                    if (l == 1) wbuf = 1;                    // layer 1 wrote abuf 0; layer 2 reads 0, writes 1
                } else if (!is_logits) {
                    // one 16-row chunk per warp when N <= 32: write the operand tile for the next GEMM first,
                    // publish it, and only then drain the global copy (needed later by wgrad / the pipeline)
                    const bool single = (c_hi - c_lo == 16);
                    float keep[16], gkeep[16];               // gkeep: GATE, the gates of `keep`
#pragma unroll
                    for (int ch = 0; ch < NTW / 2 && epi; ++ch) {
                        const int c = c_lo + 16 * ch;
                        if (c >= c_hi) break;
                        float v[16];
                        warp_acc_row16(acc, ch, v, lane);
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            float x = v[j] + bias;
                            float gm = 0.f;
                            if constexpr (GATE) {
                                if (ly.relu) x = gate_fwd(x, l, m, c + j, gm);
                            } else {
                                if (ly.relu) x = relu_f(x);
                                if constexpr (DROP) { if (ly.relu) x = drop_fwd(x, l, m, c + j); }
                            }
                            if constexpr (RES) { if (res_l && m_ok) x += skip_in(l, src, c + j, m); }
                            x = m_ok ? x : 0.f;
                            const int n = c + j;
                            st_tile(dst, n, m, x);
                            if (single) {
                                keep[j] = x;
                                if constexpr (GATE) gkeep[j] = gm;
                            } else if (m_ok && n < p.mb_rows) {
                                gout[(int64_t)n * p.act_ld[l] + m] = x;
                                if constexpr (GATE) { if (ggout != nullptr) ggout[(int64_t)n * p.act_ld[l] + m] = gm; }
                                if constexpr (FOLD) { if (l == L && p.out_peer != nullptr) p.out_peer[(int64_t)n * p.act_ld[l] + m] = x; }
                            }
                        }
                    }
                    if (l < L) hand_over(wbuf, epi, c_lo, c_hi - c_lo, 0, 3);
                    else publish();
                    if (epi && single && m_ok) {
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (c_lo + j < p.mb_rows) {
                                gout[(int64_t)(c_lo + j) * p.act_ld[l] + m] = keep[j];
                                if constexpr (GATE) { if (ggout != nullptr) ggout[(int64_t)(c_lo + j) * p.act_ld[l] + m] = gkeep[j]; }
                                if constexpr (FOLD) { if (l == L && p.out_peer != nullptr) p.out_peer[(int64_t)(c_lo + j) * p.act_ld[l] + m] = keep[j]; }
                            }
                    }
                    wbuf ^= 1;
                    if (l == 1) wbuf = 1;                    // layer 1 wrote abuf 0; layer 2 reads 0, writes 1
                } else {
                    // ---------------- loss head on the logits tile (class = feature lane, row = column)
                    // MSE: softmax contract of the reference: shift by the GLOBAL max of the micro-batch, +1e-7.
                    // Cross-entropy: per-row softmax (ptx.cuh: ce_*), so no cross-lane max at all.
                    // Step 1: the class-lane warps (q == 0, both halves) transpose logits (+bias) into a [row][class]
                    // scratch in smem.  Step 2: each lane of warp (0, 0) owns ROWS, loops over the <= 32 classes in
                    // registers - no cross-lane reductions except (MSE) one max and one sum for the whole micro-batch.
                    // CLUSTER: the <= 32 classes are rank 0's features, and every warp transposes its own tiles.
                    const int C = ly.out;
                    float* scratch = reinterpret_cast<float*>(smem_gen + scratch_off);   // [N][kScratchLd]
                    float loss = 0.f;
                    if (tile) {
#pragma unroll
                        for (int j = 0; j < NTW / 2; ++j)
#pragma unroll
                            for (int r = 0; r < 4; ++r)
                                if (j < tnt && t_feat(r) < C) scratch[t_row(j, r) * kScratchLd + t_feat(r)] = tacc[0][j][r] + t_bias[r >> 1];
                    } else if (q == 0) {
#pragma unroll
                        for (int ch = 0; ch < NTW / 2; ++ch) {
                            const int c = c_lo + 16 * ch;
                            if (c >= c_hi) break;
                            float v[16];
                            warp_acc_row16(acc, ch, v, lane);
                            if (m < C)
#pragma unroll
                                for (int j = 0; j < 16; ++j) scratch[(c + j) * kScratchLd + m] = v[j] + bias;
                        }
                    }
                    asm volatile("bar.sync 2, 256;" ::: "memory");
                    if (q == 0 && half == 0 && rank == 0) {
                        constexpr bool ce = CE;
                        float gmax = -3.0e38f;
                        if (!ce) {
                            for (int n = lane; n < p.mb_rows; n += 32)
                                for (int k = 0; k < C; ++k) gmax = max_nan(gmax, scratch[n * kScratchLd + k]);
                            gmax = warp_max_f(gmax);
                        }
                        for (int n = lane; n < N; n += 32) {
                            const bool row_ok = n < p.mb_rows;
                            const float* __restrict__ tg = p.target + (int64_t)(row0 + n) * p.ldt;
                            const float* __restrict__ zr = scratch + n * kScratchLd;
                            if (ce && C <= 16) {
                                // cross-entropy fast path: the row max, sum(exp) and sum(t) in registers, constant bounds
                                float tgv[16], ev[16];
                                float mx = -3.0e38f;
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    tgv[k] = (k < C && row_ok) ? __ldg(tg + k) : 0.f;
                                    if (k < C) mx = fmaxf(mx, zr[k]);
                                }
                                float ssum = 0.f, tsum = 0.f;
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    ev[k] = (k < C) ? ce_exp(zr[k], mx) : 0.f;
                                    ssum += ev[k];
                                    tsum += tgv[k];
                                }
                                const float log_s = logf(ssum);
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    if (k < C) {
                                        const float pr = ce_prob(ev[k], ssum);
                                        const float dzv = row_ok ? ce_dlogit(pr, tsum, tgv[k], p.inv_batch) : 0.f;
                                        if (row_ok) {
                                            loss += ce_loss_term(tgv[k], zr[k], mx, log_s);
                                            gout[(int64_t)n * p.act_ld[l] + k] = zr[k];
                                            p.probs[(int64_t)(row0 + n) * p.ldp + k] = pr;
                                            if (p.dz[l] != nullptr) p.dz[l][(int64_t)(row0 + n) * p.act_ld[l] + k] = dzv;
                                        }
                                        if (p.do_bwd) st_tile(dst, n, k, dzv);
                                    }
                                }
                            } else if (ce) {
                                float mx = -3.0e38f;
                                for (int k = 0; k < C; ++k) mx = fmaxf(mx, zr[k]);
                                float ssum = 0.f, tsum = 0.f;
                                for (int k = 0; k < C; ++k) {
                                    ssum += ce_exp(zr[k], mx);
                                    tsum += row_ok ? __ldg(tg + k) : 0.f;
                                }
                                const float log_s = logf(ssum);
                                for (int k = 0; k < C; ++k) {
                                    const float pr = ce_prob(ce_exp(zr[k], mx), ssum);
                                    const float t = row_ok ? __ldg(tg + k) : 0.f;
                                    const float dzv = row_ok ? ce_dlogit(pr, tsum, t, p.inv_batch) : 0.f;
                                    if (row_ok) {
                                        loss += ce_loss_term(t, zr[k], mx, log_s);
                                        gout[(int64_t)n * p.act_ld[l] + k] = zr[k];
                                        p.probs[(int64_t)(row0 + n) * p.ldp + k] = pr;
                                        if (p.dz[l] != nullptr) p.dz[l][(int64_t)(row0 + n) * p.act_ld[l] + k] = dzv;
                                    }
                                    if (p.do_bwd) st_tile(dst, n, k, dzv);
                                }
                            } else if (C <= 16) {
                                // fast path (the usual 10-class head): everything in registers, loops fully
                                // unrolled to a constant bound so the 16 target loads / exps are independent
                                float tgv[16], ev[16];
                                float ssum = 0.f;
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    tgv[k] = (k < C && row_ok) ? __ldg(tg + k) : 0.f;
                                    ev[k] = (k < C) ? expf(zr[k] - gmax) : 0.f;
                                    ssum += ev[k];
                                }
                                const float inv = 1.f / (ssum + 1e-7f);
                                float gs = 0.f;
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    const float pr = ev[k] * inv;
                                    const float d = tgv[k] - pr;
                                    if (k < C && row_ok) loss += d * d;
                                    const float g = pr * (-2.f * d * p.inv_batch);
                                    gs += (k < C) ? g : 0.f;
                                    ev[k] = pr;
                                    tgv[k] = g;
                                }
#pragma unroll
                                for (int k = 0; k < 16; ++k) {
                                    if (k < C) {
                                        const float dzv = row_ok ? (tgv[k] - ev[k] * gs) : 0.f;
                                        if (row_ok) {
                                            gout[(int64_t)n * p.act_ld[l] + k] = zr[k];
                                            p.probs[(int64_t)(row0 + n) * p.ldp + k] = ev[k];
                                            if (p.dz[l] != nullptr) p.dz[l][(int64_t)(row0 + n) * p.act_ld[l] + k] = dzv;
                                        }
                                        if (p.do_bwd) st_tile(dst, n, k, dzv);
                                    }
                                }
                            } else {
                                float ssum = 0.f;
                                for (int k = 0; k < C; ++k) ssum += expf(zr[k] - gmax);
                                const float inv = 1.f / (ssum + 1e-7f);
                                float gs = 0.f;
                                for (int k = 0; k < C; ++k) {
                                    const float pr = expf(zr[k] - gmax) * inv;
                                    const float d = (row_ok ? __ldg(tg + k) : pr) - pr;
                                    if (row_ok) loss += d * d;
                                    gs += pr * (-2.f * d * p.inv_batch);
                                }
                                for (int k = 0; k < C; ++k) {
                                    const float pr = expf(zr[k] - gmax) * inv;
                                    const float d = (row_ok ? __ldg(tg + k) : pr) - pr;
                                    const float dzv = row_ok ? (pr * (-2.f * d * p.inv_batch) - pr * gs) : 0.f;
                                    if (row_ok) {
                                        gout[(int64_t)n * p.act_ld[l] + k] = zr[k];
                                        p.probs[(int64_t)(row0 + n) * p.ldp + k] = pr;
                                        if (p.dz[l] != nullptr) p.dz[l][(int64_t)(row0 + n) * p.act_ld[l] + k] = dzv;
                                    }
                                    if (p.do_bwd) st_tile(dst, n, k, dzv);
                                }
                            }
                            if (p.do_bwd)                               // features [C, 32) of the k-block must be finite zeros
                                for (int k = C; k < 32; ++k) st_tile(dst, n, k, 0.f);
                        }
                        loss = warp_sum_f(loss);
                        if (lane == 0 && p.loss != nullptr) p.loss[p.mu_base + mb] = loss * p.inv_batch;
                    }
                    if (p.do_bwd) {
                        if (L >= bwd_lo) hand_over(wbuf, q == 0 && half == 0, 0, N, 0, 3);   // the head's warp: all N rows
                        else publish();
                        wbuf ^= 1;
                    }
                    signal_ready(l);                          // dz[L] written by the class-lane warp; the others arrive empty
                }
            }
        }
        if (FOLD && p.do_fwd && !p.do_bwd && p.out_peer != nullptr) {
            // the stage's output tile is in the next stage's receive slot: one fence, then its arrival flag
            asm volatile("bar.sync 2, 256;" ::: "memory");
            if (threadIdx.x == 32) {
                __threadfence_system();
                st_relaxed_sys(p.out_flag, pp_epoch);
            }
        }
        if (p.do_bwd && !(p.do_fwd && p.do_loss) && !helper) {
            // backward-only launch (pipeline stage): stage dZ_L = gout (.) relu'(act_L) into smem (GATE: gout (.) gate_L)
            const ChainLayer& ly = p.layers[L - 1];
            const bool m_ok = m < ly.out;
            const uint32_t dst = abuf0 + wbuf * abuf_bytes;
            float* __restrict__ g = p.dz[L] + (int64_t)row0 * p.act_ld[L];
            const float* __restrict__ y = (GATE ? p.gate[L] : p.act[L]) + (int64_t)row0 * p.act_ld[L];
            // RES, residual layer L: the received gradient is in gout (kept: the dgrad of layer L adds it), dz[L] is its own
            const float* __restrict__ gin = (RES && p.gout != nullptr) ? p.gout + (int64_t)row0 * p.act_ld[L] : g;
            for (int n = c_lo; n < c_hi && epi; ++n) {
                float x = 0.f;
                if (m_ok && n < p.mb_rows) {
                    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(x) : "l"(gin + (int64_t)n * p.act_ld[L] + m));   // may be peer-written
                    if constexpr (GATE) {
                        if (ly.relu) x *= y[(int64_t)n * p.act_ld[L] + m];   // the gate holds keep * s already
                    } else {
                        if (ly.relu && !(y[(int64_t)n * p.act_ld[L] + m] > 0.f)) x = 0.f;
                        if constexpr (DROP) { if (ly.relu) x *= p.drop.scale; }   // act_L was dropped: dZ_L = g * s where it passes
                    }
                    g[(int64_t)n * p.act_ld[L] + m] = x;     // the wgrad GEMM reads the masked gradient
                }
                st_tile(dst, n, m, x);
            }
            if (L >= bwd_lo) hand_over(wbuf, epi, c_lo, c_hi - c_lo, 0, 3);
            else publish();
            wbuf ^= 1;
        }
        if (p.do_bwd && !helper) {
            // RES: g_l of this warp's fragments, the pre-gate output of the previous dgrad (cluster: t_g; one CTA: r_g per
            // 16-row chunk), carried into the dgrad of layer l when layer l is residual
            float t_g[NTW / 2][4], r_g[NTW / 2][16];
            if constexpr (RES) {
#pragma unroll
                for (int j = 0; j < NTW / 2; ++j) {
#pragma unroll
                    for (int r = 0; r < 4; ++r) t_g[j][r] = 0.f;
#pragma unroll
                    for (int r = 0; r < 16; ++r) r_g[j][r] = 0.f;
                }
            }
            // the loss head / boundary loader wrote dZ_L into the buffer after the last forward output
            for (int l = L; l >= bwd_lo; --l) {
                const ChainLayer& ly = p.layers[l - 1];
                const bool m_ok = m < ly.in;                 // output feature of dgrad = input feature of layer l
                const bool mask_on = (l >= 2) && p.layers[l - 2].relu;
                const bool res_l = is_res(l), res_prev = is_res(l - 1);   // RES: add g_l / keep g_{l-1}
                const bool g_from_gout = RES && res_l && l == L && p.gout != nullptr;   // g_L: the received gradient
                // the mask of layer l - 1: its stored output (ReLU), or its gate (GATE: multiplied in, 1 where no mask)
                const float* __restrict__ yprev = (GATE ? p.gate[l - 1] : p.act[l - 1]) + (int64_t)row0 * p.act_ld[l - 1];
                float* __restrict__ gprev = p.dz[l - 1] + (int64_t)row0 * p.act_ld[l - 1];
                if constexpr (CLUSTER) {
                    // full-K form (K = out <= 128: at most 4 k-blocks): the ReLU masks of this warp's fragments are
                    // fetched before the MMAs, the epilogue runs on the fragments
                    float t_mk[NTW / 2][4];
#pragma unroll
                    for (int j = 0; j < NTW / 2; ++j)
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const int n = t_row(j, r), f = t_feat(r);
                            t_mk[j][r] = (j < tnt && mask_on && f < ly.in && n < p.mb_rows) ? yprev[(int64_t)n * p.act_ld[l - 1] + f] : 1.f;
                            if constexpr (RES) { if (g_from_gout) t_g[j][r] = (j < tnt && f < ly.in) ? g_recv(n, f) : 0.f; }
                        }
                    run_gemm_tiles((ly.out + (int)kBlockK - 1) / (int)kBlockK, true, false, abuf0 + buf * abuf_bytes, idle(ly.in));
                    buf ^= 1;
                    if (p.sync_debug) asm volatile("bar.sync 2, 256;" ::: "memory");   // racecheck aid, see kernels.h
                    const uint32_t dst = abuf0 + wbuf * abuf_bytes;
                    const bool more = (l > bwd_lo);          // another dgrad consumes this tile
#pragma unroll
                    for (int j = 0; j < NTW / 2; ++j) {
                        if (j < tnt) {
#pragma unroll
                            for (int r = 0; r < 4; ++r) {
                                float x;
                                if constexpr (RES) {
                                    float pre = tacc[0][j][r];
                                    if (res_l) pre += t_g[j][r];
                                    if (res_prev) t_g[j][r] = pre;
                                    x = pre * t_mk[j][r];
                                } else if constexpr (GATE) {
                                    x = tacc[0][j][r] * t_mk[j][r];
                                } else {
                                    x = (t_mk[j][r] > 0.f) ? tacc[0][j][r] : 0.f;
                                    if constexpr (DROP) { if (mask_on) x *= p.drop.scale; }   // layer l - 1 was dropped
                                }
                                x = t_feat(r) < ly.in ? x : 0.f;
                                tacc[0][j][r] = x;
                                if (more) st_tile(dst, t_row(j, r), t_feat(r), x);
                            }
                        }
                    }
                    if (more) {
                        hand_over(wbuf, true, t_n0, 8 * tnt, t_m0 / 4, 2);
                        wbuf ^= 1;
                    }
#pragma unroll
                    for (int j = 0; j < NTW / 2; ++j)
#pragma unroll
                        for (int r = 0; r < 4; ++r)
                            if (j < tnt && t_feat(r) < ly.in && t_row(j, r) < p.mb_rows)
                                gprev[(int64_t)t_row(j, r) * p.act_ld[l - 1] + t_feat(r)] = tacc[0][j][r];
                    signal_ready(l - 1);
                    continue;
                }
                // the masks do not depend on the MMA: fetch them before it runs (N <= 32: all of them)
                float mk0[16];
                const bool pre = (c_hi - c_lo == 16);        // N <= 32: one chunk per warp, prefetch its masks
                if (pre && epi) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        mk0[j] = (mask_on && m_ok && c_lo + j < p.mb_rows) ? yprev[(int64_t)(c_lo + j) * p.act_ld[l - 1] + m] : 1.f;
                }
                const int nkb = (ly.out + (int)kBlockK - 1) / (int)kBlockK;
                run_gemm(nkb, true, false, abuf0 + buf * abuf_bytes, idle(ly.in));
                buf ^= 1;
                if (p.sync_debug) asm volatile("bar.sync 2, 256;" ::: "memory");   // racecheck aid, see kernels.h
                const uint32_t dst = abuf0 + wbuf * abuf_bytes;
                const bool more = (l > bwd_lo);              // another dgrad consumes this tile
                const bool single = (c_hi - c_lo == 16);
                float keep[16];
#pragma unroll
                for (int ch = 0; ch < NTW / 2 && epi; ++ch) {
                    const int c = c_lo + 16 * ch;
                    if (c >= c_hi) break;
                    float v[16];
                    warp_acc_row16(acc, ch, v, lane);
                    float mk[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int n = c + j;
                        if (pre) mk[j] = mk0[j];
                        else mk[j] = (mask_on && m_ok && n < p.mb_rows) ? yprev[(int64_t)n * p.act_ld[l - 1] + m] : 1.f;
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int n = c + j;
                        float x;
                        if constexpr (RES) {
                            float pre = v[j];
                            if (res_l) pre += g_from_gout ? (m_ok ? g_recv(n, m) : 0.f) : r_g[ch][j];
                            if (res_prev) r_g[ch][j] = pre;
                            x = pre * mk[j];
                        } else if constexpr (GATE) {
                            x = v[j] * mk[j];
                        } else {
                            x = (mk[j] > 0.f) ? v[j] : 0.f;
                            if constexpr (DROP) { if (mask_on) x *= p.drop.scale; }   // layer l - 1 was dropped
                        }
                        x = m_ok ? x : 0.f;
                        if (more) st_tile(dst, n, m, x);
                        if (single) keep[j] = x;
                        else if (m_ok && n < p.mb_rows) {
                            gprev[(int64_t)n * p.act_ld[l - 1] + m] = x;
                            if constexpr (FOLD) { if (l == 1 && p.out_peer != nullptr) p.out_peer[(int64_t)n * p.act_ld[0] + m] = x; }
                        }
                    }
                }
                if (more) {
                    hand_over(wbuf, epi, c_lo, c_hi - c_lo, 0, 3);
                    wbuf ^= 1;
                }
                if (epi && single && m_ok) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (c_lo + j < p.mb_rows) {
                            gprev[(int64_t)(c_lo + j) * p.act_ld[l - 1] + m] = keep[j];
                            if constexpr (FOLD) { if (l == 1 && p.out_peer != nullptr) p.out_peer[(int64_t)(c_lo + j) * p.act_ld[0] + m] = keep[j]; }
                        }
                }
                signal_ready(l - 1);
            }
            if (FOLD && p.out_peer != nullptr && !p.first_stage) {
                // dz[0] is in the previous stage's receive slot: one fence, then its arrival flag
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (threadIdx.x == 32) {
                    __threadfence_system();
                    st_relaxed_sys(p.out_flag, pp_epoch);
                }
            }
        }
    }
    // no CTA leaves while a peer may still address its shared memory
    if constexpr (CLUSTER) cluster_sync();
}


// =========================================================================== host side: the instantiations
// Every (precision, residual) pair is instantiated in a translation unit of its own, and the build compiles them in
// parallel, so that no pair lengthens the longest compile: mlp_chain.cu PREC_3XTF32, mlp_chain_tf32.cu PREC_TF32,
// mlp_chain_bf16.cu PREC_BF16, and mlp_chain_res.cu / mlp_chain_res_tf32.cu / mlp_chain_res_bf16.cu their RES forms.

using ChainKernel = void (*)(ChainParams);
// the launch form of a plan: one CTA per micro-batch, with folded pipeline boundaries (FOLD), or a cluster (CLUSTER)
enum ChainForm : int { CHAIN_PLAIN = 0, CHAIN_FOLD = 1, CHAIN_CLUSTER = 2 };

template <int PREC, int NTW, bool CE, bool DROP, bool GATE, bool RES>
static ChainKernel chain_kernel_form(ChainForm form) {
    switch (form) {
        case CHAIN_PLAIN: return mlp_chain_kernel<PREC, false, NTW, false, CE, DROP, GATE, RES>;
        case CHAIN_FOLD: return mlp_chain_kernel<PREC, true, NTW, false, CE, DROP, GATE, RES>;
        case CHAIN_CLUSTER: return mlp_chain_kernel<PREC, false, NTW, true, CE, DROP, GATE, RES>;
    }
    return nullptr;
}

template <int PREC, int NTW, bool DROP, bool GATE, bool RES>
static ChainKernel chain_kernel_ce(ChainForm form, bool ce) {
    return ce ? chain_kernel_form<PREC, NTW, true, DROP, GATE, RES>(form) : chain_kernel_form<PREC, NTW, false, DROP, GATE, RES>(form);
}

template <int PREC, bool DROP, bool GATE, bool RES>
static ChainKernel chain_kernel_ntw(ChainForm form, int ntw, bool ce) {
    switch (ntw) {
        case 2: return chain_kernel_ce<PREC, 2, DROP, GATE, RES>(form, ce);
        case 4: return chain_kernel_ce<PREC, 4, DROP, GATE, RES>(form, ce);
        case 8: return chain_kernel_ce<PREC, 8, DROP, GATE, RES>(form, ce);
    }
    return nullptr;
}

template <int PREC, bool GATE, bool RES>
static ChainKernel chain_kernel_drop(ChainForm form, int ntw, bool ce, bool drop) {
    return drop ? chain_kernel_ntw<PREC, true, GATE, RES>(form, ntw, ce) : chain_kernel_ntw<PREC, false, GATE, RES>(form, ntw, ce);
}

// The instantiation of precision PREC, residual or not, that runs (form, ntw, ce, drop, gate); nullptr for a combination
// without one (a residual model runs gated).
template <int PREC, bool RES>
static ChainKernel chain_kernel(ChainForm form, int ntw, bool ce, bool drop, bool gate) {
    if constexpr (RES) return gate ? chain_kernel_drop<PREC, true, true>(form, ntw, ce, drop) : nullptr;
    else if (gate) return chain_kernel_drop<PREC, true, false>(form, ntw, ce, drop);
    else return chain_kernel_drop<PREC, false, false>(form, ntw, ce, drop);
}

// chain_kernel<PREC, RES> of the other translation units (the 3xTF32 one without RES is mlp_chain.cu's own)
ChainKernel chain_kernel_tf32(ChainForm form, int ntw, bool ce, bool drop, bool gate);
ChainKernel chain_kernel_bf16(ChainForm form, int ntw, bool ce, bool drop, bool gate);
ChainKernel chain_kernel_res_3xtf32(ChainForm form, int ntw, bool ce, bool drop, bool gate);
ChainKernel chain_kernel_res_tf32(ChainForm form, int ntw, bool ce, bool drop, bool gate);
ChainKernel chain_kernel_res_bf16(ChainForm form, int ntw, bool ce, bool drop, bool gate);

}  // namespace ssb
