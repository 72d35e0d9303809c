// TMA + mbarrier + tensor-core GEMM family for the Linear layer (SURVEY.md K1, K2, K3, K6, K7).
//
// One warp-specialised kernel, three instantiations (see GemmMode in kernels.h):
//   warp 0    : TMA producer  - cp.async.bulk.tensor tiles (SWIZZLE_128B) into a ring of smem stages
//   warps 1-4 : math + epilogue - each warp owns 32 rows of the 128-row tile: mma.sync TF32 (fp32 data, fp32
//                               accumulate in registers, 3xTF32 for fp32-equivalent products) straight from the
//                               swizzled stages, then fused bias / ReLU / ReLU-mask / grad-accumulate / SGD and
//                               coalesced global stores.  During the WGRAD main loop these warps also reduce
//                               db = colsum(dZ) from the staged A tiles (exact fp32, no extra pass over dZ).
//
// Operand staging (all tiles are 32 fp32 = 128 B wide, the SWIZZLE_128B span):
//   K-major  tile: one TMA box [rows x 32 k]                       -> rows 128 B apart
//   MN-major tile: panels of  [32 k-rows x 32 mn], 4096 B per panel -> k-rows 128 B apart
// Ragged edges are handled by TMA out-of-bounds zero fill, so no dimension needs padding
// beyond the 16-byte row pitch rule (the reference model's 127/126/125/123-wide layers).
#include "kernels.h"
#include "ptx.cuh"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

namespace ssb {

static constexpr int kThreads = 160;
static constexpr uint32_t kBlockM = 128;
static constexpr int kMaxBlockN = 64;                   // a math warp holds a 32 x block_n fp32 accumulator in registers
static constexpr uint32_t kBlockK = 32;                 // fp32 elements = 128 B
static constexpr uint32_t kABytes = kBlockM * 128;      // 16 KB per stage
static constexpr uint32_t kPanelBytes = 32 * 128;       // MN-major panel: 32 k-rows x 128 B

// SPLITK (FWD / DGRAD only, wide layers with few output tiles): blockIdx.z owns a contiguous range of
// k-blocks; every CTA writes its raw fp32 accumulator tile to a workspace and the LAST CTA to arrive at the
// tile's counter sums the partials in split order (deterministic) and runs the fused epilogue.  Nobody
// waits for anybody, so the CTAs of a tile need not be co-resident.
// The body is shared by the one-GEMM-per-launch kernels below and by the grouped weight-gradient kernel (several
// layers' tiles in ONE launch, tensor maps and parameters read from a device table).
// STATEFUL (WGRAD with fuse_sgd only): the SGD update uses momentum / weight decay (GemmParams::V, ...); the false
// instantiations are the plain w -= lr * dW code.
template <int MODE, bool SPLITK, bool STATEFUL = false>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                                             const GemmParams& p, const int bx, const int by, const int bz) {
    constexpr bool A_MN = (MODE != GEMM_FWD);
    constexpr bool B_MN = (MODE == GEMM_WGRAD);

    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t smem_base = (raw + 1023u) & ~1023u;     // SWIZZLE_128B wants 1024 B alignment
    uint8_t* smem_gen = smem_raw + (smem_base - raw);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = bx * kBlockM;
    const int n0 = by * p.block_n;
    int num_kb = (p.k_total + kBlockK - 1) / kBlockK;
    int kb0 = 0;                                           // first k-block of this CTA
    if constexpr (SPLITK) {
        const int per = (num_kb + p.k_splits - 1) / p.k_splits;   // host guarantees every split is non-empty
        kb0 = bz * per;
        num_kb = min(per, num_kb - kb0);
    }
    const uint32_t stage_bytes = kABytes + p.block_n * 128u;    // [A][B]
    // WGRAD stages its output tile (block_n/32 swizzled panels of [128 rows x 128 B]) behind the ring
    const uint32_t epi_base = smem_base + p.stages * stage_bytes;
    const uint32_t epi_bytes = (MODE == GEMM_WGRAD) ? (uint32_t)p.block_n * 512u : 0u;
    const uint32_t bar_base = epi_base + epi_bytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
    volatile uint32_t* flag_gen = reinterpret_cast<volatile uint32_t*>(smem_gen + p.stages * stage_bytes + epi_bytes + 8u * (2 * p.stages));

    // the bias gradient is written by the CTA of the LAST column tile: its own tile store is the one that can spill into
    // the bias column (see the epilogue), so only that CTA can order the two
    const bool db_active = (MODE == GEMM_WGRAD) && (p.db != nullptr) && (by == (p.n_total - 1) / p.block_n);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (MODE == GEMM_WGRAD) tma_prefetch_desc(&tmC);
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);                   // one arrive per math warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 0) {
        // ------------------------------------------------------------ TMA producer
        // converged warp; one elect.sync-chosen lane issues
        for (int kb = 0; kb < num_kb; ++kb) {
            const int s = kb % p.stages;
            const uint32_t ph = (kb / p.stages) & 1;
            mbar_wait(empty_bar(s), ph ^ 1);
            if (elect_one()) {
                mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                const uint32_t a_dst = smem_base + s * stage_bytes;
                const uint32_t b_dst = a_dst + kABytes;
                const int k0 = (kb0 + kb) * kBlockK;
                if (!A_MN) {
                    tma_load_2d(a_dst, &tmA, full_bar(s), k0, m0);
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) tma_load_2d(a_dst + i * kPanelBytes, &tmA, full_bar(s), m0 + 32 * i, k0);
                }
                if (!B_MN) {
                    tma_load_2d(b_dst, &tmB, full_bar(s), k0, n0);
                } else {
                    for (int j = 0; j < p.block_n / 32; ++j)
                        tma_load_2d(b_dst + j * kPanelBytes, &tmB, full_bar(s), n0 + 32 * j, k0);
                }
            }
            __syncwarp();
        }
    } else {
        // ------------------------------------------------------------ math + epilogue warps
        // warp w owns the 32 output rows q*32 .. q*32+31 of the tile (all block_n columns): tensor-core MMAs from the
        // staged tiles into registers, then one row per lane (warp_acc_row16) for the fused epilogue.
        const int q = warp & 3;
        const int m_local = q * 32 + lane;
        const int m = m0 + m_local;
        const bool m_ok = m < p.m_total;
        const int nt = p.block_n / 8;
        constexpr int kChunks = kMaxBlockN / 16;

        float acc[2][kMaxBlockN / 8][4];
        warp_acc_zero(acc);
        float dbsum = 0.f;
        // the fused update's learning rate, loaded before the main loop so that its latency hides under the GEMM.  The
        // STATEFUL epilogue loads it next to its momentum / weight loads instead: one more register live through the
        // loop would take that instantiation past 200 registers (two CTAs per SM).
        const float lr_pre = (MODE == GEMM_WGRAD && !STATEFUL && p.fuse_sgd) ? *p.lr : 0.f;
        for (int kb = 0; kb < num_kb; ++kb) {
            const int s = kb % p.stages;
            const uint32_t ph = (kb / p.stages) & 1;
            mbar_wait(full_bar(s), ph);
            const uint32_t a_src = smem_base + s * stage_bytes;
            if (p.split)
                warp_mma_kblock<kMaxBlockN / 8, A_MN, B_MN, true>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, nt, lane);
            else
                warp_mma_kblock<kMaxBlockN / 8, A_MN, B_MN, false>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, nt, lane);
            if (MODE == GEMM_WGRAD && db_active) {
                // db[m] = sum over micro-batch rows of dZ[row, m], read from the staged A panels (exact fp32)
#pragma unroll 8
                for (int r = 0; r < 32; ++r) dbsum += lds_f32(a_src + operand_off<true>((uint32_t)m_local, (uint32_t)r));
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));
        }

        if constexpr (SPLITK) {
            // ---- split-K: publish the raw partial, last arriver reduces (fixed split order) + epilogue
            const int tile = (int)(by * gridDim.x + bx);
            const size_t tile_floats = (size_t)p.block_n * kBlockM;
            float* ws = p.partial + ((size_t)tile * p.k_splits + bz) * tile_floats;
#pragma unroll
            for (int ch = 0; ch < kChunks; ++ch) {
                if (16 * ch >= p.block_n) break;
                float v[16];
                warp_acc_row16(acc, ch, v, lane);
#pragma unroll
                for (int j = 0; j < 16; ++j) __stcg(ws + (size_t)(16 * ch + j) * kBlockM + m_local, v[j]);   // lanes -> consecutive floats
            }
            __threadfence();
            asm volatile("bar.sync 1, 128;" ::: "memory");
            volatile uint32_t* last_flag = flag_gen;
            if (warp == 1 && lane == 0) {
                const unsigned old = atomicAdd(p.tile_counter + tile, 1u);
                const bool last = (old == (unsigned)p.k_splits - 1u);
                if (last) p.tile_counter[tile] = 0u;          // re-arm for the next launch (graph replay)
                *last_flag = last ? 1u : 0u;
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (*last_flag != 0u) {
                __threadfence();
                const float* wt = p.partial + (size_t)tile * p.k_splits * tile_floats;
                float bias = 0.f;
                if (MODE == GEMM_FWD && p.bias != nullptr && m_ok) bias = __ldg(p.bias + (size_t)m * p.bias_stride);
                const float* __restrict__ mask = p.mask;
                float* __restrict__ out = p.out;
                for (int c = 0; c < p.block_n; c += 16) {
                    float mk[16];
                    if (MODE == GEMM_DGRAD && mask != nullptr && m_ok) {
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int n = n0 + c + j;
                            mk[j] = (n < p.n_total) ? __ldg(mask + (size_t)n * p.ldmask + m) : 0.f;
                        }
                    }
                    float v[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = 0.f;
                    for (int sp = 0; sp < p.k_splits; ++sp) {
                        const float* src = wt + (size_t)sp * tile_floats + (size_t)c * kBlockM + m_local;
#pragma unroll
                        for (int j = 0; j < 16; ++j) v[j] += __ldcg(src + (size_t)j * kBlockM);
                    }
                    if (!m_ok) continue;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        float x = v[j] + bias;
                        if (MODE == GEMM_FWD) {
                            if (p.relu) x = fmaxf(x, 0.f);
                        } else if (mask != nullptr) {
                            x = (mk[j] > 0.f) ? x : 0.f;
                        }
                        const int n = n0 + c + j;
                        if (n < p.n_total) out[(size_t)n * p.ldo + m] = x;
                    }
                }
            }
        } else if (MODE == GEMM_FWD || MODE == GEMM_DGRAD) {
            float bias = 0.f;
            if (MODE == GEMM_FWD && p.bias != nullptr && m_ok) bias = __ldg(p.bias + (size_t)m * p.bias_stride);
            const float* __restrict__ mask = p.mask;
            float* __restrict__ out = p.out;
#pragma unroll
            for (int ch = 0; ch < kChunks; ++ch) {
                const int c = 16 * ch;
                if (c >= p.block_n) break;
                float mk[16];
                if (MODE == GEMM_DGRAD && mask != nullptr && m_ok) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) {       // all 16 loads in flight before any use
                        const int n = n0 + c + j;
                        mk[j] = (n < p.n_total) ? __ldg(mask + (size_t)n * p.ldmask + m) : 0.f;
                    }
                }
                float v[16];
                warp_acc_row16(acc, ch, v, lane);
                if (!m_ok) continue;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    float x = v[j] + bias;
                    if (MODE == GEMM_FWD) {
                        if (p.relu) x = fmaxf(x, 0.f);
                    } else if (mask != nullptr) {
                        x = (mk[j] > 0.f) ? x : 0.f;
                    }
                    v[j] = x;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int n = n0 + c + j;
                    if (n < p.n_total) out[(size_t)n * p.ldo + m] = v[j];     // lanes -> consecutive m: coalesced
                }
            }
        } else {
            // WGRAD: registers -> swizzled smem panels -> ONE TMA store (overwrite) or TMA reduce-add (accumulate,
            // performed in L2) per 32-column panel.  With fuse_sgd the tile is scaled by -lr and reduce-added straight into
            // W: dW never touches memory, zero_grad and the optimizer pass disappear.  OOB rows/columns are clipped by the
            // tensor map, so the bias column (index n_total of the same [out, ld] block) is never touched here.
            // STATEFUL (fuse_sgd with momentum / weight decay): the tile holds the final dW, so each lane turns its row's
            // 16 values into the step direction d (sgd_direction) - reading and writing its V entries, and reading W
            // only with weight decay - before the same -lr scaling and reduce-add.  Columns >= n_total get d = 0 and
            // are never stored: column n_total is the bias slot, which the bias path below updates.
            const float lr = STATEFUL ? *p.lr : lr_pre;            // STATEFUL implies fuse_sgd
            const float scale = p.fuse_sgd ? -lr : 1.f;
#pragma unroll
            for (int ch = 0; ch < kChunks; ++ch) {
                if (16 * ch >= p.block_n) break;
                float v[16];
                warp_acc_row16(acc, ch, v, lane);
                if constexpr (STATEFUL) {
                    const int nc = n0 + 16 * ch;
                    const bool has_v = p.V != nullptr, has_wd = p.weight_decay != 0.f;
                    float vm[16], wv[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) { vm[j] = 0.f; wv[j] = 0.f; }
                    // all loads in flight before any use; 16-byte accesses where all 4 columns are real (V and W rows
                    // are 16-byte aligned: TMA-legal pitch, nc a multiple of 16)
                    if (m_ok) {
                        const size_t row = (size_t)m * p.ldw + nc;
#pragma unroll
                        for (int q4 = 0; q4 < 4; ++q4) {
                            if (nc + 4 * q4 + 3 < p.n_total) {
                                if (has_v) {
                                    const float4 t = *reinterpret_cast<const float4*>(p.V + row + 4 * q4);
                                    vm[4 * q4] = t.x; vm[4 * q4 + 1] = t.y; vm[4 * q4 + 2] = t.z; vm[4 * q4 + 3] = t.w;
                                }
                                if (has_wd) {
                                    const float4 t = *reinterpret_cast<const float4*>(p.W + row + 4 * q4);
                                    wv[4 * q4] = t.x; wv[4 * q4 + 1] = t.y; wv[4 * q4 + 2] = t.z; wv[4 * q4 + 3] = t.w;
                                }
                            } else {
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const int j = 4 * q4 + e;
                                    if (nc + j < p.n_total) {
                                        if (has_v) vm[j] = p.V[row + j];
                                        if (has_wd) wv[j] = p.W[row + j];
                                    }
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const bool ok = m_ok && nc + j < p.n_total;
                        const float d = sgd_direction<false>(v[j], wv[j], vm[j], p.momentum, p.weight_decay, p.nesterov != 0);
                        v[j] = ok ? d : 0.f;
                    }
                    if (m_ok && has_v) {
                        const size_t row = (size_t)m * p.ldw + nc;
#pragma unroll
                        for (int q4 = 0; q4 < 4; ++q4) {
                            if (nc + 4 * q4 + 3 < p.n_total) {
                                *reinterpret_cast<float4*>(p.V + row + 4 * q4) =
                                    make_float4(vm[4 * q4], vm[4 * q4 + 1], vm[4 * q4 + 2], vm[4 * q4 + 3]);
                            } else {
#pragma unroll
                                for (int e = 0; e < 4; ++e)
                                    if (nc + 4 * q4 + e < p.n_total) p.V[row + 4 * q4 + e] = vm[4 * q4 + e];
                            }
                        }
                    }
                }
                const uint32_t prow = epi_base + (ch >> 1) * (kBlockM * 128u) + (uint32_t)m_local * 128u;
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) {
                    const uint32_t chunk = (uint32_t)((ch & 1) * 4 + q4) ^ ((uint32_t)m_local & 7u);
                    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(prow + (chunk << 4)),
                                 "f"(v[4 * q4] * scale), "f"(v[4 * q4 + 1] * scale), "f"(v[4 * q4 + 2] * scale),
                                 "f"(v[4 * q4 + 3] * scale)
                                 : "memory");
                }
            }
            fence_proxy_async_smem();
            asm volatile("bar.sync 1, 128;" ::: "memory");           // the 4 math warps only
            if (warp == 1 && lane == 0) {
                const bool add = p.accumulate || p.fuse_sgd;
                for (int pj = 0; pj < p.block_n / 32; ++pj) {
                    if (n0 + pj * 32 >= p.n_total) break;
                    const uint32_t src = epi_base + pj * (kBlockM * 128u);
                    if (add) tma_reduce_add_2d(&tmC, src, n0 + pj * 32, m0);
                    else tma_store_2d(&tmC, src, n0 + pj * 32, m0);
                }
                tma_store_commit();
                tma_store_wait_all();
            }
            // TMA stores clip the inner dimension at 16-byte granularity (with in % 4 != 0 the partially valid last
            // chunk may be written in full), i.e. the bias slot in column `in` may just have been overwritten with the
            // (zero) accumulator of an OOB column.  The bias gradient is therefore written strictly AFTER the tile
            // store retired, by this CTA only when it owns the last column tile: a CTA of another column tile could not
            // order its write against that store, and a plain (non-accumulating) store there would erase it.
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (db_active && m_ok) {
                if (p.fuse_sgd) {
                    const size_t boff = (size_t)m * p.ldw + (p.db - p.G);  // bias lives at the same offset in W (and V)
                    float* bp = p.W + boff;
                    if constexpr (STATEFUL) {
                        float vb = p.V != nullptr ? p.V[boff] : 0.f;
                        const float d = sgd_direction<false>(dbsum, *bp, vb, p.momentum, p.weight_decay, p.nesterov != 0);
                        if (p.V != nullptr) p.V[boff] = vb;
                        *bp -= lr * d;
                    } else {
                        *bp -= lr * dbsum;
                    }
                } else {
                    float* dbp = p.db + (size_t)m * p.db_stride;
                    *dbp = p.accumulate ? (*dbp + dbsum) : dbsum;
                }
            }
        }
    }
}

template <int MODE, bool SPLITK = false, bool STATEFUL = false>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
    tc_gemm_body<MODE, SPLITK, STATEFUL>(tmA, tmB, tmC, p, (int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z);
}

// ---- grouped weight-gradient launch: the tiles of SEVERAL layers' WGRAD GEMMs in one grid (one table entry per CTA).
// Removes the fork / join of one graph node per layer from the end of a step: with the zero-copy loss the fp32 training
// step of a narrow stage is chain kernel -> grouped wgrad (+SGD) (or chain || LL kernel under DP).
template <bool STATEFUL = false>
__global__ void __launch_bounds__(kThreads, 1) tc_wgrad_group_kernel(const GemmGroupEntry* __restrict__ entries) {
    const GemmGroupEntry& e = entries[blockIdx.x];
    const GemmParams p = e.p;                      // private copy: the body reads these fields in every loop
    tc_gemm_body<GEMM_WGRAD, false, STATEFUL>(e.tmA, e.tmB, e.tmC, p, e.bx, e.by, 0);
}

// =========================================================================== host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    });
    return fn;
}

// 2-D fp32 row-major tensor [outer, inner] with pitch ld (floats); box = [box_outer, box_inner=32], SWIZZLE_128B.
static const char* make_tmap(CUtensorMap* map, const float* base, int inner, int outer, int ld, int box_outer) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return "cuTensorMapEncodeTiled entry point not available";
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return "TMA: base address must be 16-byte aligned";
    if (ld % 4 != 0) return "TMA: leading dimension must be a multiple of 4 floats";
    if (inner <= 0 || outer <= 0) return "TMA: empty tensor";
    if (box_outer < 1 || box_outer > 256) return "TMA: box rows must be in [1, 256]";
    cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {kBlockK, (cuuint32_t)box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled failed";
}

// MN-major operand map ([rows(K) x 32 mn] panels) for other translation units (fused_dp.cu)
const char* make_tmap_mn(CUtensorMap* map, const float* base, int inner, int outer, int ld) {
    return make_tmap(map, base, inner, outer, ld, 32);
}

const char* make_tmap_k(CUtensorMap* map, const float* base, int inner, int outer, int ld, int box_outer) {
    return make_tmap(map, base, inner, outer, ld, box_outer);
}

static int round_up_i(int x, int m) { return (x + m - 1) / m * m; }

static bool is_stateful(const GemmParams& p) { return p.fuse_sgd && (p.momentum != 0.f || p.weight_decay != 0.f); }

const char* sgd_state_check(const SgdState& s) {
    if (!(s.momentum >= 0.f && s.momentum < 1.f)) return "momentum must be in [0, 1)";
    if (!(s.weight_decay >= 0.f)) return "weight_decay must be >= 0";
    if (s.nesterov && s.momentum == 0.f) return "nesterov needs momentum > 0";
    if ((s.momentum > 0.f) != (s.V != nullptr)) return "a momentum buffer is needed exactly when momentum > 0";
    return nullptr;
}

static void finish_plan(GemmPlan* plan) {
    GemmParams& p = plan->p;
    const int num_kb = (p.k_total + (int)kBlockK - 1) / (int)kBlockK;
    const int stage_bytes = (int)kABytes + p.block_n * 128;
    const int epi_bytes = plan->mode == GEMM_WGRAD ? p.block_n * 512 : 0;
    int stages = (200 * 1024 - epi_bytes) / stage_bytes;
    if (stages > 6) stages = 6;
    if (stages > num_kb) stages = num_kb;
    if (stages < 1) stages = 1;
    p.stages = stages;
    plan->smem_bytes = stages * stage_bytes + epi_bytes + 1024 /*align slack*/ + 8 * (2 * stages) + 16;
    plan->grid = dim3((p.m_total + kBlockM - 1) / kBlockM, (p.n_total + p.block_n - 1) / p.block_n, 1);
}

const char* gemm_plan_fwd(GemmPlan* plan, const float* W, int ldw, const float* X, int ldx, float* Y, int ldy, int rows,
                          int in, int out, const float* bias, int bias_stride, int relu, bool split) {
    *plan = GemmPlan{};
    plan->mode = GEMM_FWD;
    GemmParams& p = plan->p;
    p.m_total = out; p.n_total = rows; p.k_total = in;
    p.block_n = rows >= kMaxBlockN ? kMaxBlockN : round_up_i(rows, 16);
    p.out = Y; p.ldo = ldy; p.bias = bias; p.bias_stride = bias_stride; p.relu = relu;
    if (const char* e = make_tmap(&plan->tmA, W, in, out, ldw, kBlockM)) return e;
    if (const char* e = make_tmap(&plan->tmB, X, in, rows, ldx, p.block_n)) return e;
    plan->tmC = plan->tmA;
    p.split = split ? 1 : 0;
    finish_plan(plan);
    return nullptr;
}

const char* gemm_plan_dgrad(GemmPlan* plan, const float* W, int ldw, const float* dZ, int lddz, float* dX, int lddx,
                            int rows, int in, int out, const float* mask, int ldmask, bool split) {
    *plan = GemmPlan{};
    plan->mode = GEMM_DGRAD;
    GemmParams& p = plan->p;
    p.m_total = in; p.n_total = rows; p.k_total = out;
    p.block_n = rows >= kMaxBlockN ? kMaxBlockN : round_up_i(rows, 16);
    p.out = dX; p.ldo = lddx; p.mask = mask; p.ldmask = ldmask;
    if (const char* e = make_tmap(&plan->tmA, W, in, out, ldw, 32)) return e;          // MN-major panels [32 k x 32 m]
    if (const char* e = make_tmap(&plan->tmB, dZ, out, rows, lddz, p.block_n)) return e;
    plan->tmC = plan->tmA;
    p.split = split ? 1 : 0;
    finish_plan(plan);
    return nullptr;
}

const char* gemm_plan_wgrad(GemmPlan* plan, const float* dZ, int lddz, const float* X, int ldx, float* G, int ldg,
                            int rows, int in, int out, int accumulate, float* db, int db_stride, float* W, int ldw,
                            const float* lr, int fuse_sgd, bool split, const SgdState& opt) {
    *plan = GemmPlan{};
    plan->mode = GEMM_WGRAD;
    GemmParams& p = plan->p;
    p.m_total = out; p.n_total = in; p.k_total = rows;
    p.block_n = in >= kMaxBlockN ? kMaxBlockN : round_up_i(in, 32);
    p.G = G; p.ldg = ldg; p.accumulate = accumulate; p.db = db; p.db_stride = db_stride;
    p.W = W; p.ldw = ldw; p.lr = lr; p.fuse_sgd = fuse_sgd;
    if (fuse_sgd && W == nullptr) return "fuse_sgd needs W";
    if (fuse_sgd && lr == nullptr) return "fuse_sgd needs lr (a device float)";
    if (fuse_sgd && accumulate) return "fuse_sgd cannot be combined with accumulate (reduce into G, then run the SGD pass)";
    // the fused update finds the bias at db's offset from G, taken in W (and V): only the arena layout's bias column
    // (column `in` of G's block) names a slot of W
    if (fuse_sgd && db != nullptr && db != G + in) return "fuse_sgd needs db to be G's bias column (G + in)";
    if (!opt.plain()) {
        if (!fuse_sgd) return "momentum / weight decay need fuse_sgd (the update rule runs in the epilogue)";
        if (const char* e = sgd_state_check(opt)) return e;
        p.V = opt.V; p.momentum = opt.momentum; p.weight_decay = opt.weight_decay; p.nesterov = opt.nesterov;
    }
    // output tile map: [out, in] with the block's row pitch; fused SGD targets W itself
    if (const char* e = make_tmap(&plan->tmC, fuse_sgd ? W : G, in, out, fuse_sgd ? ldw : ldg, kBlockM)) return e;
    if (const char* e = make_tmap(&plan->tmA, dZ, out, rows, lddz, 32)) return e;
    if (const char* e = make_tmap(&plan->tmB, X, in, rows, ldx, 32)) return e;
    p.split = split ? 1 : 0;
    finish_plan(plan);
    return nullptr;
}

// ---- split-K (FWD / DGRAD): more CTAs pulling on HBM when the output has fewer tiles than the chip has SMs
int gemm_splitk_choice(const GemmPlan& plan, int num_sms) {
    if (plan.mode == GEMM_WGRAD) return 1;
    const GemmParams& p = plan.p;
    const int tiles = (int)(plan.grid.x * plan.grid.y);
    const int num_kb = (p.k_total + (int)kBlockK - 1) / (int)kBlockK;
    if (tiles * 2 > num_sms || num_kb < 16) return 1;       // already enough CTAs, or K too short to matter
    int splits = (2 * num_sms) / tiles;                     // aim at two resident CTAs per SM
    if (splits > 8) splits = 8;
    while (splits > 1 && num_kb / splits < 8) --splits;     // keep >= 8 k-blocks per CTA (pipeline fill)
    if (splits < 2) return 1;
    const int per = (num_kb + splits - 1) / splits;
    return (num_kb + per - 1) / per;                        // no empty split
}

size_t gemm_splitk_workspace_floats(const GemmPlan& plan, int k_splits) {
    return (size_t)plan.grid.x * plan.grid.y * (size_t)k_splits * (size_t)plan.p.block_n * kBlockM;
}

const char* gemm_plan_enable_splitk(GemmPlan* plan, int k_splits, float* workspace, unsigned int* counters) {
    if (plan->mode == GEMM_WGRAD) return "split-K is implemented for FWD / DGRAD only";
    if (k_splits < 2) return nullptr;
    GemmParams& p = plan->p;
    const int num_kb = (p.k_total + (int)kBlockK - 1) / (int)kBlockK;
    const int per = (num_kb + k_splits - 1) / k_splits;
    if ((num_kb + per - 1) / per != k_splits) return "split-K: empty split (choose k_splits with gemm_splitk_choice)";
    if (workspace == nullptr || counters == nullptr) return "split-K needs a workspace and zeroed tile counters";
    p.k_splits = k_splits; p.partial = workspace; p.tile_counter = counters;
    // two CTAs per SM: at most ~100 KB of ring per CTA
    const int stage_bytes = (int)kABytes + p.block_n * 128;
    int stages = (100 * 1024) / stage_bytes;
    if (stages > 6) stages = 6;
    if (stages > per) stages = per;
    if (stages < 2) stages = 2;
    p.stages = stages;
    plan->smem_bytes = stages * stage_bytes + 1024 + 8 * (2 * stages) + 16;
    plan->grid.z = k_splits;
    return nullptr;
}

const char* gemm_group_plan(GemmGroupPlan* out, const GemmPlan* plans, int n_plans) {
    *out = GemmGroupPlan{};
    if (n_plans < 1) return "gemm_group_plan: no plans";
    std::vector<GemmGroupEntry> host;
    int smem = 0;
    const bool stateful = is_stateful(plans[0].p);
    for (int i = 0; i < n_plans; ++i) {
        const GemmPlan& g = plans[i];
        if (g.mode != GEMM_WGRAD) return "gemm_group_plan: only weight-gradient GEMMs can be grouped";
        if (g.p.k_splits > 1) return "gemm_group_plan: split-K plans cannot be grouped";
        if (is_stateful(g.p) != stateful) return "gemm_group_plan: plans mix the plain and the stateful SGD rule";
        if (g.smem_bytes > smem) smem = g.smem_bytes;
        for (unsigned by = 0; by < g.grid.y; ++by)
            for (unsigned bx = 0; bx < g.grid.x; ++bx) {
                GemmGroupEntry e;
                memset(&e, 0, sizeof(e));
                e.tmA = g.tmA; e.tmB = g.tmB; e.tmC = g.tmC;
                e.p = g.p; e.bx = (int)bx; e.by = (int)by;
                host.push_back(e);
            }
    }
    GemmGroupEntry* dev = nullptr;
    if (cudaMalloc(&dev, host.size() * sizeof(GemmGroupEntry)) != cudaSuccess) return "gemm_group_plan: cudaMalloc failed";
    if (cudaMemcpy(dev, host.data(), host.size() * sizeof(GemmGroupEntry), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(dev);
        return "gemm_group_plan: table upload failed";
    }
    out->entries_dev = dev; out->n = (int)host.size(); out->smem_bytes = smem; out->n_gemms = n_plans;
    out->stateful = stateful ? 1 : 0;
    return nullptr;
}

void gemm_group_free(GemmGroupPlan* plan) {
    if (plan->entries_dev) cudaFree(plan->entries_dev);
    plan->entries_dev = nullptr;
}

static std::atomic<int> g_launches{0};
int gemm_kernel_count() { return g_launches.load(); }

static constexpr int kMaxDynSmem = 220 * 1024;
static bool g_configured = false;

cudaError_t gemm_configure() {
    if (g_configured) return cudaSuccess;
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_FWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_DGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_WGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_WGRAD, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_wgrad_group_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_wgrad_group_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_FWD, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(tc_gemm_kernel<GEMM_DGRAD, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem)) != cudaSuccess) return e;
    g_configured = true;
    return cudaSuccess;
}

cudaError_t gemm_group_launch(const GemmGroupPlan& plan, cudaStream_t stream) {
    if (!g_configured) {
        cudaError_t e = gemm_configure();
        if (e != cudaSuccess) return e;
    }
    if (plan.stateful)
        tc_wgrad_group_kernel<true><<<plan.n, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev);
    else
        tc_wgrad_group_kernel<false><<<plan.n, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev);
    g_launches.fetch_add(plan.n_gemms, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <int MODE>
static cudaError_t launch_mode(const GemmPlan& plan, cudaStream_t stream) {
    if (!g_configured) {
        cudaError_t e = gemm_configure();
        if (e != cudaSuccess) return e;
    }
    if constexpr (MODE != GEMM_WGRAD) {
        if (plan.p.k_splits > 1) {
            tc_gemm_kernel<MODE, true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.tmA, plan.tmB, plan.tmC, plan.p);
            g_launches.fetch_add(1, std::memory_order_relaxed);
            return cudaGetLastError();
        }
    } else {
        if (is_stateful(plan.p)) {
            tc_gemm_kernel<MODE, false, true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.tmA, plan.tmB, plan.tmC, plan.p);
            g_launches.fetch_add(1, std::memory_order_relaxed);
            return cudaGetLastError();
        }
    }
    tc_gemm_kernel<MODE><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.tmA, plan.tmB, plan.tmC, plan.p);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

cudaError_t gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
    switch (plan.mode) {
        case GEMM_FWD: return launch_mode<GEMM_FWD>(plan, stream);
        case GEMM_DGRAD: return launch_mode<GEMM_DGRAD>(plan, stream);
        case GEMM_WGRAD: return launch_mode<GEMM_WGRAD>(plan, stream);
    }
    return cudaErrorInvalidValue;
}

}  // namespace ssb
