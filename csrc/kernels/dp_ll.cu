// Latency-optimal fused data-parallel path for narrow layers (the reference's workload): ONE kernel for the whole
// stage does, per [128 x 32] weight tile,
//
//     dW tile = dZ^T X                       mma.sync (3xTF32 or TF32), accumulator in registers
//  A) every row of the partial goes to the replica that OWNS the row        (reduce-scatter hop, NVLink)
//  B) the owner sums the dp partials in rank order, applies SGD              (bit-identical everywhere: computed once)
//  C) and sends the NEW WEIGHTS of its rows to every replica                 (all-gather hop, NVLink)
//
// with no system fence, no flag round trip and no NCCL: both hops use "LL" lines - 16-byte stores
// { value, epoch, value, epoch } straight into the peer's landing zone; the receiver polls the line until both epoch
// words match (8-byte halves are single-copy atomic over NVLink: the protocol NCCL's LL kernels rely on).  A hop costs
// one NVLink one-way latency plus wire time, instead of push + __threadfence_system() (4.4 us measured) + flag +
// acquire.  Epoch-valued lines never need clearing; landing zones are double-buffered by epoch parity.
//
// The kernel is launched at the START of the step next to the layer-chain kernel (one CTA per tile, all layers in
// one grid, co-resident by construction: tiles + chain CTAs <= #SMs).  Each CTA's TMA producer waits on the chain
// kernel's per-layer device counter (dz[l] final and W_l no longer read by dgrad), so the communication of layer l
// overlaps the backward pass of layers l-1 .. 1 - the reference's overlap structure
// (shallowspeed/pipe.py:302-327, 389-400 of the reference), tile by tile instead of layer by layer.
//
// Deadlock freedom: phase A never waits; phase B waits only for phase-A lines; phase C only for phase-B lines; every
// CTA of every rank is resident; all spins are bounded (trap instead of hanging the GPU).
#include "kernels.h"
#include "ptx.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace ssb {

static constexpr int kThreads = 160;                   // warp 0 TMA, warps 1..4 MMA + epilogue / protocol
static constexpr uint32_t kBlockM = 128;
static constexpr uint32_t kBlockK = 32;
static constexpr uint32_t kABytes = kBlockM * 128;     // dZ^T tile of one k-block: 4 MN-major panels
static constexpr uint32_t kPanelBytes = 32 * 128;
static constexpr uint32_t kBBytes = kPanelBytes;       // X tile: one 32-wide MN-major panel
static constexpr int kOwnLd = 34;                      // pitch (floats) of the tile staged in shared memory: 32 values + bias gradient

__device__ __forceinline__ void st_ll(uint4* p, float a, float b, uint32_t epoch) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(__float_as_uint(a)), "r"(epoch),
                 "r"(__float_as_uint(b)), "r"(epoch)
                 : "memory");
}
__device__ __forceinline__ uint4 ld_ll(const uint4* p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ bool ll_ready(const uint4& v, uint32_t epoch) { return v.y == epoch && v.w == epoch; }
// poll one line until it carries this step's epoch (bounded)
__device__ __forceinline__ uint4 wait_ll(const uint4* p, uint4 v, uint32_t epoch) {
    if (ll_ready(v, epoch)) return v;
    const long long t0 = clock64();
    do {
        v = ld_ll(p);
        if (clock64() - t0 > SSB_SPIN_LIMIT_CYCLES) __trap();
    } while (!ll_ready(v, epoch));
    return v;
}

__device__ __forceinline__ unsigned long long gtime_ll() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// optional phase timeline (SSB_CHAIN_TIMELINE=1): 8 stamps per tile, written by the tile's first epilogue thread
#define LLDBG(i) do { if (p.dbg != nullptr && etid == 0 && e.tile < 28) p.dbg[8 * e.tile + (i)] = gtime_ll(); } while (0)

// STATEFUL: momentum / weight decay in phase B through sgd_direction; the owner of a row keeps its momentum in its LOCAL
// arena (p.opt.V, loaded with the weights before the first wait) and never sends it.
template <int DP, bool STATEFUL = false>
__global__ void __launch_bounds__(kThreads, 1) dp_ll_wgrad_kernel(const DpLLEntry* __restrict__ entries, const DpLLParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t smem_base = (raw + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - raw);

    const DpLLEntry& e = entries[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = (e.k_total + (int)kBlockK - 1) / (int)kBlockK;
    const uint32_t stage_bytes = kABytes + kBBytes;
    const uint32_t own_off = p.stages * stage_bytes;                       // tile staging [128 rows][kOwnLd] floats
    const uint32_t own_bytes = kBlockM * kOwnLd * 4u;
    const uint32_t bar_base = smem_base + own_off + own_bytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&e.tmA);
        tma_prefetch_desc(&e.tmB);
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);          // one arrive per math warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 0) {
        // ------------------------------------------------------------ TMA producer (converged warp, elected lane issues)
        if (e.gate_flag != nullptr) {
            wait_counter_ge_gpu(e.gate_flag, e.gate_mult * ld_acquire_gpu(p.gate_step));
            fence_proxy_async_global();          // the chain kernel's generic-proxy stores -> my TMA reads
            __syncwarp();
        }
        for (int kb = 0; kb < num_kb; ++kb) {
            const int s = kb % p.stages;
            mbar_wait(empty_bar(s), ((kb / p.stages) & 1) ^ 1);
            if (elect_one()) {
                mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                const uint32_t a_dst = smem_base + s * stage_bytes, b_dst = a_dst + kABytes;
                const int k0 = kb * (int)kBlockK;
#pragma unroll
                for (int i = 0; i < 4; ++i) tma_load_2d(a_dst + i * kPanelBytes, &e.tmA, full_bar(s), e.m0 + 32 * i, k0);
                tma_load_2d(b_dst, &e.tmB, full_bar(s), e.n0, k0);
            }
            __syncwarp();
        }
    } else {
        // ------------------------------------------------------------ math warps: the GEMM + the LL protocol
        const uint32_t epoch = *reinterpret_cast<const volatile uint32_t*>(p.epoch_ptr);
        const uint32_t parity = epoch & 1u;
        const int q = warp & 3;
        const int m_local = q * 32 + lane;                       // row of the tile owned by this thread after the GEMM
        const int etid = (warp - 1) * 32 + lane;                 // 0..127
        constexpr int rpo = (int)kBlockM / DP;                   // rows per owner
        const int lpr = e.has_bias ? 17 : 16;                    // lines per row (line 16 = bias gradient / new bias)
        const int rows_valid = min((int)kBlockM, e.m_total - e.m0);
        float* own = reinterpret_cast<float*>(smem_gen + own_off);

        LLDBG(0);                                                // CTA resident, waiting for operands
        // this warp's 32 rows of the tile, and the bias gradient of my row: column sum of dZ over the local rows, read
        // from the staged A panels
        float acc[2][4][4];
        warp_acc_zero(acc);
        float dbsum = 0.f;
        for (int kb = 0; kb < num_kb; ++kb) {
            const int s = kb % p.stages;
            mbar_wait(full_bar(s), (kb / p.stages) & 1);
            const uint32_t a_src = smem_base + s * stage_bytes;
            if (e.split) warp_mma_kblock<4, true, true, true>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, 4, lane);
            else warp_mma_kblock<4, true, true, false>(acc, a_src, (uint32_t)q * 32u, a_src + kABytes, 0u, 4, lane);
            if (e.has_bias) {
#pragma unroll 8
                for (int r = 0; r < 32; ++r) dbsum += lds_f32(a_src + operand_off<true>((uint32_t)m_local, (uint32_t)r));
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));
        }
        LLDBG(1);                                                // all operand tiles landed (gate open + TMA)
        LLDBG(2);                                                // accumulator complete

        // ---------------- phase A: every row of the partial goes to the owner of that row.  The tile is staged in shared
        // memory first so that consecutive lanes write consecutive 16-byte lines: a replica's slice [rpo rows][lpr lines]
        // is contiguous in its landing zone, i.e. every warp store is one 512-byte run on the wire.
        warp_acc_to_rows(acc, own + q * 32 * kOwnLd, kOwnLd, 4, lane);
        own[m_local * kOwnLd + 32] = dbsum;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        {
            const int n_lines = rows_valid * lpr;
            for (int idx = etid; idx < n_lines; idx += 128) {
                const int row = idx / lpr, j = idx - row * lpr;
                const int owner = row / rpo;
                if (owner == p.rank) continue;
                uint4* dst = p.llA[owner] + ((((size_t)parity * DP + p.rank) * p.n_tiles + e.tile) * rpo + (row - owner * rpo)) * 17 + j;
                if (j < 16) st_ll(dst, own[row * kOwnLd + 2 * j], own[row * kOwnLd + 2 * j + 1], epoch);
                else st_ll(dst, own[row * kOwnLd + 32], 0.f, epoch);
            }
        }

        LLDBG(3);                                                // phase A lines issued
        // ---------------- phase B: reduce the rows I own in rank order, SGD, publish the new weights.
        // Every thread owns up to kLB lines; ALL polls and weight loads of the batch are issued before the first wait -
        // a line-by-line loop pays one L2 round trip per poll plus one per weight load (measured: 9 us at dp = 2).
        if (e.gate_w != nullptr) {
            // the update overwrites W_l in place: the chain kernel's dgrad of this layer must have consumed it
            if (etid == 0) wait_counter_ge_gpu(e.gate_w, e.gate_mult * ld_acquire_gpu(p.gate_step));
            asm volatile("bar.sync 1, 128;" ::: "memory");
        }
        {
            constexpr int kLB = (rpo * 17 + 127) / 128;          // dp 2: 9, dp 4: 5, dp 8: 3
            const int my_rows = max(0, min(rpo, rows_valid - p.rank * rpo));
            const int n_lines = my_rows * lpr;
            const float* mine0 = own + (p.rank * rpo) * kOwnLd;
            const uint4* zoneA = p.llA[p.rank] + (size_t)parity * DP * p.n_tiles * rpo * 17;
            const float lr = *p.lr;                              // in flight with the first batch's loads
            for (int i0 = etid; i0 < n_lines; i0 += 128 * kLB) {
                uint4 ln[kLB][DP];
                float wv0[kLB], wv1[kLB];
                float vv0[kLB], vv1[kLB];                // momentum (STATEFUL only)
#pragma unroll
                for (int u = 0; u < kLB; ++u) {
                    const int idx = i0 + 128 * u;
                    if (idx >= n_lines) continue;
                    const int r = idx / lpr, j = idx - r * lpr;
#pragma unroll
                    for (int sr = 0; sr < DP; ++sr)
                        if (sr != p.rank) ln[u][sr] = ld_ll(zoneA + (((size_t)sr * p.n_tiles + e.tile) * rpo + r) * 17 + j);
                    const float* wrow = p.W + e.w_offset + (int64_t)(e.m0 + p.rank * rpo + r) * e.ldw;
                    const int n = j < 16 ? e.n0 + 2 * j : e.n_total;
                    wv0[u] = (j == 16 || n < e.n_total) ? wrow[n] : 0.f;
                    wv1[u] = (j < 16 && n + 1 < e.n_total) ? wrow[n + 1] : 0.f;
                    if constexpr (STATEFUL) {
                        const float* vrow = p.opt.V != nullptr ? p.opt.V + (wrow - p.W) : nullptr;
                        vv0[u] = (vrow != nullptr && (j == 16 || n < e.n_total)) ? vrow[n] : 0.f;
                        vv1[u] = (vrow != nullptr && j < 16 && n + 1 < e.n_total) ? vrow[n + 1] : 0.f;
                    }
                }
#pragma unroll
                for (int u = 0; u < kLB; ++u) {
                    const int idx = i0 + 128 * u;
                    if (idx >= n_lines) continue;
                    const int r = idx / lpr, j = idx - r * lpr;
                    float s0 = 0.f, s1 = 0.f;
#pragma unroll
                    for (int sr = 0; sr < DP; ++sr) {
                        float a, b;
                        if (sr == p.rank) {
                            a = mine0[r * kOwnLd + (j < 16 ? 2 * j : 32)];
                            b = j < 16 ? mine0[r * kOwnLd + 2 * j + 1] : 0.f;
                        } else {
                            const uint4 x = wait_ll(zoneA + (((size_t)sr * p.n_tiles + e.tile) * rpo + r) * 17 + j, ln[u][sr], epoch);
                            a = __uint_as_float(x.x);
                            b = __uint_as_float(x.z);
                        }
                        s0 = (sr == 0) ? a : s0 + a;             // fixed order 0, 1, .., dp-1: deterministic
                        s1 = (sr == 0) ? b : s1 + b;
                    }
                    const int row = p.rank * rpo + r;            // row inside the tile
                    float* wrow = p.W + e.w_offset + (int64_t)(e.m0 + row) * e.ldw;
                    float w0 = 0.f, w1 = 0.f;
                    if constexpr (STATEFUL) {                    // s0 / s1 become the step directions
                        const float mu = p.opt.momentum, wd = p.opt.weight_decay;
                        const bool nv = p.opt.nesterov != 0;
                        s0 = sgd_direction<false>(s0, wv0[u], vv0[u], mu, wd, nv);
                        s1 = sgd_direction<false>(s1, wv1[u], vv1[u], mu, wd, nv);
                        if (p.opt.V != nullptr) {
                            float* vrow = p.opt.V + (wrow - p.W);
                            if (j < 16) {
                                const int n = e.n0 + 2 * j;
                                if (n < e.n_total) vrow[n] = vv0[u];
                                if (n + 1 < e.n_total) vrow[n + 1] = vv1[u];
                            } else {
                                vrow[e.n_total] = vv0[u];
                            }
                        }
                    }
                    if (j < 16) {
                        const int n = e.n0 + 2 * j;
                        if (n < e.n_total) { w0 = wv0[u] - lr * s0; wrow[n] = w0; }
                        if (n + 1 < e.n_total) { w1 = wv1[u] - lr * s1; wrow[n + 1] = w1; }
                    } else {
                        w0 = wv0[u] - lr * s0;                 // bias lives in column `in` of the block
                        wrow[e.n_total] = w0;
                    }
#pragma unroll
                    for (int d = 0; d < DP; ++d)
                        if (d != p.rank) st_ll(p.llC[d] + (((size_t)parity * p.n_tiles + e.tile) * kBlockM + row) * 17 + j, w0, w1, epoch);
                }
            }
        }

        LLDBG(4);                                                // my rows reduced, updated and published
        // ---------------- phase C: rows owned by other replicas: their new weights arrive as LL lines (coalesced polls,
        // a batch of loads in flight per thread before the first wait)
        {
            const int n_lines = rows_valid * lpr;
            const uint4* zone = p.llC[p.rank] + ((size_t)parity * p.n_tiles + e.tile) * kBlockM * 17;
            constexpr int kB = 6;
            for (int i0 = etid; i0 < n_lines; i0 += 128 * kB) {
                uint4 ln[kB];
                int rowv[kB], jv[kB];
#pragma unroll
                for (int u = 0; u < kB; ++u) {
                    const int idx = i0 + 128 * u;
                    rowv[u] = -1;
                    if (idx >= n_lines) continue;
                    const int row = idx / lpr, j = idx - row * lpr;
                    if (row / rpo == p.rank) continue;
                    rowv[u] = row; jv[u] = j;
                    ln[u] = ld_ll(zone + (size_t)row * 17 + j);
                }
#pragma unroll
                for (int u = 0; u < kB; ++u) {
                    if (rowv[u] < 0) continue;
                    const uint4 x = wait_ll(zone + (size_t)rowv[u] * 17 + jv[u], ln[u], epoch);
                    float* wrow = p.W + e.w_offset + (int64_t)(e.m0 + rowv[u]) * e.ldw;
                    if (jv[u] < 16) {
                        const int n = e.n0 + 2 * jv[u];
                        if (n < e.n_total) wrow[n] = __uint_as_float(x.x);
                        if (n + 1 < e.n_total) wrow[n + 1] = __uint_as_float(x.z);
                    } else {
                        wrow[e.n_total] = __uint_as_float(x.x);
                    }
                }
            }
        }
        LLDBG(5);                                                // all replicas' rows written locally
    }
}

// =========================================================================== host side
const char* make_tmap_mn(CUtensorMap* map, const float* base, int inner, int outer, int ld);   // tc_gemm.cu

int dp_ll_tiles(int in, int out) { return ((out + (int)kBlockM - 1) / (int)kBlockM) * ((in + 31) / 32); }
size_t dp_ll_zone_lines(int dp, int n_tiles) { return (size_t)2 * n_tiles * kBlockM * 17; }   // identical for llA and llC

const char* dp_ll_plan(DpLLPlan* plan, const DpLLLayer* layers, int n_layers, int rows, const DpLLParams& base) {
    *plan = DpLLPlan{};
    plan->p = base;
    if (base.dp != 2 && base.dp != 4 && base.dp != 8) return "dp_ll_plan: dp must be 2, 4 or 8";
    if (base.lr == nullptr) return "dp_ll_plan: lr (the device learning-rate slot) is not set";
    std::vector<DpLLEntry> host;
    int tile = 0;
    bool split = false;
    for (int l = 0; l < n_layers; ++l) {
        const DpLLLayer& ly = layers[l];
        CUtensorMap tmA, tmB;
        if (const char* err = make_tmap_mn(&tmA, ly.dZ, ly.out, rows, ly.lddz)) return err;
        if (const char* err = make_tmap_mn(&tmB, ly.X, ly.in, rows, ly.ldx)) return err;
        const bool sp = ly.split != 0;                              // 3xTF32: the kernel derives the lo parts from the tiles
        split = split || sp;
        const int tm = (ly.out + (int)kBlockM - 1) / (int)kBlockM, tn = (ly.in + 31) / 32;
        for (int mt = 0; mt < tm; ++mt)
            for (int nt = 0; nt < tn; ++nt) {
                DpLLEntry e;
                memset(&e, 0, sizeof(e));
                e.tmA = tmA; e.tmB = tmB;
                e.m0 = mt * (int)kBlockM; e.n0 = nt * 32;
                e.m_total = ly.out; e.n_total = ly.in; e.k_total = rows;
                e.split = sp ? 1 : 0;
                e.has_bias = nt == 0 ? 1 : 0;
                e.tile = tile++;
                e.w_offset = ly.w_offset; e.ldw = ly.ldw;
                e.gate_flag = ly.gate_flag; e.gate_w = ly.gate_w; e.gate_mult = ly.gate_mult;
                host.push_back(e);
            }
    }
    if (tile != base.n_tiles) return "dp_ll_plan: tile count does not match the landing zones of the DpContext";
    const int num_kb = (rows + (int)kBlockK - 1) / (int)kBlockK;
    const int stage_bytes = (int)(kABytes + kBBytes);
    int stages = (190 * 1024) / stage_bytes;
    stages = std::min(stages, std::max(num_kb, 2));
    stages = std::min(stages, 8);
    plan->p.stages = stages;
    plan->smem_bytes = stages * stage_bytes + (int)kBlockM * kOwnLd * 4 + 1024 + 8 * (2 * stages) + 16;
    DpLLEntry* dev = nullptr;
    if (cudaMalloc(&dev, host.size() * sizeof(DpLLEntry)) != cudaSuccess) return "dp_ll_plan: cudaMalloc failed";
    if (cudaMemcpy(dev, host.data(), host.size() * sizeof(DpLLEntry), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(dev);
        return "dp_ll_plan: table upload failed";
    }
    plan->entries_dev = dev;
    plan->grid = (int)host.size();
    return nullptr;
}

void dp_ll_free(DpLLPlan* plan) {
    if (plan->entries_dev) cudaFree(plan->entries_dev);
    plan->entries_dev = nullptr;
}

cudaError_t dp_ll_configure() {
    cudaError_t err;
    if ((err = cudaFuncSetAttribute(dp_ll_wgrad_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024)) != cudaSuccess) return err;
    if ((err = cudaFuncSetAttribute(dp_ll_wgrad_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024)) != cudaSuccess) return err;
    if ((err = cudaFuncSetAttribute(dp_ll_wgrad_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024)) != cudaSuccess) return err;
    if ((err = cudaFuncSetAttribute(dp_ll_wgrad_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024)) != cudaSuccess) return err;
    if ((err = cudaFuncSetAttribute(dp_ll_wgrad_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024)) != cudaSuccess) return err;
    return cudaFuncSetAttribute(dp_ll_wgrad_kernel<8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
}

cudaError_t launch_dp_ll(const DpLLPlan& plan, cudaStream_t stream) {
    const bool stateful = plan.p.opt.momentum != 0.f || plan.p.opt.weight_decay != 0.f;
    switch (plan.p.dp) {
        case 2:
            if (stateful) dp_ll_wgrad_kernel<2, true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            else dp_ll_wgrad_kernel<2><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            break;
        case 4:
            if (stateful) dp_ll_wgrad_kernel<4, true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            else dp_ll_wgrad_kernel<4><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            break;
        case 8:
            if (stateful) dp_ll_wgrad_kernel<8, true><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            else dp_ll_wgrad_kernel<8><<<plan.grid, kThreads, plan.smem_bytes, stream>>>(plan.entries_dev, plan.p);
            break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace ssb
