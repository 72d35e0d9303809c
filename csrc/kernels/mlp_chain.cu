// Host side of the layer-chain kernel (mlp_chain.cuh): plans, shared-memory budgets, and the launches, with the 3xTF32
// instantiations; the TF32 and BF16 ones are in mlp_chain_tf32.cu and mlp_chain_bf16.cu, the residual ones in
// mlp_chain_res.cu (3xTF32), mlp_chain_res_tf32.cu and mlp_chain_res_bf16.cu.
#include "mlp_chain.cuh"

namespace ssb {

int chain_ksplit_kblocks(int nkb, int part, int* kblocks) {
    const int n = chain_ksplit_count(nkb, part);
    for (int i = 0; i < n; ++i) kblocks[i] = chain_ksplit_kblock(i, part);
    return n;
}

const char* make_tmap_mn(CUtensorMap* map, const float* base, int inner, int outer, int ld);                 // tc_gemm.cu
const char* make_tmap_k(CUtensorMap* map, const float* base, int inner, int outer, int ld, int box_outer);   // tc_gemm.cu

// Shared-memory plan of the chain kernel for one micro-batch size: k-panels per ring stage, ring depth, total bytes.
// Pure host arithmetic (no CUDA calls) so it can be unit-tested without a GPU (tests/test_planning.py).
// No precision needs extra shared memory: 3xTF32 derives the lo parts from the staged tiles, BF16 rounds the operands in
// registers.
bool chain_budget(int mb_rows, int prec, int* kps_out, int* stages_out, int* smem_bytes_out) {
    if (!prec_valid(prec)) return false;
    if (mb_rows < 1 || mb_rows > 128) return false;
    const int n_pad = (mb_rows + 15) / 16 * 16;
    const int abuf_bytes = 4 * n_pad * 128;
    const int scratch_bytes = n_pad * kScratchLd * 4 + 256;   // loss head
    const int budget = 222 * 1024 - 2 * abuf_bytes - scratch_bytes;
    int kps = 4, stage_bytes = 0, stages = 0;
    for (; kps >= 1; kps >>= 1) {            // biggest stage (fewest waits/commits) that still double-buffers
        stage_bytes = kps * ((int)kABytes + n_pad * 128);
        stages = budget / stage_bytes;
        if (stages >= 2) break;
    }
    if (kps < 1 || stages < 2) return false;
    if (stages > 8) stages = 8;
    *kps_out = kps;
    *stages_out = stages;
    *smem_bytes_out = stages * stage_bytes + 2 * abuf_bytes + 1024 + 8 * (2 * stages) + 128 + scratch_bytes;
    return true;
}

// accumulator width (n8 tiles) of a math warp, the NTW instantiation chain_launch picks
static int chain_ntw(int n_pad) {
    const int cols = chain_warp_cols(n_pad);
    return cols <= 16 ? 2 : cols <= 32 ? 4 : 8;
}

int chain_cluster_size(const ChainLayer* layers, int n_layers, bool do_fwd, bool do_loss, bool do_bwd, bool first_stage,
                       bool gated, bool folded) {
    // gated: the co-resident consumer's eligibility assumes the chain occupies one SM per micro-batch; folded: the
    // flag / credit protocol of the pipeline boundaries runs per CTA
    if (gated || folded || n_layers < 1) return 1;
    int w = 0;
    if (do_fwd)
        for (int l = 0; l < n_layers; ++l) w = std::max(w, layers[l].out);
    if (do_bwd) {
        for (int l = first_stage ? 2 : 1; l <= n_layers; ++l) w = std::max(w, layers[l - 1].in);
        if (!(do_fwd && do_loss)) w = std::max(w, layers[n_layers - 1].out);   // dZ_L staged from global memory
    }
    return std::min(4, std::max(1, (w + 31) / 32));
}

// Cluster form: the ring holds 32-row weight panels (plus the X tiles of layer 1); behind the three cluster-form
// barriers, the landing area of a k-split layer 1's helper (256 N bytes, 16-byte aligned) and the loss head's scratch.
bool chain_cluster_budget(int mb_rows, int cluster, int prec, int* kps_out, int* stages_out, int* smem_bytes_out) {
    if (cluster <= 1) return chain_budget(mb_rows, prec, kps_out, stages_out, smem_bytes_out);
    if (!prec_valid(prec) || cluster > 4 || mb_rows < 1 || mb_rows > 128) return false;
    const int n_pad = (mb_rows + 15) / 16 * 16;
    const int abuf_bytes = 4 * n_pad * 128;
    const int scratch_bytes = 16 + 256 * n_pad + n_pad * kScratchLd * 4 + 256;
    const int budget = 222 * 1024 - 2 * abuf_bytes - scratch_bytes;
    int kps = 4, stage_bytes = 0, stages = 0;
    for (; kps >= 1; kps >>= 1) {
        stage_bytes = kps * ((int)kPanelBytes + n_pad * 128);
        stages = budget / stage_bytes;
        if (stages >= 2) break;
    }
    if (kps < 1 || stages < 2) return false;
    if (stages > 8) stages = 8;
    *kps_out = kps;
    *stages_out = stages;
    *smem_bytes_out = stages * stage_bytes + 2 * abuf_bytes + 1024 + 8 * (2 * stages + 3) + 128 + scratch_bytes;
    return true;
}

static bool chain_smem_fits(int mb_rows, int prec) {
    int kps, stages, smem;
    return chain_budget(mb_rows, prec, &kps, &stages, &smem);
}

bool chain_eligible(const ChainLayer* layers, int n_layers, int mb_rows, int out_dim, bool has_loss, int prec) {
    if (!chain_smem_fits(mb_rows, prec)) return false;
    if (n_layers < 1 || n_layers > kChainMaxLayers || mb_rows < 1 || mb_rows > 128) return false;
    for (int l = 0; l < n_layers; ++l) {
        if (layers[l].out > 128) return false;
        if (l > 0 && layers[l].in > 128) return false;
    }
    if (has_loss && (out_dim > 32 || layers[n_layers - 1].out != out_dim)) return false;
    return true;
}

const char* chain_plan(ChainPlan* plan, const ChainParams& params, const float* x, int ldx, int total_rows, int n_mubatches,
                       int prec) {
    *plan = ChainPlan{};
    if (!prec_valid(prec)) return "chain_plan: unknown precision";
    ChainParams& p = plan->p;
    p = params;
    const int L = p.n_layers;
    p.n_pad = (p.mb_rows + 15) / 16 * 16;
    p.prec = prec;                                // 3xTF32: the kernel derives the lo parts of its operands from the staged tiles
    const bool fold = p.in_flag != nullptr || p.out_peer != nullptr || p.x_from_global != 0;
    const int C = chain_cluster_size(p.layers, L, p.do_fwd != 0, p.do_loss != 0, p.do_bwd != 0, p.first_stage != 0,
                                     p.ready != nullptr, fold);
    if (C > 1 && (p.ready != nullptr || fold)) return "chain_plan: gated and folded launches run one CTA per micro-batch";
    p.cluster = C;
    // a cluster launch whose layer 1 has more than 4 k-blocks runs it on P = 2 CTAs per feature slice (k-split)
    const int P = C > 1 && p.do_fwd && (p.layers[0].in + (int)kBlockK - 1) / (int)kBlockK > 4 ? 2 : 1;
    p.ksplit = P;
    // a k-split layer 1 has more than 128 inputs and at most 128 outputs: never residual, and the split has no skip form
    if (P > 1 && (p.res_mask & 1u)) return "chain_plan: a k-split layer 1 cannot be residual";
    std::vector<CUtensorMap> host(2 * L + 1);
    for (int l = 0; l < L; ++l) {
        const ChainLayer& ly = p.layers[l];
        // forward A operand: all 128 feature rows per k-block, or the 32 of one CTA of a cluster
        if (const char* e = make_tmap_k(&host[2 * l], p.W + ly.w_off, ly.in, ly.out, ly.ldw, C > 1 ? 32 : (int)kBlockM)) return e;
        if (const char* e = make_tmap_mn(&host[2 * l + 1], p.W + ly.w_off, ly.in, ly.out, ly.ldw)) return e;
    }
    if (x != nullptr) {
        if (const char* e = make_tmap_k(&host[2 * L], x, p.layers[0].in, total_rows, ldx, p.n_pad)) return e;
    } else {
        host[2 * L] = host[0];
    }
    CUtensorMap* dev = nullptr;
    if (cudaMalloc(&dev, host.size() * sizeof(CUtensorMap)) != cudaSuccess) return "chain_plan: cudaMalloc failed";
    if (cudaMemcpy(dev, host.data(), host.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice) != cudaSuccess)
        return "chain_plan: tensor map upload failed";
    plan->maps_dev = dev;
    p.maps = dev;
    int kps = 0, stages = 0, smem = 0;
    if (!chain_cluster_budget(p.mb_rows, C, p.prec, &kps, &stages, &smem)) return "chain_plan: shared memory budget too small";
    p.kps = kps;
    p.stages = stages;
    plan->smem_bytes = smem;
    plan->grid = n_mubatches * C * P;
    plan->cluster = C;
    plan->ksplit = P;
    return nullptr;
}

void chain_plan_free(ChainPlan* plan) {
    if (plan->maps_dev) cudaFree(plan->maps_dev);
    plan->maps_dev = nullptr;
}

// the instantiation of a (precision, residual) pair, from the translation unit that compiles it
static ChainKernel chain_kernel_of(int prec, bool res, ChainForm form, int ntw, bool ce, bool drop, bool gate) {
    switch (prec) {
        case PREC_TF32: return (res ? chain_kernel_res_tf32 : chain_kernel_tf32)(form, ntw, ce, drop, gate);
        case PREC_3XTF32:
            return res ? chain_kernel_res_3xtf32(form, ntw, ce, drop, gate)
                       : chain_kernel<PREC_3XTF32, false>(form, ntw, ce, drop, gate);
        case PREC_BF16: return (res ? chain_kernel_res_bf16 : chain_kernel_bf16)(form, ntw, ce, drop, gate);
    }
    return nullptr;
}

cudaError_t chain_configure() {
    static bool configured = false;
    if (configured) return cudaSuccess;
    for (int prec : {PREC_TF32, PREC_3XTF32, PREC_BF16})
        for (ChainForm form : {CHAIN_PLAIN, CHAIN_FOLD, CHAIN_CLUSTER})
            for (int ntw : {2, 4, 8})
                for (int key = 0; key < 16; ++key)     // residual, cross-entropy, dropout, gated
                    if (ChainKernel fn = chain_kernel_of(prec, key & 1, form, ntw, key & 2, key & 4, key & 8)) {
                        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
                        if (e != cudaSuccess) return e;
                    }
    configured = true;
    return cudaSuccess;
}

// grid = micro-batches x plan.cluster x plan.ksplit; cluster dims (plan.cluster x plan.ksplit, 1, 1) for a cluster plan
cudaError_t chain_launch(const ChainPlan& plan, cudaStream_t stream) {
    const ChainParams& p = plan.p;
    if (p.loss_kind != LOSS_MSE && p.loss_kind != LOSS_CROSS_ENTROPY) return cudaErrorInvalidValue;
    if (!act_valid(p.act_kind)) return cudaErrorInvalidValue;
    if (cudaError_t e = chain_configure(); e != cudaSuccess) return e;
    const bool fold = p.in_flag != nullptr || p.out_peer != nullptr || p.x_from_global != 0;
    const ChainForm form = plan.cluster > 1 ? CHAIN_CLUSTER : fold ? CHAIN_FOLD : CHAIN_PLAIN;
    // a residual model is gated for every activation kind
    ChainKernel fn = chain_kernel_of(p.prec, p.res != 0, form, chain_ntw(p.n_pad), p.loss_kind == LOSS_CROSS_ENTROPY,
                                     p.drop.on(), p.res != 0 || act_smooth(p.act_kind));
    if (fn == nullptr) return cudaErrorInvalidValue;
    if (form == CHAIN_CLUSTER) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)plan.grid);
        cfg.blockDim = dim3(kThreads);
        cfg.dynamicSmemBytes = (size_t)plan.smem_bytes;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)(plan.cluster * plan.ksplit);
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        if (cudaError_t e = cudaLaunchKernelEx(&cfg, fn, p); e != cudaSuccess) return e;
    } else {
        fn<<<plan.grid, kThreads, plan.smem_bytes, stream>>>(p);
    }
    return cudaGetLastError();
}

}  // namespace ssb
