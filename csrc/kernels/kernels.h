// Host-side launch API of the hand-written sm_90a kernels (no torch dependency, so the
// .cu files compile stand-alone with nvcc and the C++ runtime can call them directly).
#pragma once
#include <cstdint>
#include <vector>
#include <cuda.h>
#include <cuda_runtime.h>

namespace ssb {

enum GemmMode : int { GEMM_FWD = 0, GEMM_DGRAD = 1, GEMM_WGRAD = 2 };

// Loss of the last stage's head.  MSE: the reference's softmax (shift by the micro-batch's global max, +1e-7) followed by
// the MSE loss.  CROSS_ENTROPY: softmax cross-entropy with probability targets, per-row softmax (ptx.cuh: ce_*).
enum LossKind : int { LOSS_MSE = 0, LOSS_CROSS_ENTROPY = 1 };

// Hyper-parameters of the SGD update beyond lr (torch.optim.SGD, dampening 0).  The default is plain SGD, w -= lr * g,
// which runs the stateless kernels.  V: momentum buffer laid out like the weights it belongs to (nullptr when
// momentum == 0: weight decay alone needs no state).
struct SgdState {
    float* V = nullptr;
    float momentum = 0.f;
    float weight_decay = 0.f;
    int nesterov = 0;
    bool plain() const { return momentum == 0.f && weight_decay == 0.f; }
};
// nullptr if the combination is valid: 0 <= momentum < 1, weight_decay >= 0, nesterov only with momentum, and a
// buffer exactly when momentum > 0
const char* sgd_state_check(const SgdState& s);

// One description for the three Linear GEMMs.  Every GEMM is issued "swapped": the
// FEATURE dimension sits on the M axis of the 128-row tile and the skinny dimension
// (micro-batch rows: 4..256) on the N axis, so a 4-row micro-batch costs an N=16 tile
// instead of a 128-row tile that is 97 % padding.
//
//   FWD   D[m=out, n=row] = sum_k W[m,k]  * X[n,k]      A=W   (K-major)  B=X  (K-major)
//   DGRAD D[m=in,  n=row] = sum_k W[k,m]  * dZ[n,k]     A=W   (MN-major) B=dZ (K-major)
//   WGRAD D[m=out, n=in ] = sum_k dZ[k,m] * X[k,n]      A=dZ  (MN-major) B=X  (MN-major)
struct GemmParams {
    int m_total, n_total, k_total;
    int block_n;        // tile N: multiple of 16 (32 when B is MN-major), <= 64
    int stages;         // smem pipeline depth
    // FWD / DGRAD epilogue: out[n * ldo + m]
    float* out;
    int ldo;
    const float* bias;  // FWD: + bias[m * bias_stride] (nullable)
    int bias_stride;
    int relu;           // FWD: max(.,0)
    const float* mask;  // DGRAD: zero where mask[n * ldmask + m] <= 0 (nullable) - the ReLU
    int ldmask;         //        backward of the PREVIOUS layer fused into this epilogue
    // WGRAD epilogue: G[m * ldg + n] (+)= D ; db[m * db_stride] (+)= sum_k dZ[k, m]
    float* G;
    int ldg;
    int accumulate;
    float* db;          // nullable
    int db_stride;
    // WGRAD with the SGD update fused (single replica, not combinable with accumulate):
    // the -lr-scaled tile is TMA-reduce-added into W; G is never touched.  lr: one device float, read once per thread
    // at run time (a learning-rate schedule rewrites it between steps without re-planning)
    float* W;
    int ldw;
    const float* lr;
    int fuse_sgd;
    // stateful update rule of the fused SGD (see SgdState): V = momentum buffer with W's layout (pitch ldw, nullable
    // when momentum == 0), read and written per element; W is read as well when weight_decay != 0
    float* V;
    float momentum, weight_decay;
    int nesterov;
    // fp32-equivalent mode (3xTF32 products, the operands' lo parts x - trunc_tf32(x) derived in the kernel)
    int split;
    // split-K (FWD / DGRAD, see gemm_plan_enable_splitk): blockIdx.z owns a k-range, partial tiles go through
    // `partial` [tile][split][block_n][128], the last arriver at tile_counter[tile] reduces + runs the epilogue
    int k_splits;                 // 0 / 1 = off
    float* partial;
    unsigned int* tile_counter;   // zero before the first launch; re-armed by the kernel
};

struct GemmPlan {          // a fully prepared launch (tensor maps are 128 B each)
    CUtensorMap tmA, tmB, tmC;   // C: WGRAD output tile (G, or W when the SGD update is fused)
    GemmParams p;
    int mode;
    dim3 grid;
    int smem_bytes;
};

// Build tensor maps + launch geometry.  All matrices are fp32 row-major with a leading
// dimension that is a multiple of 4 floats and a 16-byte aligned base.
//   FWD:   W[out, in] (ldw), X[rows, in] (ldx)            -> Y[rows, out] (ldy)
//   DGRAD: W[out, in] (ldw), dZ[rows, out] (lddz)         -> dX[rows, in] (lddx)
//   WGRAD: dZ[rows, out] (lddz), X[rows, in] (ldx)        -> G[out, in] (ldg)
// split: false = plain TF32 products; true = 3xTF32 (fp32-equivalent; the kernels derive the operands' lo parts
// x - trunc_tf32(x) from the staged tiles)
const char* gemm_plan_fwd(GemmPlan* plan, const float* W, int ldw, const float* X, int ldx, float* Y, int ldy,
                          int rows, int in, int out, const float* bias, int bias_stride, int relu, bool split = false);
const char* gemm_plan_dgrad(GemmPlan* plan, const float* W, int ldw, const float* dZ, int lddz, float* dX, int lddx,
                            int rows, int in, int out, const float* mask, int ldmask, bool split = false);
const char* gemm_plan_wgrad(GemmPlan* plan, const float* dZ, int lddz, const float* X, int ldx, float* G, int ldg,
                            int rows, int in, int out, int accumulate, float* db, int db_stride, float* W, int ldw,
                            const float* lr, int fuse_sgd, bool split = false, const SgdState& opt = SgdState{});
// Split-K for FWD / DGRAD plans whose output has fewer tiles than the chip has SMs (wide, weight-bound layers):
// choice() returns the number of k-splits (1 = leave the plan alone); enable() rewires the plan (grid.z, ring
// depth for two CTAs per SM).  workspace: gemm_splitk_workspace_floats() floats; counters: one zeroed uint per tile.
int gemm_splitk_choice(const GemmPlan& plan, int num_sms);
size_t gemm_splitk_workspace_floats(const GemmPlan& plan, int k_splits);
const char* gemm_plan_enable_splitk(GemmPlan* plan, int k_splits, float* workspace, unsigned int* counters);
cudaError_t gemm_launch(const GemmPlan& plan, cudaStream_t stream);
// Grouped launch of several WGRAD plans (different layers) as ONE grid: a device table holds one entry per CTA.
struct alignas(128) GemmGroupEntry {
    CUtensorMap tmA, tmB, tmC;
    GemmParams p;
    int bx, by;                    // tile coordinates of this CTA inside its GEMM
};
struct GemmGroupPlan {
    GemmGroupEntry* entries_dev;
    int n, smem_bytes, n_gemms;
    int stateful;                  // the plans use the stateful SGD rule (all of them or none)
};
const char* gemm_group_plan(GemmGroupPlan* out, const GemmPlan* plans, int n_plans);
cudaError_t gemm_group_launch(const GemmGroupPlan& plan, cudaStream_t stream);
void gemm_group_free(GemmGroupPlan* plan);
cudaError_t gemm_configure();   // opt every instantiation into > 48 KB dynamic smem (call outside graph capture)
int gemm_kernel_count();   // number of launches issued so far by this module (bench accounting)

// ---- fused data-parallel path (csrc/kernels/fused_dp.cu) ---------------------------------
static constexpr int kMaxDp = 8;
struct DpPeers {                 // symmetric-memory pointer tables (index = DP rank)
    float* W[kMaxDp];            // weight arenas (owners publish updated tiles into every replica)
    float* stage[kMaxDp];        // partial-gradient staging: [src][layer slots]
    uint32_t* arrive[kMaxDp];    // arrive[owner][src * slots_per_src + slot] = epoch when src's partial landed
    uint32_t* done[kMaxDp];      // done[rank][tile] = epoch when the tile's new weights landed on rank
};
struct DpLayerParams {
    int m_total, n_total, k_total;   // out, in, micro-batch rows
    int block_n, stages;
    int n_tiles_m, n_tiles_n;
    int dp, rank;
    int64_t w_offset;                // float offset of the layer's [out, ld] block in the arena
    int ldw;
    int64_t stage_offset;            // float offset of the layer's slots inside one src region
    int64_t stage_src_stride;        // floats per src region
    int tile_flag_base, slot_flag_base, slots_per_src;
    const float* lr;                 // device float: learning rate of the running step
    const uint32_t* epoch_ptr;       // device step counter (bumped once per step, same value on all ranks)
    const float* G;                  // dp_reduce_sgd: accumulated gradient block to reduce
    int ldg;
    // one_shot: small (latency-bound) layers - every replica pushes its partial tile to ALL replicas
    // and every replica reduces every tile itself in the same fixed rank order (bit-identical results,
    // one NVLink hop instead of two).  Staging is double-buffered by epoch parity (stage_parity_stride).
    int one_shot;
    int64_t stage_parity_stride;
    int split;                       // 3xTF32 products (lo parts derived from the staged dZ / X tiles)
    int helpers;                     // CTAs per tile: CTA 0 computes + pushes, all of them share the reduce rows
    int bulk_push;                   // 1: push tiles with cp.async.bulk (TMA engine), 0: coalesced st.global
    unsigned long long* dbg;         // optional: 8 globaltimer stamps of CTA 0 (phase timeline)
    SgdState opt;                    // update rule; opt.V = this replica's LOCAL momentum arena (the owner's copy is the
                                     // canonical one: tile t's momentum lives at rank t % dp, every rank's with one_shot)
};
struct FusedDpPlan {
    CUtensorMap tmA, tmB;
    DpLayerParams p;
    DpPeers peers;
    int grid;
    int smem_bytes;
};
// Which replica owns (reduces, updates, keeps the momentum of) each parameter element under the DP protocol a layer
// runs: DP_PROTO_ALL = every replica (single replica, NCCL all-reduce, one-shot fused layers), LL = tile row r at rank
// r / (128 / dp), TWO_SHOT = tile t at rank t % dp (bias with tile column 0), NVLS = float4 chunk c of the arena at
// rank c % dp.  Element (m, n) of the layer's [out, ld] block at arena offset `offset`, n <= in (n == in: bias).
// Returns the rank, or -1 for every replica.  Host only.
enum DpProto : int { DP_PROTO_ALL = 0, DP_PROTO_LL = 1, DP_PROTO_TWO_SHOT = 2, DP_PROTO_NVLS = 3 };
int dp_element_owner(int proto, int in, int out, int ld, int64_t offset, int dp, int m, int n);
void dp_layer_geometry(int in, int out, int dp, int* block_n, int* n_tiles_m, int* n_tiles_n, int64_t* slots,
                       int64_t* slot_floats, int one_shot);
// dZ == nullptr: plan for dp_reduce_sgd (no GEMM)
const char* fused_dp_plan(FusedDpPlan* plan, const float* dZ, int lddz, const float* X, int ldx, int rows,
                          const DpLayerParams& lp, const DpPeers& peers, int max_ctas, bool split = false);
cudaError_t fused_dp_configure();
cudaError_t launch_fused_wgrad_dp(const FusedDpPlan& plan, cudaStream_t stream);
cudaError_t launch_dp_reduce_sgd(const FusedDpPlan& plan, cudaStream_t stream);
cudaError_t launch_bump_epoch(uint32_t* epoch, cudaStream_t stream);

// ---- LL two-shot fused DP path for narrow layers (csrc/kernels/dp_ll.cu): all layers of a stage in ONE launch
struct DpLLEntry {               // one CTA = one [128 x 32] tile of one layer's weight gradient
    CUtensorMap tmA, tmB;        // dZ (MN-major A), X (MN-major B)
    int m0, n0;                  // tile origin in (out, in)
    int m_total, n_total, k_total;
    int split, has_bias;
    int tile;                    // index in the landing zones
    int64_t w_offset;            // float offset of the layer's [out, ld] block in the arena
    int ldw;
    const uint32_t* gate_flag;   // chain-kernel counter the GEMM waits for: dz[l] final (nullptr: ordered by the stream instead)
    const uint32_t* gate_w;      // counter the in-place weight update waits for: dgrad of layer l consumed W_l (nullptr: none)
    uint32_t gate_mult;
};
struct DpLLParams {
    int dp, rank;
    const float* lr;             // device float: learning rate of the running step
    const uint32_t* epoch_ptr;   // DP step counter (same value on every replica)
    const uint32_t* gate_step;   // steps of the launching engine (gate target = gate_mult * *gate_step)
    int n_tiles, stages;
    float* W;                    // local weight arena
    uint4* llA[kMaxDp];          // reduce-scatter landing zones  [parity][src][tile][128 / dp rows][17 lines]
    uint4* llC[kMaxDp];          // all-gather landing zones      [parity][tile][128 rows][17 lines]
    unsigned long long* dbg;     // optional phase timeline: 8 globaltimer stamps per tile (first 28 tiles)
    SgdState opt;                // update rule; opt.V = LOCAL momentum arena, read / written only for the rows this rank owns
};
struct DpLLLayer {
    const float *dZ, *X;
    int split;                   // 3xTF32 products
    int lddz, ldx, in, out, ldw;
    int64_t w_offset;
    const uint32_t* gate_flag;
    const uint32_t* gate_w;
    uint32_t gate_mult;
};
struct DpLLPlan {
    DpLLParams p;
    DpLLEntry* entries_dev;
    int grid, smem_bytes;
};
int dp_ll_tiles(int in, int out);
size_t dp_ll_zone_lines(int dp, int n_tiles);
const char* dp_ll_plan(DpLLPlan* plan, const DpLLLayer* layers, int n_layers, int rows, const DpLLParams& base);
void dp_ll_free(DpLLPlan* plan);
cudaError_t dp_ll_configure();
cudaError_t launch_dp_ll(const DpLLPlan& plan, cudaStream_t stream);

// ---- layer-chain kernel (csrc/kernels/mlp_chain.cu) --------------------------------------
static constexpr int kChainMaxLayers = 16;
struct ChainLayer {
    int in, out, relu, ldw;
    int64_t w_off;                   // float offset of the [out, ld] block in the weight arena
};
struct ChainParams {
    int n_layers;
    ChainLayer layers[kChainMaxLayers];
    const CUtensorMap* maps;         // device array: [2l] W_l K-major (fwd), [2l+1] W_l MN-major (dgrad), [2L] X
    int split;                       // 3xTF32 (fp32-equivalent) products
    const float* W;                  // weight arena (bias reads)
    float* act[kChainMaxLayers + 1]; // act[0] = stage input, act[l] = output of layer l  ([all rows, ld])
    float* dz[kChainMaxLayers + 1];  // dz[l] = gradient w.r.t. the pre-activation of layer l (dz[0]: stage input grad)
    int act_ld[kChainMaxLayers + 1];
    const float* target;             // [all rows, ldt] one-hot targets (last stage)
    int ldt;
    float* probs;                    // [all rows, ldp]
    int ldp;
    float* loss;                     // [n_mubatches]
    int mb_rows, n_pad, stages;
    int kps;                         // 32-wide k-blocks per pipeline stage (one wait / one commit per stage)
    int cluster;                     // CTAs per micro-batch (thread-block cluster; 1 = one CTA owns the micro-batch)
    int mu_base;                     // first micro-batch handled by CTA 0 (per-micro-batch launches)
    float inv_batch;
    int do_fwd, do_loss, do_bwd, first_stage;
    // Pipeline boundaries folded into the kernel (peer-memory transport, one launch = one micro-batch of a stage):
    //  * in_flag  != nullptr: the tile this launch consumes (activations of the previous stage for a forward launch, output
    //    gradients of the next stage for a backward launch) is final in local memory once *in_flag >= *pp_epoch; the
    //    epilogue warps wait for it and stage the tile into shared memory - weights stream in meanwhile;
    //  * x_from_global: forward launch of a stage > 0: the input tile is read from act[0] by the epilogue warps (after the
    //    flag) instead of by TMA next to layer 1's weights;
    //  * out_peer != nullptr: the tile this launch produces for the neighbour (last forward output / dz[0]) is ALSO stored
    //    into the neighbour's receive slot, then one system fence + *out_flag = epoch; *out_credit >= epoch - 1 (the
    //    neighbour released its slots of the previous step) is awaited first.
    const uint32_t* in_flag;
    const uint32_t* pp_epoch;
    int x_from_global;
    float* out_peer;
    uint32_t* out_flag;
    const uint32_t* out_credit;
    int sync_debug;                  // SSB_RACECHECK=1: one more named barrier among the math warps per layer (racecheck aid
                                     // for the reuse of the activation ping-pong tiles)
    uint32_t* ready;                 // optional [n_layers + 1] device counters: every epilogue warp of every CTA adds 1 to
                                     // ready[l] once its part of dz[l] (and everything it wrote before) is globally visible
    unsigned long long* dbg;         // optional timeline buffer (3 roles x 256 globaltimer stamps), CTA 0 only
    // LossKind of the loss head (selects the kernel instantiation; probs are the row softmax under CROSS_ENTROPY).  Last,
    // so that the offsets of the other parameters are what they were before the field existed.
    int loss_kind;
};
struct ChainPlan {
    ChainParams p;
    CUtensorMap* maps_dev;
    int grid, smem_bytes;
    int cluster;                     // CTAs per micro-batch (grid = micro-batches x cluster)
};
bool chain_eligible(const ChainLayer* layers, int n_layers, int mb_rows, int out_dim, bool has_loss, bool split = false);
const char* chain_plan(ChainPlan* plan, const ChainParams& params, const float* x, int ldx, int total_rows, int n_mubatches,
                       bool split = false);
bool chain_budget(int mb_rows, bool split, int* kps, int* stages, int* smem_bytes);   // host arithmetic only
// Cluster plan of one chain launch (host arithmetic only).  chain_cluster_size: CTAs per micro-batch, ceil(w / 32) for the
// widest tile w the launch writes into shared memory (every forward output, every dgrad output, and dZ_L when a
// backward-only launch stages it), and 1 for launches gated for a co-resident consumer or with folded pipeline
// boundaries.  chain_cluster_budget: the shared-memory plan at that size (chain_budget's when cluster == 1).
int chain_cluster_size(const ChainLayer* layers, int n_layers, bool do_fwd, bool do_loss, bool do_bwd, bool first_stage,
                       bool gated, bool folded);
bool chain_cluster_budget(int mb_rows, int cluster, bool split, int* kps, int* stages, int* smem_bytes);
void chain_plan_free(ChainPlan* plan);
cudaError_t chain_configure();
cudaError_t chain_launch(const ChainPlan& plan, cudaStream_t stream);

// ---- small fused kernels --------------------------------------------------------------
// logits[rows, cols] (ld) -> probs (nullable) ; training: dlogits (softmax-Jacobian x MSE
// grad, 1/batch_size inside) and loss_out[0] = sum((t-p)^2)/batch_size.
// loss == LOSS_CROSS_ENTROPY: probs = row softmax; training: dlogits = (p * sum(t) - t)/batch_size and
// loss_out[0] = sum(t * ((max - z) + log s))/batch_size (ptx.cuh: ce_*).  Other values: cudaErrorInvalidValue.
cudaError_t launch_loss_head(const float* logits, int ldl, const float* target, int ldt, float* probs, int ldp,
                             float* dlogits, int ldd, float* loss_out, int rows, int cols, float inv_batch,
                             cudaStream_t stream, int rows_per_mubatch = 0,    // >0: one CTA per micro-batch, loss_out[mu]
                             int loss = LOSS_MSE);
// generic softmax backward for the functional API: dz = p*up - p*sum(p*up)
cudaError_t launch_softmax_grad(const float* logits, int ldl, const float* upstream, int ldu, float* dlogits, int ldd,
                                int rows, int cols, cudaStream_t stream);
// g[r, c] = y[r, c] > 0 ? g[r, c] : 0   (stage-boundary ReLU backward)
cudaError_t launch_relu_mask(float* g, int ldg, const float* y, int ldy, int rows, int cols, cudaStream_t stream);
cudaError_t launch_relu_fwd(const float* x, float* y, long n, cudaStream_t stream);
// y = a * x + b * t  (mse grad: a=2/B, b=-2/B)
cudaError_t launch_axpby(const float* x, const float* t, float* y, float a, float b, long n, cudaStream_t stream);
// w -= *lr * g over a flat arena (lr: one device float, read when the kernel runs)
cudaError_t launch_sgd(float* w, const float* g, const float* lr, long n, cudaStream_t stream);
// the same pass with the stateful rule (momentum buffer opt.V over the same n elements, weight decay, Nesterov)
cudaError_t launch_sgd_momentum(float* w, const float* g, const float* lr, const SgdState& opt, long n, cudaStream_t stream);
// correct[0] += #rows with argmax(pred) == argmax(target)
cudaError_t launch_argmax_correct(const float* pred, int ldp, const float* target, int ldt, int rows, int cols,
                                  int* correct, cudaStream_t stream);

}  // namespace ssb
