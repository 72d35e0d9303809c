// Native pipeline executor: lowers a stage's instruction stream (the Python Schedule IR)
// ONCE into a static plan of kernel launches / NCCL ops on CUDA streams with event
// dependencies, optionally captured into a CUDA graph, then replays it every step.
//
// This is the native replacement of the reference's Python `Worker.execute` loop
// (shallowspeed/pipe.py:434-466), which re-allocates buffers and re-dispatches Python
// objects for every batch.  Differences that matter for performance:
//   * persistent, pre-planned buffers + prebuilt TMA tensor maps (zero per-step host work
//     besides one cudaGraphLaunch);
//   * micro-batches are independent until the optimizer step, so each runs on its own
//     stream; wgrad GEMMs run on side streams in a fixed accumulation order (bitwise
//     deterministic); the graph exposes all of that parallelism to the hardware;
//   * ZeroGrad is free (first wgrad of a layer overwrites), OptimizerStep is fused into the
//     last wgrad of each layer (single replica) or into the in-kernel DP reduction;
//   * pipeline p2p uses NCCL send/recv on a dedicated stream, grouped exactly like the
//     schedule validator's rendezvous model.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <functional>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "kernels/kernels.h"
#include "runtime/dp_context.h"
#include "runtime/nvls_context.h"
#include "runtime/pp_context.h"

struct ncclComm;
typedef struct ncclComm* ncclComm_t;

namespace ssb {

struct LayerSpec {
    int in, out;
    int relu;
    int64_t offset;   // float offset of the [out, ld] block inside the W / G arenas
    int ld;           // row pitch of the block (floats); bias lives in column `in`
};

enum OpKind : int {
    OP_GEMM = 0, OP_LOSS_HEAD, OP_SOFTMAX, OP_RELU_MASK, OP_SGD, OP_COMM_GROUP, OP_ALLREDUCE, OP_FUSED_DP,
    OP_WAIT, OP_RECORD, OP_MEMCPY_LOSS, OP_ARGMAX, OP_DP_REDUCE, OP_BUMP_EPOCH, OP_CHAIN, OP_NVLS_SGD,
    OP_PP_PUSH, OP_PP_WAIT, OP_PP_CREDIT, OP_PP_BUMP, OP_WGRAD_GROUP, OP_BUMP_STEP, OP_DP_LL
};

struct CommItem {   // one send or recv inside a group
    int is_send;
    int peer;       // rank inside the pp communicator
    float* ptr;
    size_t count;
};

struct Op {
    int kind = 0;
    int stream = 0;
    int event = -1;            // OP_WAIT / OP_RECORD
    int gemm = -1;             // index into gemm plans
    int layer = -1, mu = -1;
    std::vector<CommItem> comm;
    // generic pointers for the small kernels
    float *a = nullptr, *b = nullptr, *c = nullptr, *d = nullptr;
    float* f = nullptr;        // loss head: where the loss values go when not the default device scratch
    int lda = 0, ldb = 0, ldc = 0, ldd = 0, rows = 0, cols = 0;
    float scalar = 0.f;
    const float* lr = nullptr; // OP_SGD / OP_NVLS_SGD: the learning-rate slot of the op's staging set
    int64_t n = 0;
};

struct EngineConfig {
    std::vector<LayerSpec> layers;
    int is_first = 1, is_last = 1;
    int stage = 0, n_stages = 1;
    int mb_rows = 32;       // rows per micro-batch
    int n_mu = 4;           // micro-batches per step (training) / per call (inference)
    int global_batch = 128; // for the 1/B loss scale
    float lr = 0.006f;      // initial learning rate (set_lr changes it between steps)
    int training = 1;
    int use_graph = 1;
    int dp_size = 1, dp_rank = 0;
    int dp_mode = 0;        // 0 = none/fused-sgd (dp=1), 1 = NCCL all-reduce + SGD, 2 = fused in-kernel reduction,
                            // 3 = NVLS: one kernel reduces the gradient arena in the switch, applies SGD, multicasts W
    int in_dim = 784, out_dim = 10;
    int split = 0;          // 1 = fp32-equivalent tensor-core products (3xTF32), 0 = single-pass TF32
    // SGD beyond lr (torch.optim.SGD, dampening 0).  All zero = plain SGD and the stateless kernels.  Momentum needs
    // the engine's momentum arena (same layout as the weights); under the in-kernel DP reductions (dp_mode 2, 3) each
    // replica updates only the entries it owns (layer_protocols()).
    float momentum = 0.f, weight_decay = 0.f;
    int nesterov = 0;
    int loss = LOSS_MSE;    // LossKind of the last stage's head (the chain kernel's and loss_head_kernel's)
};

class PipeEngine {
public:
    // momentum: flat momentum arena (arena_numel floats, the weights' offsets), nullptr unless cfg.momentum > 0
    explicit PipeEngine(const EngineConfig& cfg, float* weights, float* grads, int64_t arena_numel, float* momentum = nullptr);
    ~PipeEngine();

    // communicators (optional): created by the caller from ncclUniqueIds exchanged over torch.distributed
    void set_pp_comm(ncclComm_t comm) { pp_comm_ = comm; }
    void set_dp_comm(ncclComm_t comm) { dp_comm_ = comm; }
    void set_dp_context(DpContext* ctx) { dp_ctx_ = ctx; }   // fused in-kernel DP reduction (dp_mode 2)
    void set_nvls_context(NvlsContext* ctx) { nvls_ctx_ = ctx; }   // switch-side reduction (dp_mode 3)
    void set_pp_context(PpContext* ctx) { pp_ctx_ = ctx; }         // pipeline boundaries over peer memory instead of NCCL p2p

    // instrs: (opcode, buffer_id, mubatch_id) triples from parallel.instructions.encode
    void build(const std::vector<std::tuple<int, int, int>>& instrs);

    // input staging ------------------------------------------------------------------
    // dense row-major host/device sources: x [n_mu*mb_rows, in_dim], y [n_mu*mb_rows, out_dim]
    void stage_inputs(const float* x, const float* y);
    void run();                       // one step (graph launch or eager plan walk) on the main stream
    // learning rate of the steps run from now on.  Every update op reads it from the device slot of its staging set;
    // run() rewrites that slot on the copy stream only when it holds a different value.
    void set_lr(float lr) { lr_ = lr; }
    float lr() const { return lr_; }
    void synchronize();
    bool wait(double timeout_s);      // watchdog: false if the step in flight did not finish in time
    std::string comm_status() const;  // NCCL async error state of the attached communicators
    // SSB_COMM_TIMING=1: (ms the compute streams stalled on communication, ms the comm ops were busy) of the last step
    std::pair<double, double> comm_timing();
    bool comm_timing_enabled() const { return comm_timing_; }
    float last_loss();                // sum of the micro-batch losses of the most recent step (synchronizes)
    float prev_loss();                // loss of the step before the most recently launched one (pipelined readback)
    int count_correct();              // inference: # argmax matches accumulated since reset
    void reset_correct();

    // introspection
    float* act_ptr(int mu, int l) { return act_[mu][l]; }
    int act_ld(int l) const { return act_ld_[l]; }
    float* dz_ptr(int mu, int l) { return dz_[mu][l]; }
    float* probs_ptr(int mu) { return probs_[mu]; }
    float* x_staging() { return x_stage_; }
    float* y_staging() { return y_stage_; }
    int y_ld() const { return y_ld_; }
    int64_t kernels_per_step() const { return kernels_per_step_; }
    int64_t graph_nodes() const { return graph_nodes_; }
    bool coalesced() const { return coalesced_; }
    bool uses_chain() const { return chain_ok_; }
    // CTAs per micro-batch of the chain launches (the largest over the plan; 0 without chain launches)
    int chain_cluster() const {
        int c = 0;
        for (const ChainPlan& cp : chain_plans_) c = std::max(c, cp.cluster);
        return c;
    }
    cudaStream_t main_stream() { return streams_[0]; }
    const EngineConfig& config() const { return cfg_; }
    // per layer: the DpProto under which its update runs (which replica owns which momentum entries)
    const std::vector<int>& layer_protocols() const { return layer_proto_; }
    std::string describe() const;
    std::string plan_text(int set = 0) const;
    std::vector<unsigned long long> chain_timeline();   // SSB_CHAIN_TIMELINE=1: globaltimer stamps of the chain kernel

private:
    void alloc_buffers();
    void build_coalesced();
    void plan_per_mubatch();
    void select_set(int set);
    void finish_build();
    int new_event();
    float* loss_target() const;
    void maybe_splitk(GemmPlan& g);
    void emit_wait(int stream, int ev);
    int emit_record(int stream);
    void walk(int set);
    void exec(const Op& op);
    cudaStream_t stream_of(const Op& op) const;

    SgdState opt_for(int layer) const;   // the update rule for layer l's block (l = 0: the whole arena)
    EngineConfig cfg_;
    float *W_, *G_, *V_;
    std::vector<int> layer_proto_;
    int64_t arena_numel_;
    int L_;
    std::vector<int> act_ld_;                    // per layer boundary 0..L
    std::vector<std::vector<float*>> act_, dz_;  // [mu][l]
    std::vector<float*> probs_;
    std::vector<float*> act_all_, dz_all_;       // [l] contiguous over micro-batches
    bool gate_on_ = false;           // grouped wgrad forked next to the chain kernel, gated by device counters
    uint32_t* gate_ready_ = nullptr; // [L + 1] per-layer counters written by the chain kernel
    uint32_t* gate_step_ = nullptr;  // steps of THIS engine (bumped in front of the gated kernel)
    float* probs_all_ = nullptr;
    bool coalesced_ = false;
    float *x_stage_ = nullptr, *y_stage_ = nullptr, *loss_dev_ = nullptr, *loss_host_ = nullptr;
    int* correct_dev_ = nullptr;
    int y_ld_ = 0;
    std::vector<void*> owned_;

    std::vector<cudaStream_t> streams_;
    std::vector<cudaEvent_t> events_;
    std::vector<cudaEvent_t> timing_events_;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> exposed_pairs_, busy_pairs_;
    bool comm_timing_ = false;
    bool loss_zero_copy_ = false;
    std::vector<GemmPlan> gemms_;
    std::vector<FusedDpPlan> dp_plans_;
    std::vector<ChainPlan> chain_plans_;
    std::vector<GemmGroupPlan> group_plans_;
    std::vector<DpLLPlan> ll_plans_;
    bool chain_ok_ = false;
    unsigned long long* chain_dbg_ = nullptr;
    // pipeline boundaries folded into a chain launch (peer-memory transport), see ChainParams
    struct ChainFold {
        const uint32_t* in_flag = nullptr;
        bool x_from_global = false;
        float* out_peer = nullptr;
        uint32_t* out_flag = nullptr;
        const uint32_t* out_credit = nullptr;
    };
    int add_chain(int stream, int mu_base, int n_mu, bool do_fwd, bool do_loss, bool do_bwd, const ChainFold* fold = nullptr);
    DpContext* dp_ctx_ = nullptr;
    NvlsContext* nvls_ctx_ = nullptr;
    PpContext* pp_ctx_ = nullptr;
    std::vector<Op> ops_;
    std::vector<Op> ops_sets_[2];
    cudaGraph_t graph_sets_[2] = {nullptr, nullptr};
    cudaGraphExec_t graph_exec_sets_[2] = {nullptr, nullptr};
    float *x_stage_sets_[2] = {nullptr, nullptr}, *y_stage_sets_[2] = {nullptr, nullptr};
    // learning rate: one device float per staging set (lr_dev_[set]), the value last written to each, and the value the
    // next step runs with
    float* lr_dev_ = nullptr;
    float lr_written_[2] = {0.f, 0.f};
    float lr_ = 0.f;
    const float* lr_slot() const { return lr_dev_ + cur_set_; }
    cudaStream_t copy_stream_ = nullptr;
    cudaEvent_t ev_copy_[2], ev_done_[2];
    int fill_set_ = 0, run_set_ = 0, cur_set_ = 0;
    bool staged_ = false;
    std::vector<std::tuple<int, int, int>> instrs_;
    std::vector<int> mu_of_;
    int64_t kernels_per_step_ = 0, graph_nodes_ = 0;
    int kernels_extra_ = 0;
    int splitk_gemms_ = 0;
    ncclComm_t pp_comm_ = nullptr, dp_comm_ = nullptr;
    int n_mu_streams_ = 1, n_w_streams_ = 1;
    int s_comm_ = 0, s_dp_ = 0;
    bool built_ = false;
};

}  // namespace ssb
