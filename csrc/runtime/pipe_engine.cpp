#include "runtime/pipe_engine.h"

#include <nccl.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <chrono>
#include <thread>
#include <cstdlib>
#include <cstring>
#include <sstream>
#include <stdexcept>

namespace ssb {

#define CUDA_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t _e = (expr);                                                                           \
        if (_e != cudaSuccess)                                                                             \
            throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr); \
    } while (0)
#define NCCL_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        ncclResult_t _r = (expr);                                                                          \
        if (_r != ncclSuccess)                                                                             \
            throw std::runtime_error(std::string("NCCL error: ") + ncclGetErrorString(_r) + " at " #expr); \
    } while (0)

// opcodes of shallowspeed_b200/parallel/instructions.py
enum : int {
    I_ZERO_GRAD = 0, I_OPT_STEP = 1, I_RECV_ACT = 2, I_SEND_ACT = 3, I_RECV_GRAD = 4, I_SEND_GRAD = 5,
    I_FORWARD = 6, I_BWD_ACC = 7, I_BWD_AR = 8, I_LOAD_X = 9, I_LOAD_Y = 10
};

static int round_up(int x, int m) { return (x + m - 1) / m * m; }

// cuMemsetD32Async, reached through the runtime so that the extension does not link libcuda (as in nvls_context.cpp):
// writes the learning-rate slot by value.
using MemsetD32AsyncFn = CUresult (*)(CUdeviceptr, unsigned int, size_t, CUstream);
static MemsetD32AsyncFn memset_d32_async() {
    static MemsetD32AsyncFn fn = [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemsetD32Async", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess || ptr == nullptr)
            throw std::runtime_error("PipeEngine: driver entry point cuMemsetD32Async not available");
        return reinterpret_cast<MemsetD32AsyncFn>(ptr);
    }();
    return fn;
}
static void cu_check(CUresult r, const char* what) {
    if (r != CUDA_SUCCESS) throw std::runtime_error(std::string("PipeEngine: ") + what + " failed (" + std::to_string((int)r) + ")");
}
// leave some SMs to the concurrently running dgrad chain; also bounds co-residency needs
static constexpr int kFusedDpMaxCtas = 120;

PipeEngine::PipeEngine(const EngineConfig& cfg, float* weights, float* grads, int64_t arena_numel, float* momentum, float* ema)
    : cfg_(cfg), W_(weights), G_(grads), V_(momentum), E_(ema), arena_numel_(arena_numel), L_((int)cfg.layers.size()) {
    if ((cfg_.ema_decay > 0.f) != (E_ != nullptr)) throw std::runtime_error("PipeEngine: an EMA arena is needed exactly when ema_decay > 0");
    if (!(cfg_.ema_decay >= 0.f && cfg_.ema_decay < 1.f)) throw std::runtime_error("PipeEngine: ema_decay must be 0 (no EMA) or in (0, 1)");
    SgdState opt = opt_for(0);
    opt.E = nullptr;                                      // the rule alone: the EMA alpha slot does not exist yet
    if (const char* e = sgd_state_check(opt)) throw std::runtime_error(std::string("PipeEngine: ") + e);
    // who owns which momentum entries: every replica unless a layer's update runs in an owner-based DP reduction
    layer_proto_.assign(L_, (cfg_.training && cfg_.dp_mode == 3 && cfg_.dp_size > 1) ? DP_PROTO_NVLS : DP_PROTO_ALL);
    n_mu_streams_ = std::max(1, std::min(cfg_.n_mu, 8));   // one stream per micro-batch in flight (GPipe with 8 micro-batches: all 8)
    n_w_streams_ = std::max(1, std::min(L_, 8));        // one stream per layer's wgrad when possible
    const int n_streams = 1 + n_mu_streams_ + n_w_streams_ + 2;
    s_comm_ = 1 + n_mu_streams_ + n_w_streams_;
    s_dp_ = s_comm_ + 1;
    streams_.resize(n_streams);
    for (auto& s : streams_) CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        CUDA_CHECK(cudaEventCreateWithFlags(&ev_copy_[i], cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&ev_done_[i], cudaEventDisableTiming));
    }
    alloc_buffers();
}

SgdState PipeEngine::opt_for(int layer, int set) const {
    SgdState s;
    s.momentum = cfg_.momentum; s.weight_decay = cfg_.weight_decay; s.nesterov = cfg_.nesterov;
    if (V_ != nullptr) s.V = V_ + (layer >= 1 ? cfg_.layers[layer - 1].offset : 0);
    if (ema_on()) {
        s.E = E_ + (layer >= 1 ? cfg_.layers[layer - 1].offset : 0);
        s.ema_alpha = alpha_dev_ + (set >= 0 ? set : cur_set_);
    }
    return s;
}

PipeEngine::~PipeEngine() {
    cudaDeviceSynchronize();
    for (int i = 0; i < 2; ++i) {
        if (graph_exec_sets_[i]) cudaGraphExecDestroy(graph_exec_sets_[i]);
        if (graph_sets_[i]) cudaGraphDestroy(graph_sets_[i]);
        cudaEventDestroy(ev_copy_[i]);
        cudaEventDestroy(ev_done_[i]);
    }
    cudaStreamDestroy(copy_stream_);
    for (auto e : events_) cudaEventDestroy(e);
    for (auto e : timing_events_) cudaEventDestroy(e);
    for (auto s : streams_) cudaStreamDestroy(s);
    for (auto& cp : chain_plans_) chain_plan_free(&cp);
    for (auto& gp : group_plans_) gemm_group_free(&gp);
    for (auto& lp : ll_plans_) dp_ll_free(&lp);
    for (auto p : owned_) cudaFree(p);
    if (loss_host_) cudaFreeHost(loss_host_);
}

void PipeEngine::alloc_buffers() {
    const int M = cfg_.n_mu, mb = cfg_.mb_rows;
    act_ld_.resize(L_ + 1);
    act_ld_[0] = round_up(L_ > 0 ? cfg_.layers[0].in : cfg_.in_dim, 8);
    for (int l = 1; l <= L_; ++l) act_ld_[l] = round_up(cfg_.layers[l - 1].out, 8);
    auto dalloc = [&](size_t floats) {
        float* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(floats, 64) * sizeof(float)));
        CUDA_CHECK(cudaMemset(p, 0, std::max<size_t>(floats, 64) * sizeof(float)));
        owned_.push_back(p);
        return p;
    };
    // stage input of all micro-batches is ONE buffer so a step needs a single (2-D) copy
    y_ld_ = round_up(cfg_.out_dim, 8);
    for (int set = 0; set < 2; ++set) {
        x_stage_sets_[set] = dalloc((size_t)M * mb * act_ld_[0]);
        y_stage_sets_[set] = dalloc((size_t)M * mb * y_ld_);
    }
    x_stage_ = x_stage_sets_[0];
    y_stage_ = y_stage_sets_[0];
    lr_dev_ = dalloc(2);
    lr_ = lr_written_[0] = lr_written_[1] = cfg_.lr;
    const float lr_init[2] = {cfg_.lr, cfg_.lr};
    CUDA_CHECK(cudaMemcpy(lr_dev_, lr_init, sizeof(lr_init), cudaMemcpyHostToDevice));
    if (ema_on()) {
        alpha_dev_ = dalloc(2);
        const float alpha_init[2] = {alpha_, alpha_};
        CUDA_CHECK(cudaMemcpy(alpha_dev_, alpha_init, sizeof(alpha_init), cudaMemcpyHostToDevice));
    }
    if (dropout_on()) {
        step_dev_ = reinterpret_cast<uint32_t*>(dalloc(2));   // zeroed: step 0
        step_ = step_written_[0] = step_written_[1] = 0u;
    }
    // the loss head stores its per-micro-batch losses straight into this pinned, device-mapped host buffer (16 bytes over
    // PCIe): no D2H copy node in the step
    CUDA_CHECK(cudaMallocHost(&loss_host_, 2 * sizeof(float) * loss_stride()));   // one slot per staging set
    for (int i = 0; i < 2 * loss_stride(); ++i) loss_host_[i] = 0.f;
    {
        int* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, 64));
        CUDA_CHECK(cudaMemset(p, 0, 64));
        owned_.push_back(p);
        correct_dev_ = p;
    }
    // one contiguous [M * mb, ld] buffer per layer boundary: micro-batch mu owns rows
    // [mu*mb, (mu+1)*mb).  A stage without pipeline communication runs ALL micro-batches of a
    // layer in one launch (horizontal fusion); otherwise each micro-batch uses its row slice.
    act_all_.assign(L_ + 1, nullptr);
    dz_all_.assign(L_ + 1, nullptr);
    act_all_[0] = x_stage_;
    for (int l = 1; l <= L_; ++l) act_all_[l] = dalloc((size_t)M * mb * act_ld_[l]);
    if (cfg_.training)
        for (int l = 0; l <= L_; ++l) dz_all_[l] = dalloc((size_t)M * mb * act_ld_[l]);
    probs_all_ = dalloc((size_t)M * mb * act_ld_[L_]);
    if (gated()) {
        gamma_all_.assign(L_ + 1, nullptr);
        for (int l = 1; l <= L_; ++l)
            if (cfg_.layers[l - 1].relu) gamma_all_[l] = dalloc((size_t)M * mb * act_ld_[l]);
        gamma_.assign(M, std::vector<float*>(L_ + 1, nullptr));
        for (int mu = 0; mu < M; ++mu)
            for (int l = 1; l <= L_; ++l)
                if (gamma_all_[l]) gamma_[mu][l] = gamma_all_[l] + (size_t)mu * mb * act_ld_[l];
    }
    if (cfg_.training && cfg_.residual) {
        gres_all_.assign(L_ + 1, nullptr);
        for (int l = 1; l <= L_; ++l)
            if (res_layer(l)) gres_all_[l] = dalloc((size_t)M * mb * act_ld_[l]);
        gres_.assign(M, std::vector<float*>(L_ + 1, nullptr));
        for (int mu = 0; mu < M; ++mu)
            for (int l = 1; l <= L_; ++l)
                if (gres_all_[l]) gres_[mu][l] = gres_all_[l] + (size_t)mu * mb * act_ld_[l];
    }
    act_.assign(M, std::vector<float*>(L_ + 1, nullptr));
    dz_.assign(M, std::vector<float*>(L_ + 1, nullptr));
    probs_.assign(M, nullptr);
    for (int mu = 0; mu < M; ++mu) {
        for (int l = 0; l <= L_; ++l) {
            act_[mu][l] = act_all_[l] + (size_t)mu * mb * act_ld_[l];
            if (cfg_.training) dz_[mu][l] = dz_all_[l] + (size_t)mu * mb * act_ld_[l];
        }
        probs_[mu] = probs_all_ + (size_t)mu * mb * act_ld_[L_];
    }
}

DropoutSpec PipeEngine::drop_for(int layer, int row_base) const {
    if (!dropout_on() || !cfg_.layers[layer - 1].relu) return DropoutSpec{};
    DropoutSpec d = dropout_spec(cfg_.dropout, cfg_.dropout_seed);
    d.step = step_dev_ + cur_set_;
    d.layer = cfg_.layer_base + layer - 1;
    d.row_base = row_base;
    d.dp = cfg_.dp_size;
    d.rank = cfg_.dp_rank;
    return d;
}

float* PipeEngine::gamma_of(const float* act) const {
    const size_t rows = (size_t)cfg_.n_mu * cfg_.mb_rows;
    for (int l = 1; l <= L_; ++l)
        if (gamma_all_[l] != nullptr && act >= act_all_[l] && act < act_all_[l] + rows * act_ld_[l])
            return gamma_all_[l] + (act - act_all_[l]);
    throw std::runtime_error("PipeEngine: no gate buffer behind an activated layer's output");
}

// A smooth activation runs the gated GEMM variants: a FWD with relu applies f (and, training, stores its gates next to
// its output), a DGRAD with mask multiplies by the previous layer's gates instead of testing its output.
void PipeEngine::gate_gemm(GemmPlan& g) const {
    if (!act_smooth(cfg_.activation) && !cfg_.residual) return;   // a residual model gates ReLU too
    g.p.act_kind = cfg_.activation;
    if (!gated()) return;                                         // inference: f, no gates
    if (g.mode == GEMM_FWD && g.p.relu) g.p.gate = gamma_of(g.p.out);
    else if (g.mode == GEMM_DGRAD && g.p.mask != nullptr) g.p.mask = gamma_of(g.p.mask);
}

// A residual plan's FWD / DGRAD of layer l (mu: its micro-batch, -1 for all rows) runs the residual GEMM form where it adds a
// skip, stores a skip gradient, or applies a ReLU gate (gated(): every activated layer of a residual training plan).
//   FWD of a residual layer:  + act[l - 1] (for l = 1 the staged stage input or the received tile)
//   DGRAD of layer l:         + g[l] when layer l is residual; stores g[l - 1] (before the gate) when layer l - 1 is
//                             residual
void PipeEngine::skip_gemm(GemmPlan& g, int l, int mu) const {
    if (!cfg_.residual) return;
    auto act = [&](int k) { return mu >= 0 ? act_[mu][k] : act_all_[k]; };
    auto gres = [&](int k) { return mu >= 0 ? gres_[mu][k] : gres_all_[k]; };
    if (g.mode == GEMM_FWD) {
        if (res_layer(l)) { g.p.skip = act(l - 1); g.p.ldskip = act_ld_[l - 1]; }
        g.p.res = (g.p.skip != nullptr || (gated() && g.p.relu)) ? 1 : 0;
    } else if (g.mode == GEMM_DGRAD) {
        if (res_layer(l)) { g.p.skip = gres(l); g.p.ldskip = act_ld_[l]; }
        if (res_layer(l - 1)) { g.p.gpre = gres(l - 1); g.p.ldgpre = act_ld_[l - 1]; }
        g.p.res = (g.p.skip != nullptr || g.p.gpre != nullptr || g.p.mask != nullptr) ? 1 : 0;
        if ((res_layer(l) && g.p.skip == nullptr) || (res_layer(l - 1) && g.p.gpre == nullptr))
            throw std::runtime_error("PipeEngine: no skip-gradient buffer behind a residual layer");
    }
}

// Point the planner at one of the two input-staging sets (stage input = act[.][0], targets).
void PipeEngine::select_set(int set) {
    cur_set_ = set;
    x_stage_ = x_stage_sets_[set];
    y_stage_ = y_stage_sets_[set];
    act_all_[0] = x_stage_;
    for (int mu = 0; mu < cfg_.n_mu; ++mu) act_[mu][0] = act_all_[0] + (size_t)mu * cfg_.mb_rows * act_ld_[0];
}

// Automatic by default (gemm_splitk_choice); SSB_SPLITK=k forces k splits where legal, SSB_SPLITK=0 turns it off.  Gives
// FWD / DGRAD GEMMs of wide layers enough CTAs to saturate HBM (8192 outputs = only 64 tiles on 132 SMs).  Each plan
// owns its workspace and tile counters; the last CTA of a tile re-arms its counter, so every replay of the graph
// reuses them.  tests/test_gpu_gemm.py checks the variant per element against an fp64 oracle, stand-alone and in the
// engine over two steps.
void PipeEngine::maybe_splitk(GemmPlan& g) {
    const char* env = getenv("SSB_SPLITK");
    const int want = env ? atoi(env) : 1;
    if (want <= 0 || g.mode == GEMM_WGRAD) return;
    int dev = 0, sms = 132;
    CUDA_CHECK(cudaGetDevice(&dev));
    CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int splits = gemm_splitk_choice(g, sms);
    if (want > 1) {
        const int num_kb = (g.p.k_total + 31) / 32;
        const int per = (num_kb + want - 1) / want;
        if (per >= 1 && (num_kb + per - 1) / per == want) splits = want;
    }
    if (splits < 2) return;
    const size_t ws_floats = gemm_splitk_workspace_floats(g, splits);
    const size_t n_tiles = (size_t)g.grid.x * g.grid.y;
    float* ws = nullptr;
    unsigned int* counters = nullptr;
    CUDA_CHECK(cudaMalloc(&ws, ws_floats * sizeof(float)));
    owned_.push_back(ws);
    CUDA_CHECK(cudaMalloc(&counters, std::max<size_t>(n_tiles, 16) * sizeof(unsigned int)));
    CUDA_CHECK(cudaMemset(counters, 0, std::max<size_t>(n_tiles, 16) * sizeof(unsigned int)));
    owned_.push_back(counters);
    if (const char* err = gemm_plan_enable_splitk(&g, splits, ws, counters))
        throw std::runtime_error(std::string("PipeEngine split-K: ") + err);
    ++splitk_gemms_;
}

int PipeEngine::new_event() {
    cudaEvent_t e;
    CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    events_.push_back(e);
    return (int)events_.size() - 1;
}
void PipeEngine::emit_wait(int stream, int ev) {
    Op op;
    op.kind = OP_WAIT; op.stream = stream; op.event = ev;
    ops_.push_back(op);
}
int PipeEngine::emit_record(int stream) {
    Op op;
    op.kind = OP_RECORD; op.stream = stream; op.event = new_event();
    ops_.push_back(op);
    return op.event;
}

// One launch that walks micro-batches [mu_base, mu_base + n_mu) through the whole stage
// (csrc/kernels/mlp_chain.cu).  Returns the op index.
int PipeEngine::add_chain(int stream, int mu_base, int n_mu, bool do_fwd, bool do_loss, bool do_bwd, const ChainFold* fold) {
    ChainParams cp{};
    cp.n_layers = L_;
    for (int l = 0; l < L_; ++l) {
        const LayerSpec& ls = cfg_.layers[l];
        cp.layers[l].in = ls.in; cp.layers[l].out = ls.out; cp.layers[l].relu = ls.relu; cp.layers[l].ldw = ls.ld;
        cp.layers[l].w_off = ls.offset;
    }
    cp.W = W_;
    for (int l = 0; l <= L_; ++l) {
        cp.act[l] = act_all_[l];
        cp.dz[l] = cfg_.training ? dz_all_[l] : nullptr;
        cp.act_ld[l] = act_ld_[l];
    }
    cp.target = y_stage_; cp.ldt = y_ld_;
    cp.probs = probs_all_; cp.ldp = act_ld_[L_];
    cp.loss = loss_slot(cur_set_);
    cp.loss_kind = cfg_.loss;
    cp.act_kind = cfg_.activation;
    if (gated())
        for (int l = 0; l <= L_; ++l) cp.gate[l] = gamma_all_[l];
    if (cfg_.residual) {                                  // training and inference: the RES form adds the skips
        cp.res = 1;
        for (int l = 1; l <= L_; ++l)
            if (res_layer(l)) cp.res_mask |= 1u << (l - 1);
        // a residual last layer of a non-last stage: the received gradient stays in g[L], the staging gates it into dz[L]
        if (cfg_.training && do_bwd && !(do_fwd && do_loss) && res_layer(L_)) cp.gout = gres_all_[L_];
    }
    if (dropout_on()) {
        // one spec for the launch: the kernel drops only the ReLU'd layers, layer l's counter is drop.layer + l - 1
        cp.drop = dropout_spec(cfg_.dropout, cfg_.dropout_seed);
        cp.drop.step = step_dev_ + cur_set_;
        cp.drop.layer = cfg_.layer_base;
        cp.drop.dp = cfg_.dp_size;
        cp.drop.rank = cfg_.dp_rank;
    }
    cp.mb_rows = cfg_.mb_rows; cp.mu_base = mu_base;
    cp.inv_batch = 1.0f / (float)cfg_.global_batch;
    cp.do_fwd = do_fwd; cp.do_loss = do_loss; cp.do_bwd = do_bwd; cp.first_stage = cfg_.is_first;
    cp.dbg = nullptr;
    cp.sync_debug = (getenv("SSB_RACECHECK") && atoi(getenv("SSB_RACECHECK")) > 0) ? 1 : 0;
    if (fold != nullptr && pp_ctx_ != nullptr) {
        cp.in_flag = fold->in_flag; cp.x_from_global = fold->x_from_global ? 1 : 0;
        cp.out_peer = fold->out_peer; cp.out_flag = fold->out_flag; cp.out_credit = fold->out_credit;
        cp.pp_epoch = pp_ctx_->epoch_ptr();
    }
    cp.ready = (gate_on_ && do_bwd && do_fwd) ? gate_ready_ : nullptr;
    if (getenv("SSB_CHAIN_TIMELINE")) {
        if (!chain_dbg_) {
            CUDA_CHECK(cudaMalloc(&chain_dbg_, 4 * 256 * sizeof(unsigned long long)));
            CUDA_CHECK(cudaMemset(chain_dbg_, 0, 4 * 256 * sizeof(unsigned long long)));
            owned_.push_back(chain_dbg_);
        }
        cp.dbg = chain_dbg_;
    }
    ChainPlan plan;
    const char* err = chain_plan(&plan, cp, act_all_[0], act_ld_[0], cfg_.n_mu * cfg_.mb_rows, n_mu, cfg_.prec);
    if (err) throw std::runtime_error(std::string("PipeEngine chain plan: ") + err);
    chain_plans_.push_back(plan);
    Op op;
    op.kind = OP_CHAIN; op.stream = stream; op.gemm = (int)chain_plans_.size() - 1; op.mu = mu_base;
    ops_.push_back(op);
    return (int)ops_.size() - 1;
}

void PipeEngine::build(const std::vector<std::tuple<int, int, int>>& instrs) {
    if (built_) throw std::runtime_error("PipeEngine::build called twice");
    const int M = cfg_.n_mu, n = (int)instrs.size();

    // ---- resolve which micro-batch every comm instruction carries
    std::vector<int> mu_of(n, -1);
    for (int i = 0; i < n; ++i) {
        const int op = std::get<0>(instrs[i]), b = std::get<1>(instrs[i]);
        if (op == I_RECV_ACT || op == I_RECV_GRAD) {
            for (int j = i + 1; j < n; ++j) {
                const int oj = std::get<0>(instrs[j]);
                const bool match = (op == I_RECV_ACT) ? (oj == I_FORWARD) : (oj == I_BWD_ACC || oj == I_BWD_AR);
                if (match && std::get<1>(instrs[j]) == b) { mu_of[i] = std::get<2>(instrs[j]); break; }
            }
        } else if (op == I_SEND_ACT || op == I_SEND_GRAD) {
            for (int j = i - 1; j >= 0; --j) {
                const int oj = std::get<0>(instrs[j]);
                const bool match = (op == I_SEND_ACT) ? (oj == I_FORWARD) : (oj == I_BWD_ACC || oj == I_BWD_AR);
                if (match && std::get<1>(instrs[j]) == b) { mu_of[i] = std::get<2>(instrs[j]); break; }
            }
        } else {
            mu_of[i] = std::get<2>(instrs[i]);
        }
        if ((op >= I_RECV_ACT && op <= I_SEND_GRAD) && mu_of[i] < 0)
            throw std::runtime_error("PipeEngine: cannot resolve the micro-batch of a comm instruction");
        if (mu_of[i] >= M) throw std::runtime_error("PipeEngine: micro-batch id out of range");
    }

    bool has_comm = false;
    for (int i = 0; i < n; ++i) {
        const int op = std::get<0>(instrs[i]);
        if (op >= I_RECV_ACT && op <= I_SEND_GRAD) has_comm = true;
    }
    coalesced_ = !has_comm && !getenv("SSB_NO_COALESCE");
    {
        ChainLayer cl[kChainMaxLayers];
        const int nl = std::min(L_, (int)kChainMaxLayers);
        for (int l = 0; l < nl; ++l) { cl[l].in = cfg_.layers[l].in; cl[l].out = cfg_.layers[l].out; }
        chain_ok_ = L_ >= 1 && L_ <= kChainMaxLayers && !getenv("SSB_NO_CHAIN") &&
                    chain_eligible(cl, L_, cfg_.mb_rows, cfg_.out_dim, cfg_.is_last != 0, cfg_.prec);
    }
    if (chain_ok_ && !gres_all_.empty()) {
        // the chain kernel carries the skip gradients in registers: only a residual last layer of a non-last stage keeps
        // one, the gradient it receives
        for (int l = 1; l <= L_; ++l) {
            if (l == L_ && !cfg_.is_last) continue;
            gres_all_[l] = nullptr;
            for (int mu = 0; mu < M; ++mu) gres_[mu][l] = nullptr;
        }
    }
    if (pp_ctx_) {
        // peer-memory transport: the neighbours write straight into my receive slots, which therefore live in the
        // IPC-shared PpContext (one set of slots; reuse across steps is protected by the credit flags)
        if (pp_ctx_->n_mu() != M || pp_ctx_->mb_rows() != cfg_.mb_rows || pp_ctx_->ld_in() != act_ld_[0] || pp_ctx_->ld_out() != act_ld_[L_])
            throw std::runtime_error("PipeEngine: PpContext geometry does not match this stage");
        if (!cfg_.is_first) x_stage_sets_[0] = x_stage_sets_[1] = pp_ctx_->act_in();
        if (!cfg_.is_last && cfg_.training && res_layer(L_)) {
            // a residual last layer keeps the received gradient as its skip gradient g[L]; dz[L] = g[L] * gamma_L is its own
            gres_all_[L_] = pp_ctx_->dz_in();
            for (int mu = 0; mu < M; ++mu) gres_[mu][L_] = gres_all_[L_] + (size_t)mu * cfg_.mb_rows * act_ld_[L_];
        } else if (!cfg_.is_last && cfg_.training) {
            dz_all_[L_] = pp_ctx_->dz_in();
            for (int mu = 0; mu < M; ++mu) dz_[mu][L_] = dz_all_[L_] + (size_t)mu * cfg_.mb_rows * act_ld_[L_];
        }
    }
    instrs_ = instrs;
    mu_of_ = mu_of;
    // Two complete plans, one per input-staging buffer: step i reads staging set i % 2 while the copy
    // stream already fills the other set for step i + 1.
    for (int set = 0; set < 2; ++set) {
        select_set(set);
        ops_.clear();
        if (coalesced_) build_coalesced();
        else plan_per_mubatch();
        ops_sets_[set] = std::move(ops_);
        ops_.clear();
    }
    finish_build();
}

void PipeEngine::plan_per_mubatch() {
    const std::vector<std::tuple<int, int, int>>& instrs = instrs_;
    const std::vector<int>& mu_of = mu_of_;
    const int M = cfg_.n_mu, mb = cfg_.mb_rows, n = (int)instrs.size();
    const bool first = cfg_.is_first, last = cfg_.is_last;
    std::vector<bool> started(streams_.size(), false);
    started[0] = true;
    Op begin;
    begin.kind = OP_RECORD; begin.stream = 0; begin.event = new_event();
    ops_.push_back(begin);
    const int ev_begin = begin.event;
    auto use = [&](int s) {
        if (!started[s]) { emit_wait(s, ev_begin); started[s] = true; }
    };
    auto sm = [&](int mu) { return 1 + (mu % n_mu_streams_); };
    auto sw = [&](int l) { return 1 + n_mu_streams_ + (l % n_w_streams_); };

    std::vector<int> ev_in(M, -1), ev_fwd(M, -1), ev_gout(M, -1), ev_bwd(M, -1);
    // Deferred weight-gradient wave (narrow stages, chain kernel): a micro-batch's backward only runs the dgrad chain; the
    // weight gradients of ALL micro-batches are computed at the optimizer step by ONE launch over all rows (k-blocks in
    // micro-batch order, SGD fused; with data parallelism the LL two-shot kernel), instead of n_mu accumulating GEMMs per
    // layer chained through memory (pp=2 GPipe with 8 micro-batches: 32 serialised wgrad launches on stage 0).  dz / act of
    // every micro-batch live in their own rows of the stage's buffers until the step ends, for every schedule.
    auto env_on = [](const char* name, bool dflt) { const char* v = getenv(name); return v ? atoi(v) > 0 : dflt; };
    const bool ll_ok = cfg_.dp_mode == 2 && dp_ctx_ != nullptr && dp_ctx_->ll_enabled();
    // Folded pipeline boundaries (peer transport + chain kernel): no push / wait kernels at all - the chain launch of a
    // micro-batch waits for its input tile's arrival flag itself (while its weights already stream in) and stores its
    // output tile into the neighbour's receive slot from the epilogue that produces it.
    const bool fold_pp = chain_ok_ && pp_ctx_ != nullptr && env_on("SSB_PP_FOLD", true);
    const bool defer_wgrad = chain_ok_ && cfg_.training && (cfg_.dp_mode == 0 || ll_ok) && env_on("SSB_PP_DEFER_WGRAD", true);
    std::vector<bool> first_write(L_ + 1, true);
    std::vector<bool> sw_joined(streams_.size(), false);
    std::vector<int> ev_allreduce;
    std::vector<std::pair<int, int>> pending_dp;         // (layer, event after its final wgrad)
    if (cfg_.dp_mode == 2 && cfg_.training) {
        Op be;
        be.kind = OP_BUMP_EPOCH; be.stream = 0;
        ops_.insert(ops_.begin(), be);   // before the 'begin' event every stream forks from
        ++kernels_extra_;
    }
    if (pp_ctx_) {
        Op be;
        be.kind = OP_PP_BUMP; be.stream = 0;
        ops_.insert(ops_.begin(), be);   // step counter of the boundary flags, before every stream forks
    }
    auto add_gemm = [&](const GemmPlan& g, int stream, int layer, int mu) {
        gemms_.push_back(g);
        maybe_splitk(gemms_.back());
        // FWD drops layer `layer`'s output, DGRAD scales by the mask of layer - 1 (the same p): the spec of the GEMM's
        // rows, micro-batch mu of this stage
        gemms_.back().p.drop = drop_for(g.mode == GEMM_DGRAD ? std::max(layer - 1, 1) : layer, mu * cfg_.mb_rows);
        gate_gemm(gemms_.back());
        skip_gemm(gemms_.back(), layer, mu);
        Op op;
        op.kind = OP_GEMM; op.stream = stream; op.gemm = (int)gemms_.size() - 1; op.layer = layer; op.mu = mu;
        ops_.push_back(op);
    };
    auto check = [](const char* err) { if (err) throw std::runtime_error(std::string("PipeEngine plan: ") + err); };
    auto Wl = [&](int l) { return W_ + cfg_.layers[l - 1].offset; };
    auto Gl = [&](int l) { return G_ + cfg_.layers[l - 1].offset; };

    for (int i = 0; i < n;) {
        const int opc = std::get<0>(instrs[i]);
        // ------------------------------------------------ communication group
        if (fold_pp && opc >= I_RECV_ACT && opc <= I_SEND_GRAD) {
            ++i;                                            // sends and receives happen inside the chain launches
            continue;
        }
        if (pp_ctx_ && opc >= I_RECV_ACT && opc <= I_SEND_GRAD) {
            // ---- peer-memory transport: pushes first (one-sided: they never wait for the peer's schedule position,
            // only for the credit of the previous step), then the waits for what this group receives
            // Small boundary tiles (<= 32 KB: one-CTA push kernel, no shared completion counter) travel on the stream of
            // their micro-batch: the push sits right behind the kernel that produced the tile and the flag wait right in
            // front of the kernel that consumes it - no hop through a shared communication stream, micro-batches do not
            // serialise on each other.  Bigger tiles keep the multi-CTA push on the communication stream.
            const bool act_small = (int64_t)mb * act_ld_[L_] / 4 <= kPpSmallTileF4;
            const bool dz_small = (int64_t)mb * act_ld_[0] / 4 <= kPpSmallTileF4;
            std::vector<std::pair<int, int>> recvs;  // (mu, is_act)
            std::vector<Op> waits;
            int j = i;
            for (; j < n; ++j) {
                const int o = std::get<0>(instrs[j]);
                if (!(o >= I_RECV_ACT && o <= I_SEND_GRAD)) break;
                const int mu = mu_of[j];
                Op x;
                x.stream = s_comm_; x.mu = mu;
                if (o == I_SEND_ACT) {
                    x.stream = act_small ? sm(mu) : s_comm_;
                    use(x.stream);
                    if (ev_fwd[mu] >= 0) emit_wait(x.stream, ev_fwd[mu]);
                    x.kind = OP_PP_PUSH; x.a = act_[mu][L_]; x.b = pp_ctx_->next_act_in(mu); x.n = (int64_t)mb * act_ld_[L_];
                    x.c = reinterpret_cast<float*>(pp_ctx_->next_act_arrived(mu));
                    x.d = reinterpret_cast<float*>(const_cast<uint32_t*>(pp_ctx_->act_credit()));
                    if (!x.b) throw std::runtime_error("PipeEngine: SendActivations without a successor mapping");
                    ops_.push_back(x);
                } else if (o == I_SEND_GRAD) {
                    x.stream = dz_small ? sm(mu) : s_comm_;
                    use(x.stream);
                    if (ev_bwd[mu] >= 0) emit_wait(x.stream, ev_bwd[mu]);
                    x.kind = OP_PP_PUSH; x.a = dz_[mu][0]; x.b = pp_ctx_->prev_dz_in(mu); x.n = (int64_t)mb * act_ld_[0];
                    x.c = reinterpret_cast<float*>(pp_ctx_->prev_dz_arrived(mu));
                    x.d = reinterpret_cast<float*>(const_cast<uint32_t*>(pp_ctx_->dz_credit()));
                    if (!x.b) throw std::runtime_error("PipeEngine: SendInputGrad without a predecessor mapping");
                    ops_.push_back(x);
                } else if (o == I_RECV_ACT) {
                    x.stream = sm(mu);                       // the wait is a one-warp kernel: always on the consumer's stream
                    x.kind = OP_PP_WAIT; x.a = reinterpret_cast<float*>(const_cast<uint32_t*>(pp_ctx_->act_arrived(mu)));
                    waits.push_back(x);
                    recvs.push_back({mu, 1});
                } else {
                    x.stream = sm(mu);
                    x.kind = OP_PP_WAIT; x.a = reinterpret_cast<float*>(const_cast<uint32_t*>(pp_ctx_->dz_arrived(mu)));
                    waits.push_back(x);
                    recvs.push_back({mu, 0});
                }
            }
            for (size_t w = 0; w < waits.size(); ++w) {
                use(waits[w].stream);
                ops_.push_back(waits[w]);
                (recvs[w].second ? ev_in : ev_gout)[recvs[w].first] = emit_record(waits[w].stream);
            }
            i = j;
            continue;
        }
        if (opc >= I_RECV_ACT && opc <= I_SEND_GRAD) {
            Op grp;
            grp.kind = OP_COMM_GROUP; grp.stream = s_comm_;
            std::vector<std::pair<int, int>> recvs;  // (mu, is_act)
            use(s_comm_);
            int j = i;
            for (; j < n; ++j) {
                const int o = std::get<0>(instrs[j]);
                if (!(o >= I_RECV_ACT && o <= I_SEND_GRAD)) break;
                const int mu = mu_of[j];
                CommItem it{};
                if (o == I_SEND_ACT) {
                    it = {1, cfg_.stage + 1, act_[mu][L_], (size_t)mb * act_ld_[L_]};
                    if (ev_fwd[mu] >= 0) emit_wait(s_comm_, ev_fwd[mu]);
                } else if (o == I_RECV_ACT) {
                    it = {0, cfg_.stage - 1, act_[mu][0], (size_t)mb * act_ld_[0]};
                    recvs.push_back({mu, 1});
                } else if (o == I_SEND_GRAD) {
                    it = {1, cfg_.stage - 1, dz_[mu][0], (size_t)mb * act_ld_[0]};
                    if (ev_bwd[mu] >= 0) emit_wait(s_comm_, ev_bwd[mu]);
                } else {   // a residual last layer receives its skip gradient g[L] (gated into dz[L] below)
                    it = {0, cfg_.stage + 1, res_layer(L_) && cfg_.training ? gres_[mu][L_] : dz_[mu][L_], (size_t)mb * act_ld_[L_]};
                    recvs.push_back({mu, 0});
                }
                grp.comm.push_back(it);
            }
            ops_.push_back(grp);
            if (!recvs.empty()) {
                const int ev = emit_record(s_comm_);
                for (auto& r : recvs) (r.second ? ev_in : ev_gout)[r.first] = ev;
            }
            i = j;
            continue;
        }
        const int mu = mu_of[i];
        switch (opc) {
            case I_ZERO_GRAD:
                std::fill(first_write.begin(), first_write.end(), true);
                break;
            case I_LOAD_X:
            case I_LOAD_Y:
                break;   // the whole DP-local batch is staged with one copy before the step
            case I_FORWARD: {
                const int s = sm(mu);
                use(s);
                if (ev_in[mu] >= 0) {
                    emit_wait(s, ev_in[mu]);
                    ev_in[mu] = -1;
                }
                if (chain_ok_) {
                    // whole stage forward (+ loss head on the last stage) of this micro-batch in one launch
                    ChainFold cf;
                    if (fold_pp) {
                        if (!first) { cf.in_flag = pp_ctx_->act_arrived(mu); cf.x_from_global = true; }
                        if (!last) {
                            cf.out_peer = pp_ctx_->next_act_in(mu); cf.out_flag = pp_ctx_->next_act_arrived(mu);
                            cf.out_credit = pp_ctx_->act_credit();
                        }
                    }
                    add_chain(s, mu, 1, true, last, false, fold_pp ? &cf : nullptr);
                    if (!cfg_.training && last) {
                        Op am;
                        am.kind = OP_ARGMAX; am.stream = s;
                        am.a = probs_[mu]; am.lda = act_ld_[L_]; am.b = y_stage_ + (size_t)mu * mb * y_ld_; am.ldb = y_ld_;
                        am.rows = mb; am.cols = cfg_.out_dim;
                        ops_.push_back(am);
                    }
                } else {
                    for (int l = 1; l <= L_; ++l) {
                        const LayerSpec& ls = cfg_.layers[l - 1];
                        GemmPlan g;
                        check(gemm_plan_fwd(&g, Wl(l), ls.ld, act_[mu][l - 1], act_ld_[l - 1], act_[mu][l], act_ld_[l], mb,
                                            ls.in, ls.out, Wl(l) + ls.in, ls.ld, ls.relu, cfg_.prec));
                        add_gemm(g, s, l, mu);
                    }
                    if (!cfg_.training && last) {
                        Op sm_op;
                        sm_op.kind = OP_SOFTMAX; sm_op.stream = s;
                        sm_op.a = act_[mu][L_]; sm_op.lda = act_ld_[L_]; sm_op.b = probs_[mu]; sm_op.ldb = act_ld_[L_];
                        sm_op.rows = mb; sm_op.cols = cfg_.out_dim;
                        ops_.push_back(sm_op);
                        Op am;
                        am.kind = OP_ARGMAX; am.stream = s;
                        am.a = probs_[mu]; am.lda = act_ld_[L_]; am.b = y_stage_ + (size_t)mu * mb * y_ld_; am.ldb = y_ld_;
                        am.rows = mb; am.cols = cfg_.out_dim;
                        ops_.push_back(am);
                    }
                }
                ev_fwd[mu] = emit_record(s);
                break;
            }
            case I_BWD_ACC:
            case I_BWD_AR: {
                const bool final_bwd = (opc == I_BWD_AR);
                const int s = sm(mu);
                use(s);
                if (ev_gout[mu] >= 0) { emit_wait(s, ev_gout[mu]); ev_gout[mu] = -1; }
                if (chain_ok_) {
                    // dZ_L (from the loss head at forward time, or received from the next stage) -> ReLU mask ->
                    // the whole dgrad chain in one launch; then one wave of weight-gradient GEMMs
                    ChainFold cb;
                    if (fold_pp) {
                        if (!last) cb.in_flag = pp_ctx_->dz_arrived(mu);
                        if (!first) {
                            cb.out_peer = pp_ctx_->prev_dz_in(mu); cb.out_flag = pp_ctx_->prev_dz_arrived(mu);
                            cb.out_credit = pp_ctx_->dz_credit();
                        }
                    }
                    add_chain(s, mu, 1, false, false, true, fold_pp ? &cb : nullptr);
                    const int ev_dz_all = emit_record(s);
                    for (int l = L_; l >= 1 && !defer_wgrad; --l) {
                        const LayerSpec& ls = cfg_.layers[l - 1];
                        const int w = sw(l);
                        use(w);
                        emit_wait(w, ev_dz_all);
                        GemmPlan g;
                        check(gemm_plan_wgrad(&g, dz_[mu][l], act_ld_[l], act_[mu][l - 1], act_ld_[l - 1], Gl(l), ls.ld, mb,
                                              ls.in, ls.out, first_write[l] ? 0 : 1, Gl(l) + ls.in, ls.ld, nullptr, 0, nullptr, 0,
                                              cfg_.prec));
                        add_gemm(g, w, l, mu);
                        first_write[l] = false;
                        if (final_bwd && cfg_.dp_mode == 1 && cfg_.dp_size > 1) {
                            const int ev_g = emit_record(w);
                            use(s_dp_);
                            emit_wait(s_dp_, ev_g);
                            Op ar;
                            ar.kind = OP_ALLREDUCE; ar.stream = s_dp_; ar.a = Gl(l); ar.n = (int64_t)ls.out * ls.ld; ar.layer = l;
                            ops_.push_back(ar);
                        }
                        if (final_bwd && cfg_.dp_mode == 2) pending_dp.push_back({l, emit_record(w)});
                    }
                } else {
                    if (last) {
                        Op lh;
                        lh.kind = OP_LOSS_HEAD; lh.stream = s;
                        lh.a = act_[mu][L_]; lh.lda = act_ld_[L_];
                        lh.b = y_stage_ + (size_t)mu * mb * y_ld_; lh.ldb = y_ld_;
                        lh.c = probs_[mu]; lh.ldc = act_ld_[L_];
                        lh.d = dz_[mu][L_]; lh.ldd = act_ld_[L_];
                        lh.rows = mb; lh.cols = cfg_.out_dim; lh.scalar = 1.0f / (float)cfg_.global_batch; lh.mu = mu;
                        ops_.push_back(lh);
                    } else if (L_ > 0 && cfg_.layers[L_ - 1].relu) {
                        Op rm;
                        rm.kind = OP_RELU_MASK; rm.stream = s;
                        rm.a = dz_[mu][L_]; rm.lda = act_ld_[L_]; rm.b = act_[mu][L_]; rm.ldb = act_ld_[L_];
                        rm.rows = mb; rm.cols = cfg_.layers[L_ - 1].out;
                        if (dropout_on()) {                                     // act_L was dropped
                            rm.dropout = true;
                            rm.scalar = dropout_spec(cfg_.dropout, cfg_.dropout_seed).scale;
                        }
                        if (gated()) { rm.gated = true; rm.b = gamma_[mu][L_]; }   // the gate (with the scale) replaces both
                        if (res_layer(L_)) { rm.c = gres_[mu][L_]; rm.ldc = act_ld_[L_]; }   // out of place: g[L] stays
                        ops_.push_back(rm);
                    }
                    for (int l = L_; l >= 1; --l) {
                        const LayerSpec& ls = cfg_.layers[l - 1];
                        const int ev_dz = emit_record(s);
                        const int w = sw(l);
                        use(w);
                        emit_wait(w, ev_dz);
                        GemmPlan g;
                        check(gemm_plan_wgrad(&g, dz_[mu][l], act_ld_[l], act_[mu][l - 1], act_ld_[l - 1], Gl(l), ls.ld, mb,
                                              ls.in, ls.out, first_write[l] ? 0 : 1, Gl(l) + ls.in, ls.ld, nullptr, 0, nullptr, 0,
                                              cfg_.prec));
                        add_gemm(g, w, l, mu);
                        first_write[l] = false;
                        if (final_bwd && cfg_.dp_mode == 1 && cfg_.dp_size > 1) {
                            const int ev_g = emit_record(w);
                            use(s_dp_);
                            emit_wait(s_dp_, ev_g);
                            Op ar;
                            ar.kind = OP_ALLREDUCE; ar.stream = s_dp_; ar.a = Gl(l); ar.n = (int64_t)ls.out * ls.ld; ar.layer = l;
                            ops_.push_back(ar);
                        }
                        if (final_bwd && cfg_.dp_mode == 2) pending_dp.push_back({l, emit_record(w)});
                        if (l > 1 || !first) {
                            const float* mask = (l >= 2 && cfg_.layers[l - 2].relu) ? act_[mu][l - 1] : nullptr;
                            GemmPlan g2;
                            check(gemm_plan_dgrad(&g2, Wl(l), ls.ld, dz_[mu][l], act_ld_[l], dz_[mu][l - 1], act_ld_[l - 1], mb, ls.in,
                                                  ls.out, mask, act_ld_[l - 1], cfg_.prec));
                            add_gemm(g2, s, l, mu);
                        }
                    }
                }
                ev_bwd[mu] = emit_record(s);
                if (final_bwd && cfg_.dp_mode == 2 && !defer_wgrad) {
                    // G is final: reduce across replicas + SGD + weight broadcast in ONE kernel per layer
                    // over peer memory.  W is rewritten, so every reader (all micro-batches) must be done.
                    if (!dp_ctx_) throw std::runtime_error("PipeEngine: dp_mode fused needs a DpContext");
                    use(s_dp_);
                    for (int m2 = 0; m2 < M; ++m2)
                        if (ev_bwd[m2] >= 0) emit_wait(s_dp_, ev_bwd[m2]);
                        else if (ev_fwd[m2] >= 0) emit_wait(s_dp_, ev_fwd[m2]);
                    for (auto& pd : pending_dp) {
                        emit_wait(s_dp_, pd.second);
                        DpLayerParams lp = dp_ctx_->layer_params(pd.first - 1);
                        lp.opt = opt_for(0);
                        lp.lr = lr_slot();
                        layer_proto_[pd.first - 1] = lp.one_shot ? DP_PROTO_ALL : DP_PROTO_TWO_SHOT;
                        lp.G = Gl(pd.first);
                        FusedDpPlan fp;
                        check(fused_dp_plan(&fp, nullptr, 0, nullptr, 0, mb, lp, dp_ctx_->peers(), kFusedDpMaxCtas));
                        dp_plans_.push_back(fp);
                        Op fo;
                        fo.kind = OP_DP_REDUCE; fo.stream = s_dp_; fo.gemm = (int)dp_plans_.size() - 1; fo.layer = pd.first;
                        ops_.push_back(fo);
                    }
                    pending_dp.clear();
                }
                break;
            }
            case I_OPT_STEP: {
                if (defer_wgrad) {
                    const int rows_all = M * mb;
                    use(s_dp_);
                    for (int m2 = 0; m2 < M; ++m2)           // every reader of W and every producer of dz is done
                        if (ev_bwd[m2] >= 0) emit_wait(s_dp_, ev_bwd[m2]);
                        else if (ev_fwd[m2] >= 0) emit_wait(s_dp_, ev_fwd[m2]);
                    if (cfg_.dp_mode == 0) {
                        std::vector<GemmPlan> grouped;
                        for (int l = L_; l >= 1; --l) {
                            const LayerSpec& ls = cfg_.layers[l - 1];
                            GemmPlan g;
                            check(gemm_plan_wgrad(&g, dz_all_[l], act_ld_[l], act_all_[l - 1], act_ld_[l - 1], Gl(l), ls.ld, rows_all, ls.in,
                                                  ls.out, 0, Gl(l) + ls.in, ls.ld, Wl(l), ls.ld, lr_slot(), 1, cfg_.prec,
                                                  opt_for(l)));
                            grouped.push_back(g);
                        }
                        GemmGroupPlan gp;
                        check(gemm_group_plan(&gp, grouped.data(), (int)grouped.size()));
                        group_plans_.push_back(gp);
                        Op go;
                        go.kind = OP_WGRAD_GROUP; go.stream = s_dp_; go.gemm = (int)group_plans_.size() - 1;
                        ops_.push_back(go);
                    } else {
                        std::vector<DpLLLayer> lls;
                        for (int l = L_; l >= 1; --l) {
                            const LayerSpec& ls = cfg_.layers[l - 1];
                            DpLLLayer ly{};
                            ly.dZ = dz_all_[l]; ly.X = act_all_[l - 1]; ly.prec = cfg_.prec;
                            ly.lddz = act_ld_[l]; ly.ldx = act_ld_[l - 1]; ly.in = ls.in; ly.out = ls.out; ly.ldw = ls.ld; ly.w_offset = ls.offset;
                            lls.push_back(ly);
                        }
                        DpLLPlan lp;
                        DpLLParams base = dp_ctx_->ll_params();
                        base.opt = opt_for(0);
                        base.lr = lr_slot();
                        for (int l = 0; l < L_; ++l) layer_proto_[l] = DP_PROTO_LL;
                        check(dp_ll_plan(&lp, lls.data(), (int)lls.size(), rows_all, base));
                        ll_plans_.push_back(lp);
                        Op lo;
                        lo.kind = OP_DP_LL; lo.stream = s_dp_; lo.gemm = (int)ll_plans_.size() - 1;
                        ops_.push_back(lo);
                    }
                    break;
                }
                if (cfg_.dp_mode == 2) break;            // the update already happened inside the fused kernels
                {
                    use(s_dp_);
                    for (int m2 = 0; m2 < M; ++m2)
                        if (ev_bwd[m2] >= 0) emit_wait(s_dp_, ev_bwd[m2]);
                    for (int w = 0; w < n_w_streams_; ++w) {
                        const int ws = 1 + n_mu_streams_ + w;
                        if (started[ws]) { const int e = emit_record(ws); emit_wait(s_dp_, e); }
                    }
                    Op sg;
                    sg.kind = (cfg_.dp_mode == 3) ? OP_NVLS_SGD : OP_SGD;
                    sg.stream = s_dp_; sg.a = W_; sg.b = G_; sg.lr = lr_slot(); sg.n = arena_numel_;
                    ops_.push_back(sg);
                }
                break;
            }
            default:
                throw std::runtime_error("PipeEngine: unknown opcode");
        }
        ++i;
    }
    // ---- join every side stream back into the main stream
    for (size_t s = 1; s < streams_.size(); ++s)
        if (started[s]) { const int e = emit_record((int)s); emit_wait(0, e); }
    if (pp_ctx_) {                           // everything that read my receive slots is done: hand them back
        Op cr;
        cr.kind = OP_PP_CREDIT; cr.stream = 0;
        cr.a = reinterpret_cast<float*>(pp_ctx_->prev_act_credit());
        cr.b = cfg_.training ? reinterpret_cast<float*>(pp_ctx_->next_dz_credit()) : nullptr;
        ops_.push_back(cr);
    }
}

// Stage without pipeline communication (pp == 1): micro-batches are independent until the
// optimizer step, so every layer runs ONCE over all of them (rows = n_mu * mb_rows).  The
// loss head still runs one CTA per micro-batch (its global-max contract is per micro-batch),
// the weight gradient accumulates over the micro-batches in registers (k-blocks in micro-batch
// order) instead of through memory, and with a single replica the SGD update is fused into
// the wgrad epilogue (TMA reduce-add of -lr * dW into W): ZeroGrad / OptimizerStep vanish.
void PipeEngine::build_coalesced() {
    const int M = cfg_.n_mu, mb = cfg_.mb_rows, rows = M * mb;
    auto check = [](const char* err) { if (err) throw std::runtime_error(std::string("PipeEngine plan: ") + err); };
    auto Wl = [&](int l) { return W_ + cfg_.layers[l - 1].offset; };
    auto Gl = [&](int l) { return G_ + cfg_.layers[l - 1].offset; };
    auto add_gemm = [&](const GemmPlan& g, int stream, int layer) {
        gemms_.push_back(g);
        maybe_splitk(gemms_.back());
        gemms_.back().p.drop = drop_for(g.mode == GEMM_DGRAD ? std::max(layer - 1, 1) : layer, 0);   // all rows
        gate_gemm(gemms_.back());
        skip_gemm(gemms_.back(), layer, -1);
        Op op;
        op.kind = OP_GEMM; op.stream = stream; op.gemm = (int)gemms_.size() - 1; op.layer = layer; op.mu = -1;
        ops_.push_back(op);
    };
    std::vector<bool> started(streams_.size(), false);
    started[0] = true;
    Op begin;
    begin.kind = OP_RECORD; begin.stream = 0; begin.event = new_event();
    ops_.push_back(begin);
    const int ev_begin = begin.event;
    auto use = [&](int s) { if (!started[s]) { emit_wait(s, ev_begin); started[s] = true; } };
    auto sw = [&](int l) { return 1 + n_mu_streams_ + (l % n_w_streams_); };

    const bool chain = chain_ok_;
    // Gated launch: the LL data-parallel kernel (dp_ll.cu) is forked at the START of the step next to the chain kernel
    // instead of behind it.  The chain kernel's epilogue warps count up a per-layer device counter when dz[l] is
    // globally visible; the tiles of layer l wait for ready[l] before their first TMA load and for ready[l-1] (the dgrad
    // that reads W_l retired) before they update W_l in place.  Only layer 1's tiles remain behind the chain kernel.
    // (The same gate in front of the single-GPU grouped wgrad launch was measured neutral - 79.7 vs 78.7 us - and removed.)
    auto env_on = [](const char* name, bool dflt) { const char* v = getenv(name); return v ? atoi(v) > 0 : dflt; };
    // fused DP over narrow layers: the LL two-shot kernel (dp_ll.cu), all layers in one launch, gated the same way
    const bool ll_on = chain && cfg_.training && cfg_.dp_mode == 2 && dp_ctx_ != nullptr && dp_ctx_->ll_enabled();
    gate_on_ = ll_on && env_on("SSB_DP_GATE", true);
    if (gate_on_ && gate_ready_ == nullptr) {
        uint32_t* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, 256));
        CUDA_CHECK(cudaMemset(p, 0, 256));
        owned_.push_back(p);
        gate_ready_ = p;              // [0 .. L] per-layer counters, [32] step counter of this engine
        gate_step_ = p + 32;
    }
    if (chain) {
        // forward + loss head (+ whole dgrad chain when training) of every micro-batch in ONE launch
        add_chain(0, 0, M, true, true, cfg_.training != 0);
        if (!cfg_.training) {
            Op am;
            am.kind = OP_ARGMAX; am.stream = 0;
            am.a = probs_all_; am.lda = act_ld_[L_]; am.b = y_stage_; am.ldb = y_ld_; am.rows = rows; am.cols = cfg_.out_dim;
            ops_.push_back(am);
            return;
        }
    } else {
        for (int l = 1; l <= L_; ++l) {
            const LayerSpec& ls = cfg_.layers[l - 1];
            GemmPlan g;
            check(gemm_plan_fwd(&g, Wl(l), ls.ld, act_all_[l - 1], act_ld_[l - 1], act_all_[l], act_ld_[l], rows, ls.in, ls.out,
                                Wl(l) + ls.in, ls.ld, ls.relu, cfg_.prec));
            add_gemm(g, 0, l);
        }
        if (!cfg_.training) {
            Op sm_op;
            sm_op.kind = OP_SOFTMAX; sm_op.stream = 0;
            sm_op.a = act_all_[L_]; sm_op.lda = act_ld_[L_]; sm_op.b = probs_all_; sm_op.ldb = act_ld_[L_];
            sm_op.rows = rows; sm_op.cols = cfg_.out_dim; sm_op.n = mb;
            ops_.push_back(sm_op);
            Op am;
            am.kind = OP_ARGMAX; am.stream = 0;
            am.a = probs_all_; am.lda = act_ld_[L_]; am.b = y_stage_; am.ldb = y_ld_; am.rows = rows; am.cols = cfg_.out_dim;
            ops_.push_back(am);
            return;
        }
        Op lh;
        lh.kind = OP_LOSS_HEAD; lh.stream = 0;
        lh.a = act_all_[L_]; lh.lda = act_ld_[L_]; lh.b = y_stage_; lh.ldb = y_ld_; lh.c = probs_all_; lh.ldc = act_ld_[L_];
        lh.d = dz_all_[L_]; lh.ldd = act_ld_[L_]; lh.rows = rows; lh.cols = cfg_.out_dim;
        lh.scalar = 1.0f / (float)cfg_.global_batch; lh.mu = 0; lh.n = mb;
        ops_.push_back(lh);
    }
    const bool fuse = (cfg_.dp_mode == 0);
    const bool fused_dp = (cfg_.dp_mode == 2);
    // chain stages: all layers' weight-gradient tiles in ONE launch on the main stream right behind the chain kernel
    // (which has produced every dZ and is the last reader of every W) - no fork / join per layer (also with the NVLS
    // path, whose single reduce+SGD kernel follows the whole wgrad wave anyway)
    const bool group_wgrad = chain && (fuse || cfg_.dp_mode == 3);
    std::vector<GemmPlan> grouped;
    std::vector<DpLLLayer> ll_layers;
    int ev_bump = -1;
    if (fused_dp) {
        if (!dp_ctx_) throw std::runtime_error("PipeEngine: dp_mode fused needs a DpContext");
        // step counter for the flag protocol: bumped on the DP stream, off the forward critical path
        use(s_dp_);
        Op be;
        be.kind = OP_BUMP_EPOCH; be.stream = s_dp_;
        ops_.push_back(be);
        ev_bump = emit_record(s_dp_);
    }
    for (int l = L_; l >= 1; --l) {
        const LayerSpec& ls = cfg_.layers[l - 1];
        const int ev_dz = emit_record(0);
        int ev_dg = -1;
        if (l > 1 && !chain) {
            const float* mask = cfg_.layers[l - 2].relu ? act_all_[l - 1] : nullptr;
            GemmPlan g;
            check(gemm_plan_dgrad(&g, Wl(l), ls.ld, dz_all_[l], act_ld_[l], dz_all_[l - 1], act_ld_[l - 1], rows, ls.in, ls.out,
                                  mask, act_ld_[l - 1], cfg_.prec));
            add_gemm(g, 0, l);
            ev_dg = emit_record(0);
        }
        if (fused_dp && ll_on) {
            DpLLLayer ly{};
            ly.dZ = dz_all_[l]; ly.X = act_all_[l - 1];
            ly.prec = cfg_.prec;
            ly.lddz = act_ld_[l]; ly.ldx = act_ld_[l - 1]; ly.in = ls.in; ly.out = ls.out; ly.ldw = ls.ld; ly.w_offset = ls.offset;
            if (gate_on_) {
                // GEMM + reduce-scatter hop start when dz[l] is final; the in-place update of W_l additionally waits until
                // the dgrad that reads W_l has produced dz[l-1] (layer 1 of the first stage has no dgrad)
                ly.gate_flag = gate_ready_ + l;
                ly.gate_w = l >= 2 ? gate_ready_ + (l - 1) : nullptr;
                // 8 epilogue warps per micro-batch count up every counter: gated chain launches run one CTA per micro-batch
                if (chain_cluster() != 1) throw std::runtime_error("PipeEngine: a gated chain launch must run one CTA per micro-batch");
                ly.gate_mult = 8u * (uint32_t)M;
            }
            ll_layers.push_back(ly);
            continue;
        }
        if (fused_dp) {
            // ONE kernel per layer: wgrad GEMM -> NVLink push -> owner reduce -> SGD -> weight broadcast.
            // All fused kernels of all layers go through ONE stream in the same order on every rank.
            // (big layers).  When the CTAs of ALL layers fit on the chip together they may overlap freely.
            const int sdp = (dp_ctx_->total_ctas() <= kFusedDpMaxCtas) ? sw(l) : s_dp_;
            use(sdp);
            if (sdp != s_dp_) emit_wait(sdp, ev_bump);
            emit_wait(sdp, ev_dz);
            if (ev_dg >= 0) emit_wait(sdp, ev_dg);
            FusedDpPlan fp;
            DpLayerParams lp = dp_ctx_->layer_params(l - 1);
            lp.opt = opt_for(0);
            lp.lr = lr_slot();
            layer_proto_[l - 1] = lp.one_shot ? DP_PROTO_ALL : DP_PROTO_TWO_SHOT;
            if (getenv("SSB_CHAIN_TIMELINE")) {
                if (!chain_dbg_) {
                    CUDA_CHECK(cudaMalloc(&chain_dbg_, 4 * 256 * sizeof(unsigned long long)));
                    CUDA_CHECK(cudaMemset(chain_dbg_, 0, 4 * 256 * sizeof(unsigned long long)));
                    owned_.push_back(chain_dbg_);
                }
                lp.dbg = chain_dbg_ + 3 * 256 + 8 * l;
            }
            check(fused_dp_plan(&fp, dz_all_[l], act_ld_[l], act_all_[l - 1], act_ld_[l - 1], rows, lp, dp_ctx_->peers(), kFusedDpMaxCtas,
                                cfg_.prec));
            dp_plans_.push_back(fp);
            Op fo;
            fo.kind = OP_FUSED_DP; fo.stream = sdp; fo.gemm = (int)dp_plans_.size() - 1; fo.layer = l;
            ops_.push_back(fo);
            continue;
        }
        const int w = group_wgrad ? 0 : sw(l);
        if (!group_wgrad) {
            use(w);
            emit_wait(w, ev_dz);
            if (fuse && ev_dg >= 0) emit_wait(w, ev_dg);  // W_l is updated in place: its last reader must be done
        }
        GemmPlan g;
        check(gemm_plan_wgrad(&g, dz_all_[l], act_ld_[l], act_all_[l - 1], act_ld_[l - 1], Gl(l), ls.ld, rows, ls.in, ls.out, 0,
                              Gl(l) + ls.in, ls.ld, fuse ? Wl(l) : nullptr, ls.ld, lr_slot(), fuse ? 1 : 0, cfg_.prec,
                              fuse ? opt_for(l) : SgdState{}));
        if (group_wgrad) {                                  // launched together after the loop
            grouped.push_back(g);
            continue;
        }
        add_gemm(g, w, l);
        if (cfg_.dp_mode == 1 && cfg_.dp_size > 1) {
            const int ev_g = emit_record(w);
            use(s_dp_);
            emit_wait(s_dp_, ev_g);
            Op ar;
            ar.kind = OP_ALLREDUCE; ar.stream = s_dp_; ar.a = Gl(l); ar.n = (int64_t)ls.out * ls.ld; ar.layer = l;
            ops_.push_back(ar);
        }
    }
    if (!ll_layers.empty()) {
        // deepest layer first: its tiles get the lowest block indices, i.e. they are resident first and their gate opens first
        DpLLParams base = dp_ctx_->ll_params();
        base.opt = opt_for(0);
        base.lr = lr_slot();
        for (int l = 0; l < L_; ++l) layer_proto_[l] = DP_PROTO_LL;
        base.gate_step = gate_on_ ? gate_step_ : nullptr;
        if (getenv("SSB_CHAIN_TIMELINE")) {
            if (!chain_dbg_) {
                CUDA_CHECK(cudaMalloc(&chain_dbg_, 4 * 256 * sizeof(unsigned long long)));
                CUDA_CHECK(cudaMemset(chain_dbg_, 0, 4 * 256 * sizeof(unsigned long long)));
                owned_.push_back(chain_dbg_);
            }
            base.dbg = chain_dbg_ + 3 * 256;              // role 3 of the timeline buffer: 8 stamps x 28 tiles + spare
        }
        DpLLPlan lp;
        check(dp_ll_plan(&lp, ll_layers.data(), (int)ll_layers.size(), rows, base));
        ll_plans_.push_back(lp);
        if (gate_on_) {
            Op bs;
            bs.kind = OP_BUMP_STEP; bs.stream = s_dp_;
            ops_.push_back(bs);
        } else {
            emit_wait(s_dp_, emit_record(0));               // behind the chain kernel
        }
        Op lo;
        lo.kind = OP_DP_LL; lo.stream = s_dp_; lo.gemm = (int)ll_plans_.size() - 1;
        ops_.push_back(lo);
    }
    if (group_wgrad && !grouped.empty()) {
        GemmGroupPlan gp;
        check(gemm_group_plan(&gp, grouped.data(), (int)grouped.size()));
        group_plans_.push_back(gp);
        Op go;
        go.kind = OP_WGRAD_GROUP; go.stream = 0; go.gemm = (int)group_plans_.size() - 1;
        ops_.push_back(go);
    }
    if (!fuse && !fused_dp) {
        const int ev_main = emit_record(0);
        use(s_dp_);
        emit_wait(s_dp_, ev_main);
        for (int w = 0; w < n_w_streams_; ++w) {
            const int ws = 1 + n_mu_streams_ + w;
            if (started[ws]) { const int e = emit_record(ws); emit_wait(s_dp_, e); }
        }
        Op sg;
        sg.kind = (cfg_.dp_mode == 3) ? OP_NVLS_SGD : OP_SGD;
        sg.stream = s_dp_; sg.a = W_; sg.b = G_; sg.lr = lr_slot(); sg.n = arena_numel_;
        ops_.push_back(sg);
    }
    for (size_t s = 1; s < streams_.size(); ++s)
        if (started[s]) { const int e = emit_record((int)s); emit_wait(0, e); }
}

void PipeEngine::finish_build() {
    kernels_per_step_ = 0;
    for (auto& op : ops_sets_[0]) {
        if (op.kind == OP_GEMM || op.kind == OP_LOSS_HEAD || op.kind == OP_SOFTMAX || op.kind == OP_RELU_MASK ||
            op.kind == OP_SGD || op.kind == OP_ARGMAX || op.kind == OP_FUSED_DP || op.kind == OP_DP_REDUCE ||
            op.kind == OP_BUMP_EPOCH || op.kind == OP_CHAIN || op.kind == OP_NVLS_SGD ||
            op.kind == OP_PP_PUSH || op.kind == OP_PP_WAIT || op.kind == OP_PP_CREDIT || op.kind == OP_PP_BUMP ||
            op.kind == OP_WGRAD_GROUP || op.kind == OP_BUMP_STEP || op.kind == OP_DP_LL)
            ++kernels_per_step_;
    }
    built_ = true;

    // kernel attributes are configured up front (never inside a capture); communicators are
    // warmed up by their creator.  No eager pass here: a training step mutates the weights.
    CUDA_CHECK(gemm_configure());
    if (!chain_plans_.empty()) CUDA_CHECK(chain_configure());
    if (cfg_.dp_mode == 2) CUDA_CHECK(fused_dp_configure());
    if (!ll_plans_.empty()) CUDA_CHECK(dp_ll_configure());
    comm_timing_ = getenv("SSB_COMM_TIMING") != nullptr;   // needs timing events between ops: eager plan walk
    if (cfg_.use_graph && !comm_timing_) {
        for (int set = 0; set < 2; ++set) {
            CUDA_CHECK(cudaStreamBeginCapture(streams_[0], cudaStreamCaptureModeThreadLocal));
            walk(set);
            CUDA_CHECK(cudaStreamEndCapture(streams_[0], &graph_sets_[set]));
            CUDA_CHECK(cudaGraphInstantiate(&graph_exec_sets_[set], graph_sets_[set], 0));
        }
        size_t nn = 0;
        CUDA_CHECK(cudaGraphGetNodes(graph_sets_[0], nullptr, &nn));
        graph_nodes_ = (int64_t)nn;
    }
}

cudaStream_t PipeEngine::stream_of(const Op& op) const {
    static const bool serialize = getenv("SSB_SERIALIZE") != nullptr;
    return streams_[serialize ? 0 : op.stream];
}

void PipeEngine::exec(const Op& op, int set) {
    cudaStream_t st = stream_of(op);
    switch (op.kind) {
        case OP_WAIT: CUDA_CHECK(cudaStreamWaitEvent(st, events_[op.event], 0)); break;
        case OP_RECORD: CUDA_CHECK(cudaEventRecord(events_[op.event], st)); break;
        case OP_GEMM: CUDA_CHECK(gemm_launch(gemms_[op.gemm], st)); break;
        case OP_WGRAD_GROUP: CUDA_CHECK(gemm_group_launch(group_plans_[op.gemm], st)); break;
        case OP_LOSS_HEAD:
            CUDA_CHECK(launch_loss_head(op.a, op.lda, op.b, op.ldb, op.c, op.ldc, op.d, op.ldd, loss_slot(set) + op.mu, op.rows,
                                        op.cols, op.scalar, st, (int)op.n, cfg_.loss));
            break;
        case OP_SOFTMAX:
            CUDA_CHECK(launch_loss_head(op.a, op.lda, nullptr, 0, op.b, op.ldb, nullptr, 0, nullptr, op.rows, op.cols, 0.f, st,
                                        (int)op.n, cfg_.loss));
            break;
        case OP_ARGMAX:
            CUDA_CHECK(launch_argmax_correct(op.a, op.lda, op.b, op.ldb, op.rows, op.cols, correct_dev_, st));
            break;
        case OP_RELU_MASK:
            if (op.gated && op.c != nullptr) CUDA_CHECK(launch_gate_mul_to(op.a, op.lda, op.c, op.ldc, op.b, op.ldb, op.rows, op.cols, st));
            else if (op.gated) CUDA_CHECK(launch_gate_mul(op.a, op.lda, op.b, op.ldb, op.rows, op.cols, st));
            else if (op.dropout) CUDA_CHECK(launch_relu_mask_scaled(op.a, op.lda, op.b, op.ldb, op.rows, op.cols, op.scalar, st));
            else CUDA_CHECK(launch_relu_mask(op.a, op.lda, op.b, op.ldb, op.rows, op.cols, st));
            break;
        case OP_SGD: {
            const SgdState opt = opt_for(0, set);
            if (opt.form() == SGD_PLAIN) CUDA_CHECK(launch_sgd(op.a, op.b, op.lr, op.n, st));
            else CUDA_CHECK(launch_sgd_momentum(op.a, op.b, op.lr, opt, op.n, st));
            break;
        }
        case OP_NVLS_SGD: {
            if (!nvls_ctx_) throw std::runtime_error("PipeEngine: dp_mode nvls needs an NvlsContext");
            if (nvls_ctx_->weights() != W_ || nvls_ctx_->grads() != G_)
                throw std::runtime_error("PipeEngine: the parameter arena must live in the NVLS allocation");
            int dev = 0, sms = 132;
            CUDA_CHECK(cudaGetDevice(&dev));
            CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            NvlsParams np = nvls_ctx_->params();
            np.opt = opt_for(0, set);
            np.lr = op.lr;
            CUDA_CHECK(launch_nvls_reduce_sgd(np, sms, st));
            break;
        }
        case OP_ALLREDUCE:
            if (!dp_comm_) throw std::runtime_error("PipeEngine: DP all-reduce without a communicator");
            NCCL_CHECK(ncclAllReduce(op.a, op.a, (size_t)op.n, ncclFloat, ncclSum, dp_comm_, st));
            break;
        case OP_COMM_GROUP: {
            if (!pp_comm_) throw std::runtime_error("PipeEngine: pipeline send/recv without a communicator");
            NCCL_CHECK(ncclGroupStart());
            for (const auto& it : op.comm) {
                if (it.is_send) NCCL_CHECK(ncclSend(it.ptr, it.count, ncclFloat, it.peer, pp_comm_, st));
                else NCCL_CHECK(ncclRecv(it.ptr, it.count, ncclFloat, it.peer, pp_comm_, st));
            }
            NCCL_CHECK(ncclGroupEnd());
            break;
        }
        case OP_CHAIN: CUDA_CHECK(chain_launch(chain_plans_[op.gemm], st)); break;
        case OP_FUSED_DP: CUDA_CHECK(launch_fused_wgrad_dp(dp_plans_[op.gemm], st)); break;
        case OP_DP_REDUCE: CUDA_CHECK(launch_dp_reduce_sgd(dp_plans_[op.gemm], st)); break;
        case OP_BUMP_EPOCH: CUDA_CHECK(launch_bump_epoch(dp_ctx_->epoch_ptr(), st)); break;
        case OP_BUMP_STEP: CUDA_CHECK(launch_bump_epoch(gate_step_, st)); break;
        case OP_DP_LL: CUDA_CHECK(launch_dp_ll(ll_plans_[op.gemm], st)); break;
        case OP_PP_BUMP: CUDA_CHECK(launch_bump_epoch(pp_ctx_->epoch_ptr(), st)); break;
        case OP_PP_PUSH:
            CUDA_CHECK(launch_pp_push(op.a, op.b, op.n, reinterpret_cast<uint32_t*>(op.c), reinterpret_cast<const uint32_t*>(op.d),
                                      pp_ctx_->epoch_ptr(), pp_ctx_->push_done_ptr(), st));
            break;
        case OP_PP_WAIT: CUDA_CHECK(launch_pp_wait(reinterpret_cast<const uint32_t*>(op.a), pp_ctx_->epoch_ptr(), st)); break;
        case OP_PP_CREDIT:
            CUDA_CHECK(launch_pp_credit(reinterpret_cast<uint32_t*>(op.a), reinterpret_cast<uint32_t*>(op.b), pp_ctx_->epoch_ptr(), st));
            break;
        default: throw std::runtime_error("PipeEngine: bad op");
    }
}

static const char* op_name(int kind) {
    switch (kind) {
        case OP_GEMM: return "gemm";
        case OP_WGRAD_GROUP: return "wgrad_group";
        case OP_LOSS_HEAD: return "loss_head";
        case OP_SOFTMAX: return "softmax";
        case OP_RELU_MASK: return "relu_mask";
        case OP_SGD: return "sgd";
        case OP_NVLS_SGD: return "nvls_reduce_sgd";
        case OP_COMM_GROUP: return "pp_send_recv";
        case OP_ALLREDUCE: return "dp_allreduce_nccl";
        case OP_FUSED_DP: return "fused_wgrad_dp";
        case OP_DP_REDUCE: return "dp_reduce_sgd";
        case OP_BUMP_EPOCH: return "bump_epoch";
        case OP_BUMP_STEP: return "bump_step";
        case OP_DP_LL: return "dp_ll";
        case OP_PP_BUMP: return "pp_bump_epoch";
        case OP_PP_PUSH: return "pp_push";
        case OP_PP_WAIT: return "pp_wait";
        case OP_PP_CREDIT: return "pp_credit";
        case OP_CHAIN: return "mlp_chain";
        case OP_ARGMAX: return "argmax_correct";
        case OP_WAIT: return "wait_event";
        case OP_RECORD: return "record_event";
    }
    return "op";
}

// Eager plan walk.  SSB_NVTX=1 wraps every op in an NVTX range (one range per lowered pipe operation,
// visible in Nsight Systems); SSB_SERIALIZE=1 is the debugging mode that issues every op on the main
// stream (no cross-stream concurrency) - the first thing to try when a race is suspected
// (scripts/sanitize.sh runs compute-sanitizer racecheck / memcheck / synccheck on top of it).
//
// SSB_COMM_TIMING=1 (eager only) brackets with timing events (a) every communication op on its own
// stream  -> "busy" time of the links, and (b) every wait of a COMPUTE stream on an event recorded by a
// communication stream -> the time compute actually stalled on communication ("exposed").
void PipeEngine::walk(int set) {
    static const bool nvtx = getenv("SSB_NVTX") != nullptr;
    const bool timing = comm_timing_;
    std::vector<int> recorded_on;
    size_t next_ev = 0;
    auto tev = [&]() {
        if (next_ev == timing_events_.size()) {
            cudaEvent_t e;
            CUDA_CHECK(cudaEventCreate(&e));
            timing_events_.push_back(e);
        }
        return timing_events_[next_ev++];
    };
    if (timing) {
        recorded_on.assign(events_.size(), -1);
        exposed_pairs_.clear();
        busy_pairs_.clear();
    }
    auto is_comm_stream = [&](int s) { return s == s_comm_ || s == s_dp_; };
    for (const auto& op : ops_sets_[set]) {
        if (nvtx) nvtxRangePushA(op_name(op.kind));
        bool bracket = false, busy = false;
        if (timing) {
            if (op.kind == OP_RECORD) recorded_on[op.event] = op.stream;
            const bool comm_op = op.kind == OP_COMM_GROUP || op.kind == OP_ALLREDUCE || op.kind == OP_DP_REDUCE ||
                                 op.kind == OP_FUSED_DP || op.kind == OP_NVLS_SGD || op.kind == OP_PP_PUSH || op.kind == OP_PP_WAIT;
            busy = comm_op;
            bracket = comm_op || (op.kind == OP_WAIT && !is_comm_stream(op.stream) && recorded_on[op.event] >= 0 &&
                                  is_comm_stream(recorded_on[op.event]));
        }
        cudaEvent_t a = nullptr, b = nullptr;
        if (bracket) {
            a = tev();
            CUDA_CHECK(cudaEventRecord(a, stream_of(op)));
        }
        exec(op, set);
        if (bracket) {
            b = tev();
            CUDA_CHECK(cudaEventRecord(b, stream_of(op)));
            (busy ? busy_pairs_ : exposed_pairs_).push_back({a, b});
        }
        if (nvtx) nvtxRangePop();
    }
}

// (exposed_ms, busy_ms) of the most recent step walked with SSB_COMM_TIMING=1; synchronizes.
std::pair<double, double> PipeEngine::comm_timing() {
    synchronize();
    CUDA_CHECK(cudaDeviceSynchronize());
    double exposed = 0.0, busy = 0.0;
    float ms = 0.f;
    for (auto& pr : exposed_pairs_) { CUDA_CHECK(cudaEventElapsedTime(&ms, pr.first, pr.second)); exposed += ms; }
    for (auto& pr : busy_pairs_) { CUDA_CHECK(cudaEventElapsedTime(&ms, pr.first, pr.second)); busy += ms; }
    return {exposed, busy};
}

// Inputs of step i go into staging set i % 2 on the COPY stream; the compute graph of that set waits
// for the copy, and the next copy into the same set waits until that graph finished reading it.  The
// host enqueues step i + 1's copy while step i still computes, so H2D traffic hides behind compute.
void PipeEngine::stage_inputs(const float* x, const float* y) {
    const int set = fill_set_;
    const size_t rows = (size_t)cfg_.n_mu * cfg_.mb_rows;
    // cudaMemcpyDefault: the driver derives the direction per pointer (UVA), so x and y may live on different sides
    // (device-resident inputs with pinned-host targets, or the reverse)
    const cudaMemcpyKind kind = cudaMemcpyDefault;
    CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, ev_done_[set], 0));
    if (x != nullptr && cfg_.is_first)
        CUDA_CHECK(cudaMemcpy2DAsync(x_stage_sets_[set], (size_t)act_ld_[0] * 4, x, (size_t)cfg_.in_dim * 4, (size_t)cfg_.in_dim * 4,
                                     rows, kind, copy_stream_));
    if (y != nullptr && cfg_.is_last)
        CUDA_CHECK(cudaMemcpy2DAsync(y_stage_sets_[set], (size_t)y_ld_ * 4, y, (size_t)cfg_.out_dim * 4, (size_t)cfg_.out_dim * 4,
                                     rows, kind, copy_stream_));
    CUDA_CHECK(cudaEventRecord(ev_copy_[set], copy_stream_));
    staged_ = true;
}

// The shuffled counterpart of stage_inputs, with the same staging-set protocol: one gather launch on the copy stream picks
// global batch `batch`'s rows of this rank out of the device-resident dataset (x_all / y_all: [spec.n, in_dim / out_dim],
// nullptr where this stage takes no such input).  The spec travels by value, so the captured step graphs do not change.
void PipeEngine::stage_gather(const float* x_all, const float* y_all, const ShuffleSpec& spec, int batch) {
    const int set = fill_set_;
    const int rows = cfg_.n_mu * cfg_.mb_rows;
    const float* x = cfg_.is_first ? x_all : nullptr;
    const float* y = cfg_.is_last ? y_all : nullptr;
    CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, ev_done_[set], 0));
    if (x != nullptr || y != nullptr)   // a middle stage launches nothing
        CUDA_CHECK(launch_gather_rows(x, y, spec, batch, x_stage_sets_[set], act_ld_[0], y_stage_sets_[set], y_ld_, rows,
                                      cfg_.in_dim, cfg_.out_dim, copy_stream_));
    CUDA_CHECK(cudaEventRecord(ev_copy_[set], copy_stream_));
    staged_ = true;
}

void PipeEngine::run() {
    if (!built_) throw std::runtime_error("PipeEngine::run before build");
    const int set = fill_set_;
    // The update ops of this set read lr_dev_[set].  A new value is written by value (captured now, not read from host
    // memory later) on the copy stream, after the set's previous step - its last reader - and before ev_copy_[set],
    // which the step waits for.  With or without staging, that previous step is ev_done_[set].
    bool wait_copy = staged_;
    if (cfg_.training && lr_written_[set] != lr_) {
        uint32_t bits;
        memcpy(&bits, &lr_, sizeof(bits));
        CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, ev_done_[set], 0));
        cu_check(memset_d32_async()(reinterpret_cast<CUdeviceptr>(lr_dev_ + set), bits, 1, copy_stream_), "cuMemsetD32Async");
        CUDA_CHECK(cudaEventRecord(ev_copy_[set], copy_stream_));
        lr_written_[set] = lr_;
        wait_copy = true;
    }
    if (dropout_on() && step_written_[set] != step_) {   // the same protocol for the dropout step
        CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, ev_done_[set], 0));
        cu_check(memset_d32_async()(reinterpret_cast<CUdeviceptr>(step_dev_ + set), step_, 1, copy_stream_), "cuMemsetD32Async");
        CUDA_CHECK(cudaEventRecord(ev_copy_[set], copy_stream_));
        step_written_[set] = step_;
        wait_copy = true;
    }
    if (ema_on() && alpha_written_[set] != alpha_) {   // the same protocol for the EMA alpha
        uint32_t bits;
        memcpy(&bits, &alpha_, sizeof(bits));
        CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, ev_done_[set], 0));
        cu_check(memset_d32_async()(reinterpret_cast<CUdeviceptr>(alpha_dev_ + set), bits, 1, copy_stream_), "cuMemsetD32Async");
        CUDA_CHECK(cudaEventRecord(ev_copy_[set], copy_stream_));
        alpha_written_[set] = alpha_;
        wait_copy = true;
    }
    if (wait_copy) CUDA_CHECK(cudaStreamWaitEvent(streams_[0], ev_copy_[set], 0));
    if (graph_exec_sets_[set]) CUDA_CHECK(cudaGraphLaunch(graph_exec_sets_[set], streams_[0]));
    else walk(set);
    CUDA_CHECK(cudaEventRecord(ev_done_[set], streams_[0]));
    run_set_ = set;
    if (staged_) fill_set_ ^= 1;
    staged_ = false;
}

void PipeEngine::synchronize() { CUDA_CHECK(cudaStreamSynchronize(streams_[0])); }

// Failure detection: bounded wait for the step in flight.  Returns true when the main stream drained,
// false when `timeout_s` elapsed first (a peer died, a schedule bug, a lost NCCL message ...).  A sticky
// CUDA error (e.g. the __trap() of a device-flag spin that hit its own bound) surfaces as an exception.
bool PipeEngine::wait(double timeout_s) {
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        const cudaError_t e = cudaStreamQuery(streams_[0]);
        if (e == cudaSuccess) return true;
        if (e != cudaErrorNotReady) CUDA_CHECK(e);
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > timeout_s) return false;
        std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
}

// What the communicators know about a stalled step (ncclCommGetAsyncError), for the watchdog's report.
std::string PipeEngine::comm_status() const {
    std::ostringstream os;
    auto one = [&](const char* name, ncclComm_t c) {
        if (!c) return;
        ncclResult_t r = ncclSuccess;
        const ncclResult_t q = ncclCommGetAsyncError(c, &r);
        os << name << "=" << (q == ncclSuccess ? ncclGetErrorString(r) : ncclGetErrorString(q)) << " ";
    };
    one("pp_comm", pp_comm_);
    one("dp_comm", dp_comm_);
    return os.str();
}

float PipeEngine::last_loss() {
    synchronize();
    const float* h = loss_slot(run_set_);
    float s = 0.f;
    for (int i = 0; i < cfg_.n_mu; ++i) s += h[i];
    return s;
}

// Loss of the step BEFORE the most recently launched one: waits only for that step's event, so the
// GPU queue stays non-empty (H2D of step i+1 / compute of step i / D2H of step i-1 overlap).
float PipeEngine::prev_loss() {
    const int set = run_set_ ^ 1;
    CUDA_CHECK(cudaEventSynchronize(ev_done_[set]));
    const float* h = loss_slot(set);
    float s = 0.f;
    for (int i = 0; i < cfg_.n_mu; ++i) s += h[i];
    return s;
}

int PipeEngine::count_correct() {
    int v = 0;
    CUDA_CHECK(cudaMemcpyAsync(&v, correct_dev_, sizeof(int), cudaMemcpyDeviceToHost, streams_[0]));
    synchronize();
    return v;
}
void PipeEngine::reset_correct() { CUDA_CHECK(cudaMemsetAsync(correct_dev_, 0, sizeof(int), streams_[0])); }

std::vector<unsigned long long> PipeEngine::chain_timeline() {
    std::vector<unsigned long long> v(4 * 256, 0);
    if (chain_dbg_) {
        synchronize();
        CUDA_CHECK(cudaMemcpy(v.data(), chain_dbg_, v.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    }
    return v;
}

// One line per lowered op of staging set `set`: "<index> <op> stream=<s> [event=<e>] [layer=<l>] [mu=<m>]" - the plan a
// step replays, for debugging and for the plan self-check in the tests.
std::string PipeEngine::plan_text(int set) const {
    std::ostringstream os;
    const auto& ops = ops_sets_[set & 1];
    for (size_t i = 0; i < ops.size(); ++i) {
        const Op& op = ops[i];
        os << i << " " << op_name(op.kind) << " stream=" << op.stream;
        if (op.event >= 0) os << " event=" << op.event;
        if (op.layer >= 0) os << " layer=" << op.layer;
        if (op.mu >= 0) os << " mu=" << op.mu;
        if (op.kind == OP_GEMM) {                      // the variant a GEMM launches beyond the plain one
            const GemmPlan& g = gemms_[op.gemm];
            if (g.p.k_splits > 1) os << " splits=" << g.p.k_splits;
            if (gemm_drops(g)) os << " drop=" << (g.mode == GEMM_FWD ? "fwd" : "dgrad");
            if (gemm_gated(g)) os << " act=" << act_name(g.p.act_kind);
            if (gemm_skips(g)) os << " res=1";
        }
        if (op.kind == OP_RELU_MASK && op.dropout) os << " drop=scaled";
        if (op.kind == OP_RELU_MASK && op.gated) os << " act=" << act_name(cfg_.activation);
        if (op.kind == OP_RELU_MASK && op.c != nullptr) os << " res=1";
        if (op.kind == OP_CHAIN && act_smooth(cfg_.activation)) os << " act=" << act_name(cfg_.activation);
        if (op.kind == OP_CHAIN && cfg_.residual) os << " res=1";
        if (op.kind == OP_COMM_GROUP) {
            os << " [";
            for (const auto& it : op.comm) os << (it.is_send ? "send->" : "recv<-") << it.peer << ":" << it.count << " ";
            os << "]";
        }
        os << "\n";
    }
    return os.str();
}

std::string PipeEngine::describe() const {
    std::ostringstream os;
    os << "PipeEngine(stage " << cfg_.stage << "/" << cfg_.n_stages << ", layers=" << L_ << ", mb_rows=" << cfg_.mb_rows
       << ", n_mu=" << cfg_.n_mu << ", ops=" << ops_sets_[0].size() << ", kernels/step=" << kernels_per_step_
       << ", graph_nodes=" << graph_nodes_ << ", splitk_gemms=" << splitk_gemms_ << ", streams=" << streams_.size() << ", events=" << events_.size();
    if (cfg_.training) {
        os << ", update=sgd(lr=" << lr_;
        if (cfg_.momentum != 0.f) os << ", momentum=" << cfg_.momentum << (cfg_.nesterov ? ", nesterov" : "");
        if (cfg_.weight_decay != 0.f) os << ", weight_decay=" << cfg_.weight_decay;
        if (ema_on()) os << ", ema=" << cfg_.ema_decay;
        os << ")";
    }
    if (cfg_.loss == LOSS_CROSS_ENTROPY) os << ", loss=cross_entropy";
    os << ")";
    return os.str();
}

}  // namespace ssb
