// pybind11 face of the native runtime: NCCL communicators + PipeEngine.
#include <torch/extension.h>
#include <pybind11/stl.h>
#include <c10/cuda/CUDAGuard.h>
#include <nccl.h>

#include "runtime/nvls_context.h"
#include "runtime/pipe_engine.h"

namespace py = pybind11;

namespace ssb {

#define NCCL_OK(expr)                                                                              \
    do {                                                                                           \
        ncclResult_t _r = (expr);                                                                  \
        TORCH_CHECK(_r == ncclSuccess, "NCCL error: ", ncclGetErrorString(_r), " at " #expr);      \
    } while (0)

// Own NCCL communicator (not torch's ProcessGroup): the C++ executor issues ncclSend/Recv/
// AllReduce itself on its own streams, inside CUDA-graph capture.
class NcclComm {
public:
    static py::bytes unique_id() {
        ncclUniqueId id;
        NCCL_OK(ncclGetUniqueId(&id));
        return py::bytes(reinterpret_cast<const char*>(&id), sizeof(id));
    }
    NcclComm(const std::string& id_bytes, int nranks, int rank) : nranks_(nranks), rank_(rank) {
        TORCH_CHECK(id_bytes.size() == sizeof(ncclUniqueId), "bad ncclUniqueId size");
        ncclUniqueId id;
        memcpy(&id, id_bytes.data(), sizeof(id));
        NCCL_OK(ncclCommInitRank(&comm_, nranks, id, rank));
    }
    ~NcclComm() {
        if (comm_) ncclCommDestroy(comm_);
    }
    // open the channels now so the first captured step does not pay for it
    void warmup() {
        float* buf = nullptr;
        cudaMalloc(&buf, 1024);
        cudaMemset(buf, 0, 1024);
        NCCL_OK(ncclAllReduce(buf, buf, 256, ncclFloat, ncclSum, comm_, nullptr));
        if (nranks_ > 1) {
            NCCL_OK(ncclGroupStart());
            const int next = (rank_ + 1) % nranks_, prev = (rank_ + nranks_ - 1) % nranks_;
            NCCL_OK(ncclSend(buf, 64, ncclFloat, next, comm_, nullptr));
            NCCL_OK(ncclRecv(buf + 128, 64, ncclFloat, prev, comm_, nullptr));
            NCCL_OK(ncclGroupEnd());
        }
        cudaStreamSynchronize(nullptr);
        cudaFree(buf);
    }
    // failure handling: async error state, and a non-blocking teardown that also unblocks the peers
    std::string async_error() {
        ncclResult_t r = ncclSuccess;
        NCCL_OK(ncclCommGetAsyncError(comm_, &r));
        return r == ncclSuccess ? std::string() : std::string(ncclGetErrorString(r));
    }
    void abort() {
        if (comm_) ncclCommAbort(comm_);
        comm_ = nullptr;
    }
    ncclComm_t get() const { return comm_; }
    int nranks() const { return nranks_; }
    int rank() const { return rank_; }

private:
    ncclComm_t comm_ = nullptr;
    int nranks_, rank_;
};

static torch::Tensor view_of(float* ptr, int64_t rows, int64_t cols, int64_t ld) {
    int dev = 0;
    cudaGetDevice(&dev);
    auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, dev);
    return torch::from_blob(ptr, {rows, cols}, {ld, 1}, [](void*) {}, opts);
}

class PyDpContext {
public:
    PyDpContext(int dp, int rank, int64_t arena_numel, const std::vector<std::tuple<int, int, int64_t, int>>& layers, double lr)
        : ctx_(std::make_unique<DpContext>(dp, rank, arena_numel, layers, (float)lr)) {}
    py::bytes export_handles() { return py::bytes(ctx_->export_handles()); }
    void open_peers(const std::vector<std::string>& handles) { ctx_->open_peers(handles); }
    torch::Tensor weights() {
        int dev = 0;
        cudaGetDevice(&dev);
        auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, dev);
        return torch::from_blob(ctx_->weights(), {ctx_->arena_numel()}, [](void*) {}, opts);
    }
    int64_t stage_bytes() { return ctx_->stage_bytes(); }
    // test-facing: peers that live in this process (index = DP rank, own entry ignored; None allowed there)
    void open_local_peers(const std::vector<std::shared_ptr<PyDpContext>>& ctxs) {
        std::vector<const DpContext*> raw;
        for (const auto& c : ctxs) raw.push_back(c ? c->ctx_.get() : nullptr);
        ctx_->open_local_peers(raw);
    }
    // test-facing: {name: (device pointer, bytes)} of every buffer a peer reads or writes (llA / llC: (0, 0) without
    // LL landing zones)
    py::dict buffers() {
        const DpContext& c = *ctx_;
        py::dict d;
        auto put = [&](const char* name, const void* p, int64_t bytes) {
            d[name] = py::make_tuple((int64_t) reinterpret_cast<uintptr_t>(p), bytes);
        };
        put("W", c.weights(), c.arena_numel() * 4);
        put("stage", c.stage(), c.stage_bytes());
        put("arrive", c.arrive(), c.arrive_bytes());
        put("done", c.done(), c.done_bytes());
        put("epoch", c.epoch_ptr(), 64);
        put("llA", c.ll_a(), c.ll_zone_bytes());
        put("llC", c.ll_c(), c.ll_zone_bytes());
        return d;
    }
    // test-facing: per layer, the geometry that addresses its staging slots and flags
    py::list layer_geometry() {
        const DpContext& c = *ctx_;
        py::list out;
        for (const DpLayerGeom& g : c.geometry()) {
            py::dict d;
            d["in"] = g.in; d["out"] = g.out; d["ld"] = g.ld; d["w_offset"] = g.w_offset;
            d["block_n"] = g.block_n; d["n_tiles_m"] = g.n_tiles_m; d["n_tiles_n"] = g.n_tiles_n;
            d["slots"] = g.slots; d["slot_floats"] = g.slot_floats; d["stage_offset"] = g.stage_offset;
            d["tile_flag_base"] = g.tile_flag_base; d["slot_flag_base"] = g.slot_flag_base; d["one_shot"] = g.one_shot;
            d["slots_per_src"] = c.slots_per_src(); d["stage_src_stride"] = c.stage_src_stride();
            d["stage_parity_stride"] = c.stage_parity_stride();
            out.append(d);
        }
        return out;
    }
    int dp() { return ctx_->dp(); }
    int rank() { return ctx_->rank(); }
    int ll_tiles() { return ctx_->ll_tiles(); }
    DpContext* get() { return ctx_.get(); }

private:
    std::unique_ptr<DpContext> ctx_;
};

// NVLS symmetric memory (multicast object shared by the DP replicas); see runtime/nvls_context.h
class PyNvlsContext {
public:
    PyNvlsContext(int dp, int rank, int64_t arena_numel, double lr, int devices)
        : ctx_(std::make_unique<NvlsContext>(dp, rank, arena_numel, (float)lr, devices)) {}
    explicit PyNvlsContext(std::unique_ptr<NvlsContext> ctx) : ctx_(std::move(ctx)) {}
    static bool supported() { return NvlsContext::supported(); }
    // test-facing: a member of a local team (plain device memory of this process, the kernels' replay transport)
    static std::shared_ptr<PyNvlsContext> local(int dp, int rank, int64_t arena_numel) {
        return std::make_shared<PyNvlsContext>(NvlsContext::local(dp, rank, arena_numel));
    }
    // test-facing: every member of the team, rank order, this one included
    void open_local(const std::vector<std::shared_ptr<PyNvlsContext>>& team) {
        std::vector<const NvlsContext*> raw;
        for (const auto& c : team) raw.push_back(c ? c->ctx_.get() : nullptr);
        ctx_->open_local(raw);
    }
    // test-facing: {name: (device pointer, bytes)} of this member's W and G (numel_pad floats each), its two flag words,
    // the epoch and the last-CTA counter
    py::dict buffers() {
        const NvlsContext& c = *ctx_;
        py::dict d;
        auto put = [&](const char* name, const void* p, int64_t bytes) {
            d[name] = py::make_tuple((int64_t) reinterpret_cast<uintptr_t>(p), bytes);
        };
        put("W", c.weights(), c.numel_pad() * 4);
        put("G", c.grads(), c.numel_pad() * 4);
        put("flag_in", c.flag_in(), 4);
        put("flag_out", c.flag_out(), 4);
        put("epoch", c.epoch_ptr(), 4);
        put("cta_done", c.cta_done_ptr(), 4);
        return d;
    }
    int64_t arena_numel() { return ctx_->arena_numel(); }
    int64_t numel_pad() { return ctx_->numel_pad(); }
    int dp() { return ctx_->dp(); }
    int rank() { return ctx_->rank(); }
    int export_fd() { return ctx_->export_fd(); }
    void import_fd(int fd) { ctx_->import_fd(fd); }
    void add_device() { ctx_->add_device(); }
    void bind_and_map() { ctx_->bind_and_map(); }
    torch::Tensor weights() { return blob(ctx_->weights()); }
    torch::Tensor grads() { return blob(ctx_->grads()); }
    int64_t bytes() { return (int64_t)ctx_->bytes(); }
    // stand-alone collectives on the current torch stream (tests / link benchmark)
    void all_reduce_grads() {
        TORCH_CHECK(launch_nvls_allreduce(ctx_->params(), num_sms(), c10::cuda::getCurrentCUDAStream()) == cudaSuccess, "nvls allreduce launch");
    }
    // lr: one-element fp32 tensor on this device, read by the kernel when it runs
    void reduce_sgd(const torch::Tensor& lr) {
        TORCH_CHECK(lr.is_cuda() && lr.scalar_type() == torch::kFloat32 && lr.numel() == 1, "reduce_sgd: lr must be a one-element fp32 CUDA tensor");
        NvlsParams p = ctx_->params();
        p.lr = lr.data_ptr<float>();
        TORCH_CHECK(launch_nvls_reduce_sgd(p, num_sms(), c10::cuda::getCurrentCUDAStream()) == cudaSuccess, "nvls reduce_sgd launch");
    }
    NvlsContext* get() { return ctx_.get(); }

private:
    static int num_sms() {
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        return sms;
    }
    torch::Tensor blob(float* p) {
        int dev = 0;
        cudaGetDevice(&dev);
        auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, dev);
        return torch::from_blob(p, {ctx_->arena_numel()}, [](void*) {}, opts);
    }
    std::unique_ptr<NvlsContext> ctx_;
};

// Peer-memory pipeline transport (runtime/pp_context.h)
class PyPpContext {
public:
    PyPpContext(int n_mu, int mb_rows, int ld_in, int ld_out, bool is_first, bool is_last)
        : ctx_(std::make_unique<PpContext>(n_mu, mb_rows, ld_in, ld_out, is_first, is_last)) {}
    py::bytes export_handles() { return py::bytes(ctx_->export_handles()); }
    void open_prev(const std::string& h) { ctx_->open_prev(h); }
    void open_next(const std::string& h) { ctx_->open_next(h); }
    // test-facing: neighbours that live in this process (None: no such neighbour)
    void open_local(const std::shared_ptr<PyPpContext>& prev, const std::shared_ptr<PyPpContext>& next) {
        ctx_->open_local(prev ? prev->ctx_.get() : nullptr, next ? next->ctx_.get() : nullptr);
    }
    // test-facing: {name: (device pointer, bytes)} of the receive slots, the epoch, the push completion counter, the whole
    // flag array and its named word ranges
    py::dict buffers() {
        const PpContext& c = *ctx_;
        py::dict d;
        auto put = [&](const char* name, const void* p, int64_t bytes) {
            d[name] = py::make_tuple((int64_t) reinterpret_cast<uintptr_t>(p), bytes);
        };
        const int64_t slots = (int64_t)c.n_mu() * c.mb_rows() * sizeof(float);
        put("act_in", c.act_in(), slots * c.ld_in());
        put("dz_in", c.dz_in(), slots * c.ld_out());
        put("epoch", c.epoch_ptr(), 64);
        put("push_done", c.push_done_ptr(), 64);
        put("flags", c.flags(), PpContext::kFlagWords * 4);
        put("act_arrived", c.act_arrived(0), PpContext::kMaxMu * 4);
        put("dz_arrived", c.dz_arrived(0), PpContext::kMaxMu * 4);
        put("act_credit", c.act_credit(), 4);
        put("dz_credit", c.dz_credit(), 4);
        return d;
    }
    PpContext* get() { return ctx_.get(); }

private:
    std::unique_ptr<PpContext> ctx_;
};

class PyEngine {
public:
    PyEngine(const std::vector<std::tuple<int, int, int, int64_t, int>>& layers, py::dict cfg, torch::Tensor weights,
             torch::Tensor grads, c10::optional<torch::Tensor> momentum, c10::optional<torch::Tensor> ema)
        : weights_(weights), grads_(grads), momentum_(momentum), ema_(ema) {
        TORCH_CHECK(weights.is_cuda() && grads.is_cuda() && weights.is_contiguous() && grads.is_contiguous());
        TORCH_CHECK(weights.scalar_type() == torch::kFloat32 && grads.scalar_type() == torch::kFloat32);
        if (momentum.has_value())
            TORCH_CHECK(momentum->is_cuda() && momentum->is_contiguous() && momentum->scalar_type() == torch::kFloat32 &&
                            momentum->numel() >= weights.numel() && momentum->device() == weights.device(),
                        "PipeEngine: the momentum arena must be a contiguous fp32 CUDA buffer covering the weight arena");
        if (ema.has_value())
            TORCH_CHECK(ema->is_cuda() && ema->is_contiguous() && ema->scalar_type() == torch::kFloat32 &&
                            ema->numel() >= weights.numel() && ema->device() == weights.device(),
                        "PipeEngine: the EMA arena must be a contiguous fp32 CUDA buffer covering the weight arena");
        EngineConfig c;
        for (auto& t : layers) c.layers.push_back({std::get<0>(t), std::get<1>(t), std::get<2>(t), std::get<3>(t), std::get<4>(t)});
        auto geti = [&](const char* k, int dflt) { return cfg.contains(k) ? cfg[k].cast<int>() : dflt; };
        c.is_first = geti("is_first", 1); c.is_last = geti("is_last", 1);
        c.stage = geti("stage", 0); c.n_stages = geti("n_stages", 1);
        c.mb_rows = geti("mb_rows", 32); c.n_mu = geti("n_mu", 4); c.global_batch = geti("global_batch", 128);
        c.lr = cfg.contains("lr") ? cfg["lr"].cast<float>() : 0.006f;
        c.training = geti("training", 1); c.use_graph = geti("use_graph", 1);
        c.dp_size = geti("dp_size", 1); c.dp_rank = geti("dp_rank", 0); c.dp_mode = geti("dp_mode", 0);
        c.in_dim = geti("in_dim", 784); c.out_dim = geti("out_dim", 10);
        c.prec = geti("prec", ssb::PREC_TF32);
        TORCH_CHECK(ssb::prec_valid(c.prec), "PipeEngine: cfg['prec'] must be 0 (tf32), 1 (3xtf32) or 2 (bf16), got ", c.prec);
        c.momentum = cfg.contains("momentum") ? cfg["momentum"].cast<float>() : 0.f;
        c.weight_decay = cfg.contains("weight_decay") ? cfg["weight_decay"].cast<float>() : 0.f;
        c.nesterov = geti("nesterov", 0);
        c.ema_decay = cfg.contains("ema_decay") ? cfg["ema_decay"].cast<float>() : 0.f;
        TORCH_CHECK(c.ema_decay == 0.f || (c.ema_decay > 0.f && c.ema_decay < 1.f),
                    "PipeEngine: cfg['ema_decay'] must be in (0, 1), got ", c.ema_decay);
        TORCH_CHECK((c.ema_decay > 0.f) == ema.has_value(), "PipeEngine: an EMA arena is needed exactly when cfg['ema_decay'] is set");
        c.loss = geti("loss", ssb::LOSS_MSE);
        TORCH_CHECK(c.loss == ssb::LOSS_MSE || c.loss == ssb::LOSS_CROSS_ENTROPY,
                    "PipeEngine: cfg['loss'] must be 0 (MSE) or 1 (cross-entropy), got ", c.loss);
        c.dropout = cfg.contains("dropout") ? cfg["dropout"].cast<double>() : 0.0;
        TORCH_CHECK(c.dropout >= 0.0 && c.dropout < 1.0, "PipeEngine: cfg['dropout'] must be in [0, 1), got ", c.dropout);
        c.dropout_seed = cfg.contains("dropout_seed") ? cfg["dropout_seed"].cast<uint64_t>() : 0;
        c.layer_base = geti("layer_base", 0);
        c.activation = geti("activation", ssb::ACT_RELU);
        TORCH_CHECK(ssb::act_valid(c.activation), "PipeEngine: cfg['activation'] must be 0 (relu), 1 (gelu), 2 (silu) or 3 (tanh), got ",
                    c.activation);
        if (cfg.contains("residual")) {   // one 0 / 1 per layer: an identity skip around it
            const auto res = cfg["residual"].cast<std::vector<int>>();
            TORCH_CHECK(res.size() == c.layers.size(), "PipeEngine: cfg['residual'] needs one entry per layer");
            for (size_t l = 0; l < res.size(); ++l) {
                const ssb::LayerSpec& ls = c.layers[l];
                TORCH_CHECK(!res[l] || (ls.relu && ls.in == ls.out),
                            "PipeEngine: a residual layer needs an activation and as many outputs as inputs (layer ", l + 1, ")");
                c.layers[l].res = res[l] ? 1 : 0;
                c.residual |= c.layers[l].res;
            }
        }
        c10::cuda::CUDAGuard guard(weights.device());
        engine_ = std::make_unique<PipeEngine>(c, weights.data_ptr<float>(), grads.data_ptr<float>(), weights.numel(),
                                               momentum.has_value() ? momentum->data_ptr<float>() : nullptr,
                                               ema.has_value() ? ema->data_ptr<float>() : nullptr);
    }
    void set_pp_comm(std::shared_ptr<NcclComm> c) { pp_ = c; engine_->set_pp_comm(c->get()); }
    void set_dp_comm(std::shared_ptr<NcclComm> c) { dp_ = c; engine_->set_dp_comm(c->get()); }
    void set_dp_context(std::shared_ptr<PyDpContext> c) { dpctx_ = c; engine_->set_dp_context(c->get()); }
    void set_nvls_context(std::shared_ptr<PyNvlsContext> c) { nvls_ = c; engine_->set_nvls_context(c->get()); }
    void set_pp_context(std::shared_ptr<PyPpContext> c) { ppctx_ = c; engine_->set_pp_context(c->get()); }
    std::pair<int, int> boundary_lds() { return {engine_->act_ld(0), engine_->act_ld((int)engine_->config().layers.size())}; }
    void build(const std::vector<std::tuple<int, int, int>>& instrs) {
        c10::cuda::CUDAGuard guard(weights_.device());
        engine_->build(instrs);
    }
    void stage_inputs(const c10::optional<torch::Tensor>& x, const c10::optional<torch::Tensor>& y) {
        const auto& cfg = engine_->config();
        const int64_t rows = (int64_t)cfg.n_mu * cfg.mb_rows;
        const float *xp = nullptr, *yp = nullptr;
        if (x.has_value()) {
            TORCH_CHECK(x->is_contiguous() && x->scalar_type() == torch::kFloat32 && x->numel() == rows * cfg.in_dim, "x shape");
            xp = x->data_ptr<float>();
        }
        if (y.has_value()) {
            TORCH_CHECK(y->is_contiguous() && y->scalar_type() == torch::kFloat32 && y->numel() == rows * cfg.out_dim, "y shape");
            yp = y->data_ptr<float>();
        }
        engine_->stage_inputs(xp, yp);
        // the copies are asynchronous: keep the source tensors alive until a later staging call of the same set
        // (which first waits for this set's compute, hence for these copies) replaces them
        held_[hold_i_ & 1] = {x, y};
        ++hold_i_;
    }
    // shuffled staging (PipeEngine::stage_gather): x_all [n, in_dim] / y_all [n, out_dim], the whole dataset on this
    // engine's device (each is ignored by a stage that does not take it); rows of global batch `batch` of DP rank `rank`
    // under the epoch's permutation
    void stage_gather(const c10::optional<torch::Tensor>& x_all, const c10::optional<torch::Tensor>& y_all, uint64_t seed,
                      int64_t epoch, int64_t gbs, int64_t dp, int64_t rank, int64_t batch) {
        const auto& cfg = engine_->config();
        const int64_t rows = (int64_t)cfg.n_mu * cfg.mb_rows;
        int64_t n = -1;
        const float *xp = nullptr, *yp = nullptr;
        auto check = [&](const torch::Tensor& t, int64_t cols, const char* name) {
            TORCH_CHECK(t.is_cuda() && t.device() == weights_.device(), "stage_gather: ", name, " must live on the engine's device");
            TORCH_CHECK(t.scalar_type() == torch::kFloat32 && t.is_contiguous() && t.dim() == 2 && t.size(1) == cols,
                        "stage_gather: ", name, " must be a dense fp32 [n, ", cols, "] tensor");
            TORCH_CHECK(n < 0 || t.size(0) == n, "stage_gather: x and y hold different numbers of rows");
            n = t.size(0);
        };
        // like stage_inputs, a stage ignores the source it does not take (x unless first, y unless last)
        if (x_all.has_value() && cfg.is_first) { check(*x_all, cfg.in_dim, "x"); xp = x_all->data_ptr<float>(); }
        if (y_all.has_value() && cfg.is_last) { check(*y_all, cfg.out_dim, "y"); yp = y_all->data_ptr<float>(); }
        TORCH_CHECK(n < (int64_t(1) << 32) && epoch >= 0 && gbs < (1 << 30) && dp < (1 << 30) && batch < (1 << 30),
                    "stage_gather: argument out of range");
        const ShuffleSpec spec{(uint32_t)std::max<int64_t>(n, 0), seed, (uint32_t)(epoch & 0xffffffffLL), (int)gbs, (int)dp,
                               (int)rank};
        if (n >= 0) {   // a stage without inputs gathers nothing (it only keeps the staging-set protocol)
            const char* err = shuffle_spec_check(spec, (int)batch, (int)rows);
            TORCH_CHECK(err == nullptr, "stage_gather: ", err ? err : "");
        }
        engine_->stage_gather(xp, yp, spec, (int)batch);
        held_[hold_i_ & 1] = {x_all, y_all};   // the gather is asynchronous, like the copies of stage_inputs
        ++hold_i_;
    }
    // test-facing: the two staging buffers of set `set`, over their whole row pitch (x [rows, act ld 0], y [rows, y ld])
    std::pair<torch::Tensor, torch::Tensor> staging(int set) {
        const auto& cfg = engine_->config();
        TORCH_CHECK(set == 0 || set == 1, "PipeEngine.staging: set must be 0 or 1");
        const int64_t rows = (int64_t)cfg.n_mu * cfg.mb_rows;
        return {view_of(engine_->x_staging_set(set), rows, engine_->act_ld(0), engine_->act_ld(0)),
                view_of(engine_->y_staging_set(set), rows, engine_->y_ld(), engine_->y_ld())};
    }
    int fill_set() { return engine_->fill_set(); }
    int n_mubatches() { return engine_->config().n_mu; }
    void run() { engine_->run(); }
    void set_lr(double lr) {
        TORCH_CHECK(std::isfinite(lr) && lr >= 0.0, "PipeEngine.set_lr: the learning rate must be finite and >= 0, got ", lr);
        engine_->set_lr((float)lr);
    }
    float lr() { return engine_->lr(); }
    void set_ema_alpha(double alpha) {
        TORCH_CHECK(alpha > 0.0 && alpha <= 1.0, "PipeEngine.set_ema_alpha: alpha must be in (0, 1], got ", alpha);
        engine_->set_ema_alpha((float)alpha);
    }
    void set_dropout_step(int64_t step) {
        TORCH_CHECK(step >= 0, "PipeEngine.set_dropout_step: the step must be >= 0, got ", step);
        engine_->set_dropout_step((uint32_t)(step & 0xffffffffLL));   // the masks' step counter is the step mod 2^32
    }
    void synchronize() { engine_->synchronize(); }
    bool wait(double timeout_s) {
        py::gil_scoped_release nogil;
        return engine_->wait(timeout_s);
    }
    std::string comm_status() { return engine_->comm_status(); }
    std::pair<double, double> comm_timing() { return engine_->comm_timing(); }
    bool comm_timing_enabled() { return engine_->comm_timing_enabled(); }
    float last_loss() { return engine_->last_loss(); }
    float prev_loss() { return engine_->prev_loss(); }
    int count_correct() { return engine_->count_correct(); }
    void reset_correct() { engine_->reset_correct(); }
    torch::Tensor act(int mu, int l) {
        const auto& cfg = engine_->config();
        return view_of(engine_->act_ptr(mu, l), cfg.mb_rows, boundary_cols(l), engine_->act_ld(l));
    }
    torch::Tensor dz(int mu, int l) {
        const auto& cfg = engine_->config();
        return view_of(engine_->dz_ptr(mu, l), cfg.mb_rows, boundary_cols(l), engine_->act_ld(l));
    }
    // the gates f'(z) * keep * s of layer l's output (a gated training plan's activated layers only)
    torch::Tensor gate(int mu, int l) {
        const auto& cfg = engine_->config();
        float* g = engine_->gate_ptr(mu, l);
        TORCH_CHECK(g != nullptr, "PipeEngine.gate: layer ", l, " has no gate buffer (ReLU, inference, or no activation)");
        return view_of(g, cfg.mb_rows, boundary_cols(l), engine_->act_ld(l));
    }
    // the skip gradient dL/da of residual layer l's output (a residual training plan only)
    torch::Tensor g(int mu, int l) {
        const auto& cfg = engine_->config();
        float* p = engine_->g_ptr(mu, l);
        TORCH_CHECK(p != nullptr, "PipeEngine.g: layer ", l, " has no skip-gradient buffer (not residual, or inference)");
        return view_of(p, cfg.mb_rows, boundary_cols(l), engine_->act_ld(l));
    }
    torch::Tensor probs(int mu) {
        const auto& cfg = engine_->config();
        return view_of(engine_->probs_ptr(mu), cfg.mb_rows, cfg.out_dim, engine_->act_ld((int)cfg.layers.size()));
    }
    int64_t kernels_per_step() { return engine_->kernels_per_step(); }
    int64_t graph_nodes() { return engine_->graph_nodes(); }
    bool uses_chain() { return engine_->uses_chain(); }
    int chain_cluster() { return engine_->chain_cluster(); }
    int chain_ksplit() { return engine_->chain_ksplit(); }
    bool coalesced() { return engine_->coalesced(); }
    int64_t main_stream() { return reinterpret_cast<int64_t>(engine_->main_stream()); }
    std::string describe() { return engine_->describe(); }
    std::vector<int> layer_protocols() { return engine_->layer_protocols(); }
    std::string plan_text(int set) { return engine_->plan_text(set); }
    std::vector<unsigned long long> chain_timeline() { return engine_->chain_timeline(); }

private:
    // features at layer boundary l (l = 0: the stage's input; a stage without Linears has only that one, in_dim wide)
    int boundary_cols(int l) const {
        const auto& cfg = engine_->config();
        TORCH_CHECK(l >= 0 && l <= (int)cfg.layers.size(), "PipeEngine: layer boundary ", l, " out of range");
        if (l > 0) return cfg.layers[l - 1].out;
        return cfg.layers.empty() ? cfg.in_dim : cfg.layers[0].in;
    }
    torch::Tensor weights_, grads_;
    c10::optional<torch::Tensor> momentum_;   // kept alive: the plan holds raw pointers into it
    c10::optional<torch::Tensor> ema_;        // the same
    std::pair<c10::optional<torch::Tensor>, c10::optional<torch::Tensor>> held_[2];
    unsigned hold_i_ = 0;
    std::shared_ptr<NcclComm> pp_, dp_;
    std::shared_ptr<PyDpContext> dpctx_;
    std::shared_ptr<PyNvlsContext> nvls_;
    std::shared_ptr<PyPpContext> ppctx_;
    std::unique_ptr<PipeEngine> engine_;
};

void bind_runtime(py::module_& m) {
    py::class_<NcclComm, std::shared_ptr<NcclComm>>(m, "NcclComm")
        .def_static("unique_id", &NcclComm::unique_id)
        .def(py::init<const std::string&, int, int>())
        .def("warmup", &NcclComm::warmup)
        .def("async_error", &NcclComm::async_error)
        .def("abort", &NcclComm::abort)
        .def("nranks", &NcclComm::nranks)
        .def("rank", &NcclComm::rank);
    py::class_<PyDpContext, std::shared_ptr<PyDpContext>>(m, "DpContext")
        .def(py::init<int, int, int64_t, const std::vector<std::tuple<int, int, int64_t, int>>&, double>())
        .def("export_handles", &PyDpContext::export_handles)
        .def("open_peers", &PyDpContext::open_peers)
        .def("weights", &PyDpContext::weights)
        .def("stage_bytes", &PyDpContext::stage_bytes)
        .def("open_local_peers", &PyDpContext::open_local_peers)
        .def("buffers", &PyDpContext::buffers)
        .def("layer_geometry", &PyDpContext::layer_geometry)
        .def("dp", &PyDpContext::dp)
        .def("rank", &PyDpContext::rank)
        .def("ll_tiles", &PyDpContext::ll_tiles);
    py::class_<PyNvlsContext, std::shared_ptr<PyNvlsContext>>(m, "NvlsContext")
        .def(py::init<int, int, int64_t, double, int>(), py::arg("dp"), py::arg("rank"), py::arg("arena_numel"), py::arg("lr"),
             py::arg("devices") = 0)
        .def_static("supported", &PyNvlsContext::supported)
        .def_static("local", &PyNvlsContext::local, py::arg("dp"), py::arg("rank"), py::arg("arena_numel"))
        .def("open_local", &PyNvlsContext::open_local)
        .def("buffers", &PyNvlsContext::buffers)
        .def("arena_numel", &PyNvlsContext::arena_numel)
        .def("numel_pad", &PyNvlsContext::numel_pad)
        .def("dp", &PyNvlsContext::dp)
        .def("rank", &PyNvlsContext::rank)
        .def("export_fd", &PyNvlsContext::export_fd)
        .def("import_fd", &PyNvlsContext::import_fd)
        .def("add_device", &PyNvlsContext::add_device)
        .def("bind_and_map", &PyNvlsContext::bind_and_map)
        .def("weights", &PyNvlsContext::weights)
        .def("grads", &PyNvlsContext::grads)
        .def("bytes", &PyNvlsContext::bytes)
        .def("all_reduce_grads", &PyNvlsContext::all_reduce_grads)
        .def("reduce_sgd", &PyNvlsContext::reduce_sgd, py::arg("lr"));
    py::class_<PyPpContext, std::shared_ptr<PyPpContext>>(m, "PpContext")
        .def(py::init<int, int, int, int, bool, bool>())
        .def("export_handles", &PyPpContext::export_handles)
        .def("open_prev", &PyPpContext::open_prev)
        .def("open_next", &PyPpContext::open_next)
        .def("open_local", &PyPpContext::open_local, py::arg("prev"), py::arg("next"))
        .def("buffers", &PyPpContext::buffers);
    py::class_<PyEngine>(m, "PipeEngine")
        .def(py::init<const std::vector<std::tuple<int, int, int, int64_t, int>>&, py::dict, torch::Tensor, torch::Tensor,
                      c10::optional<torch::Tensor>, c10::optional<torch::Tensor>>(),
             py::arg("layers"), py::arg("cfg"), py::arg("weights"), py::arg("grads"), py::arg("momentum") = py::none(),
             py::arg("ema") = py::none())
        .def("set_pp_comm", &PyEngine::set_pp_comm)
        .def("set_dp_comm", &PyEngine::set_dp_comm)
        .def("set_dp_context", &PyEngine::set_dp_context)
        .def("set_nvls_context", &PyEngine::set_nvls_context)
        .def("set_pp_context", &PyEngine::set_pp_context)
        .def("boundary_lds", &PyEngine::boundary_lds)
        .def("build", &PyEngine::build)
        .def("stage_inputs", &PyEngine::stage_inputs)
        .def("stage_gather", &PyEngine::stage_gather, py::arg("x_all"), py::arg("y_all"), py::arg("seed"), py::arg("epoch"),
             py::arg("gbs"), py::arg("dp"), py::arg("rank"), py::arg("batch"))
        .def("staging", &PyEngine::staging, py::arg("set"))
        .def("fill_set", &PyEngine::fill_set)
        .def("n_mubatches", &PyEngine::n_mubatches)
        .def("run", &PyEngine::run)
        .def("set_lr", &PyEngine::set_lr, py::arg("lr"))
        .def("lr", &PyEngine::lr)
        .def("set_dropout_step", &PyEngine::set_dropout_step, py::arg("step"))
        .def("set_ema_alpha", &PyEngine::set_ema_alpha, py::arg("alpha"))
        .def("synchronize", &PyEngine::synchronize)
        .def("wait", &PyEngine::wait)
        .def("comm_status", &PyEngine::comm_status)
        .def("comm_timing", &PyEngine::comm_timing)
        .def("comm_timing_enabled", &PyEngine::comm_timing_enabled)
        .def("last_loss", &PyEngine::last_loss)
        .def("prev_loss", &PyEngine::prev_loss)
        .def("count_correct", &PyEngine::count_correct)
        .def("reset_correct", &PyEngine::reset_correct)
        .def("act", &PyEngine::act)
        .def("dz", &PyEngine::dz)
        .def("gate", &PyEngine::gate)
        .def("g", &PyEngine::g)
        .def("probs", &PyEngine::probs)
        .def("kernels_per_step", &PyEngine::kernels_per_step)
        .def("graph_nodes", &PyEngine::graph_nodes)
        .def("uses_chain", &PyEngine::uses_chain)
        .def("chain_cluster", &PyEngine::chain_cluster)
        .def("chain_ksplit", &PyEngine::chain_ksplit)
        .def("coalesced", &PyEngine::coalesced)
        .def("main_stream", &PyEngine::main_stream)
        .def("describe", &PyEngine::describe)
        .def("layer_protocols", &PyEngine::layer_protocols)
        .def("plan_text", &PyEngine::plan_text, py::arg("set") = 0)
        .def("chain_timeline", &PyEngine::chain_timeline);
}

}  // namespace ssb
