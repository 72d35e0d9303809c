// Python bindings (torch extension) for the sm_90a kernels and the native runtime.
#include <torch/extension.h>
#include <pybind11/stl.h>
#include <sstream>
#include <stdexcept>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include "kernels/kernels.h"

namespace py = pybind11;
using torch::Tensor;

namespace ssb {
void bind_runtime(py::module_& m);   // csrc/runtime/bindings_runtime.cpp
}

static void check_mat(const Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, name, " must be fp32");
    TORCH_CHECK(t.dim() == 2, name, " must be 2-D");
    TORCH_CHECK(t.size(0) > 0 && t.size(1) > 0, name, " is empty");
    TORCH_CHECK(t.stride(1) == 1 || t.size(1) == 1, name, " must have unit inner stride");
}
static int ld_of(const Tensor& t) { return (int)t.stride(0); }
static void cuda_ok(cudaError_t e, const char* what) {
    TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e));
}
static cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// The update kernels read lr from device memory when they run.  `lr` is a Python number, written into a fresh device
// scalar on the current stream, or a one-element fp32 tensor on `like`'s device that the caller may rewrite after the
// launch has been enqueued.
static Tensor lr_scalar(const py::handle& lr, const Tensor& like, const char* what) {
    if (THPVariable_Check(lr.ptr())) {
        Tensor t = py::cast<Tensor>(lr);
        TORCH_CHECK(t.is_cuda() && t.device() == like.device() && t.scalar_type() == torch::kFloat32 && t.numel() == 1,
                    what, ": a tensor lr must be one fp32 element on the kernel's device");
        return t;
    }
    return torch::full({1}, py::cast<double>(lr), like.options().dtype(torch::kFloat32));
}

// k_splits: 0 / 1 = plain kernel, -1 = let the planner decide, k >= 2 = force k (must not leave a split empty).
// The workspace and the tile counters are torch tensors owned by the caller's scope (stream-ordered reuse).
static void enable_splitk(ssb::GemmPlan& plan, int64_t k_splits, const Tensor& like, Tensor& ws, Tensor& counters) {
    if (k_splits == 0 || k_splits == 1) return;
    int splits = (int)k_splits;
    if (k_splits < 0) {
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        splits = ssb::gemm_splitk_choice(plan, sms);
        if (splits < 2) return;
    }
    ws = torch::empty({(int64_t)ssb::gemm_splitk_workspace_floats(plan, splits)}, like.options());
    counters = torch::zeros({(int64_t)plan.grid.x * plan.grid.y}, like.options().dtype(torch::kInt32));
    const char* err = ssb::gemm_plan_enable_splitk(&plan, splits, ws.data_ptr<float>(),
                                                   reinterpret_cast<unsigned int*>(counters.data_ptr<int32_t>()));
    TORCH_CHECK(err == nullptr, "split-K: ", err ? err : "");
}

// The dropout of a stand-alone GEMM: None, or (p, seed, layer, step, row_base, dp, rank) as DropoutSpec describes them.
// `step` goes into a fresh device scalar on the current stream, which `step_dev` keeps alive until the launch is enqueued.
static ssb::DropoutSpec drop_arg(const py::object& drop, const Tensor& like, Tensor& step_dev, const char* what) {
    if (drop.is_none()) return ssb::DropoutSpec{};
    const auto d = py::cast<std::tuple<double, uint64_t, int64_t, int64_t, int64_t, int64_t, int64_t>>(drop);
    const double p = std::get<0>(d);
    const int64_t layer = std::get<2>(d), step = std::get<3>(d), row_base = std::get<4>(d), dp = std::get<5>(d),
                  rank = std::get<6>(d);
    TORCH_CHECK(p > 0.0 && p < 1.0, what, ": dropout p must lie in (0, 1)");
    TORCH_CHECK(layer >= 0 && layer < (1 << 30) && step >= 0 && step < (int64_t(1) << 32) && row_base >= 0 &&
                    row_base < (1 << 30) && dp >= 1 && dp < (1 << 30) && rank >= 0 && rank < dp,
                what, ": dropout argument out of range");
    ssb::DropoutSpec spec = ssb::dropout_spec(p, std::get<1>(d));
    step_dev = torch::full({1}, (int32_t)(uint32_t)step, like.options().dtype(torch::kInt32));
    spec.step = reinterpret_cast<const uint32_t*>(step_dev.data_ptr<int32_t>());
    spec.layer = (int)layer; spec.row_base = (int)row_base; spec.dp = (int)dp; spec.rank = (int)rank;
    return spec;
}

// y[rows, out] = act?(x @ W^T + b); prec: the products' Precision (precision.h; a bool: false TF32, true 3xTF32).  relu selects the layer's activation
// act_kind (activation.h: ReLU by default); a smooth kind can store its gate f'(z) (* keep * s under dropout) to `gate`,
// which the kernel addresses with y's row pitch.  drop: see drop_arg, applied after the activation.
// res: the residual form (GemmParams::res), gated for every act_kind (a ReLU gate is 1[z > 0] * keep * s), and
// y = skip + act(z) when `skip` ([rows, out], a row pitch of its own) is given.
static void linear_fwd(const Tensor& x, const Tensor& W, const c10::optional<Tensor>& bias, int64_t bias_stride,
                       bool relu, Tensor& y, int64_t prec, int64_t k_splits, int64_t act_kind,
                       const c10::optional<Tensor>& gate, const py::object& drop, bool res,
                       const c10::optional<Tensor>& skip) {
    check_mat(x, "x"); check_mat(W, "W"); check_mat(y, "y");
    const int rows = x.size(0), in = x.size(1), out = W.size(0);
    TORCH_CHECK(W.size(1) == in && y.size(0) == rows && y.size(1) == out, "linear_fwd: shape mismatch");
    TORCH_CHECK(ssb::act_valid((int)act_kind), "linear_fwd: act_kind must be 0 (ReLU), 1 (GELU), 2 (SiLU) or 3 (tanh)");
    TORCH_CHECK(relu || (act_kind == ssb::ACT_RELU && !gate.has_value() && drop.is_none()),
                "linear_fwd: an activation kind, a gate or dropout needs relu (an activated layer)");
    if (gate.has_value()) {
        check_mat(*gate, "gate");
        TORCH_CHECK(res || ssb::act_smooth((int)act_kind), "linear_fwd: only a smooth activation or a residual layer stores a gate");
        TORCH_CHECK(gate->size(0) == rows && gate->size(1) == out && gate->device() == y.device(), "linear_fwd: gate shape");
        TORCH_CHECK(ld_of(*gate) == ld_of(y), "linear_fwd: the gate must have y's row pitch (the kernel writes it with y's)");
    }
    if (skip.has_value()) {
        TORCH_CHECK(res, "linear_fwd: a skip needs residual");
        check_mat(*skip, "skip");
        TORCH_CHECK(skip->size(0) == rows && skip->size(1) == out && skip->device() == y.device(), "linear_fwd: skip shape");
    }
    c10::cuda::CUDAGuard guard(x.device());
    ssb::GemmPlan plan;
    const char* err = ssb::gemm_plan_fwd(&plan, W.data_ptr<float>(), ld_of(W), x.data_ptr<float>(), ld_of(x),
                                         y.data_ptr<float>(), ld_of(y), rows, in, out,
                                         bias.has_value() ? bias->data_ptr<float>() : nullptr, (int)bias_stride, relu, (int)prec);
    TORCH_CHECK(err == nullptr, "linear_fwd: ", err ? err : "");
    Tensor step_dev;
    plan.p.act_kind = (int)act_kind;
    plan.p.gate = gate.has_value() ? gate->data_ptr<float>() : nullptr;
    plan.p.drop = drop_arg(drop, x, step_dev, "linear_fwd");
    if (res) {
        plan.p.res = 1;
        plan.p.skip = skip.has_value() ? skip->data_ptr<float>() : nullptr;
        plan.p.ldskip = skip.has_value() ? ld_of(*skip) : 0;
    }
    Tensor ws, counters;
    enable_splitk(plan, k_splits, x, ws, counters);
    cuda_ok(ssb::gemm_launch(plan, cur_stream()), "linear_fwd launch");
}

// dx[rows, in] = (dz @ W) * (mask > 0), or * s where the mask passes under dropout (only its p is read), or * mask for a
// smooth act_kind (the mask is then the previous layer's gate, which holds the dropout scale itself)
// res: the residual form (GemmParams::res): x = dz @ W + skip (skip: the layer's output gradient, [rows, in]), stored to
// gpre before the mask, then dx = x * mask (the mask is the previous layer's gate for every act_kind).  skip, gpre and
// the mask each have a row pitch of their own.
static void linear_dgrad(const Tensor& dz, const Tensor& W, const c10::optional<Tensor>& mask, Tensor& dx,
                         int64_t prec, int64_t k_splits, int64_t act_kind, const py::object& drop, bool res,
                         const c10::optional<Tensor>& skip, const c10::optional<Tensor>& gpre) {
    check_mat(dz, "dz"); check_mat(W, "W"); check_mat(dx, "dx");
    const int rows = dz.size(0), out = dz.size(1), in = W.size(1);
    TORCH_CHECK(W.size(0) == out && dx.size(0) == rows && dx.size(1) == in, "linear_dgrad: shape mismatch");
    if (mask.has_value()) { check_mat(*mask, "mask"); TORCH_CHECK(mask->size(0) == rows && mask->size(1) == in, "mask shape"); }
    TORCH_CHECK(ssb::act_valid((int)act_kind), "linear_dgrad: act_kind must be 0 (ReLU), 1 (GELU), 2 (SiLU) or 3 (tanh)");
    TORCH_CHECK(mask.has_value() || (act_kind == ssb::ACT_RELU && drop.is_none()),
                "linear_dgrad: an activation kind or dropout needs a mask");
    TORCH_CHECK(drop.is_none() || !ssb::act_smooth((int)act_kind),
                "linear_dgrad: a gate holds its dropout scale already; pass no dropout with a smooth act_kind");
    TORCH_CHECK(drop.is_none() || !res, "linear_dgrad: a residual gate holds its dropout scale already; pass no dropout");
    TORCH_CHECK(res || (!skip.has_value() && !gpre.has_value()), "linear_dgrad: skip and gpre need residual");
    if (skip.has_value()) {
        check_mat(*skip, "skip");
        TORCH_CHECK(skip->size(0) == rows && skip->size(1) == in && skip->device() == dx.device(), "linear_dgrad: skip shape");
    }
    if (gpre.has_value()) {
        check_mat(*gpre, "gpre");
        TORCH_CHECK(gpre->size(0) == rows && gpre->size(1) == in && gpre->device() == dx.device(), "linear_dgrad: gpre shape");
    }
    if (mask.has_value()) TORCH_CHECK(mask->device() == dx.device(), "linear_dgrad: mask device");
    c10::cuda::CUDAGuard guard(dz.device());
    ssb::GemmPlan plan;
    const char* err = ssb::gemm_plan_dgrad(&plan, W.data_ptr<float>(), ld_of(W), dz.data_ptr<float>(), ld_of(dz),
                                           dx.data_ptr<float>(), ld_of(dx), rows, in, out,
                                           mask.has_value() ? mask->data_ptr<float>() : nullptr,
                                           mask.has_value() ? ld_of(*mask) : 0, (int)prec);
    TORCH_CHECK(err == nullptr, "linear_dgrad: ", err ? err : "");
    Tensor step_dev;
    plan.p.act_kind = (int)act_kind;
    plan.p.drop = drop_arg(drop, dz, step_dev, "linear_dgrad");
    if (res) {
        plan.p.res = 1;
        plan.p.skip = skip.has_value() ? skip->data_ptr<float>() : nullptr;
        plan.p.ldskip = skip.has_value() ? ld_of(*skip) : 0;
        plan.p.gpre = gpre.has_value() ? gpre->data_ptr<float>() : nullptr;
        plan.p.ldgpre = gpre.has_value() ? ld_of(*gpre) : 0;
    }
    Tensor ws, counters;
    enable_splitk(plan, k_splits, dz, ws, counters);
    cuda_ok(ssb::gemm_launch(plan, cur_stream()), "linear_dgrad launch");
}

// G[out, in] (+)= dz^T @ x ; db[out] (+)= colsum(dz) ; optionally W -= lr * (G + ...)
// With momentum / weight decay the fused update follows the stateful rule; V is the momentum buffer with W's layout
// (same row pitch; its column `in` belongs to the bias).
static void linear_wgrad(const Tensor& dz, const Tensor& x, Tensor& G, bool accumulate, const c10::optional<Tensor>& db,
                         int64_t db_stride, const c10::optional<Tensor>& W, const py::object& lr, bool fuse_sgd,
                         int64_t prec, const c10::optional<Tensor>& V, double momentum, double weight_decay, bool nesterov,
                         const c10::optional<Tensor>& E, const py::object& ema_alpha) {
    check_mat(dz, "dz"); check_mat(x, "x"); check_mat(G, "G");
    const int rows = dz.size(0), out = dz.size(1), in = x.size(1);
    TORCH_CHECK(x.size(0) == rows && G.size(0) == out && G.size(1) == in, "linear_wgrad: shape mismatch");
    ssb::SgdState opt;
    opt.momentum = (float)momentum; opt.weight_decay = (float)weight_decay; opt.nesterov = nesterov ? 1 : 0;
    if (V.has_value()) {
        check_mat(*V, "V");
        TORCH_CHECK(W.has_value() && V->size(0) == out && V->size(1) == in && ld_of(*V) == ld_of(*W),
                    "linear_wgrad: V must have W's shape and row pitch");
        opt.V = V->data_ptr<float>();
    }
    TORCH_CHECK(E.has_value() == !ema_alpha.is_none(), "linear_wgrad: ema and ema_alpha go together");
    Tensor alpha_dev;
    if (E.has_value()) {
        check_mat(*E, "ema");
        TORCH_CHECK(W.has_value() && E->size(0) == out && E->size(1) == in && ld_of(*E) == ld_of(*W),
                    "linear_wgrad: ema must have W's shape and row pitch");
        alpha_dev = lr_scalar(ema_alpha, dz, "linear_wgrad (ema_alpha)");
        opt.E = E->data_ptr<float>();
        opt.ema_alpha = alpha_dev.data_ptr<float>();
    }
    c10::cuda::CUDAGuard guard(dz.device());
    const Tensor lr_dev = fuse_sgd ? lr_scalar(lr, dz, "linear_wgrad") : Tensor();
    ssb::GemmPlan plan;
    const char* err = ssb::gemm_plan_wgrad(&plan, dz.data_ptr<float>(), ld_of(dz), x.data_ptr<float>(), ld_of(x),
                                           G.data_ptr<float>(), ld_of(G), rows, in, out, accumulate,
                                           db.has_value() ? db->data_ptr<float>() : nullptr, (int)db_stride,
                                           W.has_value() ? W->data_ptr<float>() : nullptr,
                                           W.has_value() ? ld_of(*W) : 0, fuse_sgd ? lr_dev.data_ptr<float>() : nullptr,
                                           fuse_sgd, (int)prec, opt);
    TORCH_CHECK(err == nullptr, "linear_wgrad: ", err ? err : "");
    cuda_ok(ssb::gemm_launch(plan, cur_stream()), "linear_wgrad launch");
}

static void loss_head(const Tensor& logits, const c10::optional<Tensor>& target, const c10::optional<Tensor>& probs,
                      const c10::optional<Tensor>& dlogits, const c10::optional<Tensor>& loss_out, double inv_batch,
                      int loss) {
    check_mat(logits, "logits");
    TORCH_CHECK(loss == ssb::LOSS_MSE || loss == ssb::LOSS_CROSS_ENTROPY, "loss_head: loss must be 0 (MSE) or 1 (cross-entropy)");
    TORCH_CHECK(!target.has_value() || dlogits.has_value(), "loss_head: training (a target) needs dlogits");
    c10::cuda::CUDAGuard guard(logits.device());
    const int rows = logits.size(0), cols = logits.size(1);
    cuda_ok(ssb::launch_loss_head(logits.data_ptr<float>(), ld_of(logits),
                                  target.has_value() ? target->data_ptr<float>() : nullptr, target.has_value() ? ld_of(*target) : 0,
                                  probs.has_value() ? probs->data_ptr<float>() : nullptr, probs.has_value() ? ld_of(*probs) : 0,
                                  dlogits.has_value() ? dlogits->data_ptr<float>() : nullptr, dlogits.has_value() ? ld_of(*dlogits) : 0,
                                  loss_out.has_value() ? loss_out->data_ptr<float>() : nullptr, rows, cols, (float)inv_batch,
                                  cur_stream(), 0, loss), "loss_head");
}

static void softmax_grad(const Tensor& logits, const Tensor& upstream, Tensor& dlogits) {
    check_mat(logits, "logits"); check_mat(upstream, "upstream"); check_mat(dlogits, "dlogits");
    c10::cuda::CUDAGuard guard(logits.device());
    cuda_ok(ssb::launch_softmax_grad(logits.data_ptr<float>(), ld_of(logits), upstream.data_ptr<float>(), ld_of(upstream),
                                     dlogits.data_ptr<float>(), ld_of(dlogits), logits.size(0), logits.size(1), cur_stream()),
            "softmax_grad");
}

static void relu_mask_(Tensor& g, const Tensor& y) {
    check_mat(g, "g"); check_mat(y, "y");
    c10::cuda::CUDAGuard guard(g.device());
    cuda_ok(ssb::launch_relu_mask(g.data_ptr<float>(), ld_of(g), y.data_ptr<float>(), ld_of(y), g.size(0), g.size(1), cur_stream()), "relu_mask");
}
static void relu_fwd(const Tensor& x, Tensor& y) {
    TORCH_CHECK(x.is_contiguous() && y.is_contiguous() && x.numel() == y.numel());
    c10::cuda::CUDAGuard guard(x.device());
    cuda_ok(ssb::launch_relu_fwd(x.data_ptr<float>(), y.data_ptr<float>(), x.numel(), cur_stream()), "relu_fwd");
}
// smooth activation (ptx.cuh: act_fwd) of a dense tensor: y = f(z), gamma = f'(z)
static void act_fwd(int64_t kind, const Tensor& z, Tensor& y, Tensor& gamma) {
    TORCH_CHECK(ssb::act_smooth((int)kind), "act_fwd: kind must be GELU (1), SiLU (2) or tanh (3), got ", kind);
    for (const Tensor* t : std::initializer_list<const Tensor*>{&z, &y, &gamma})
        TORCH_CHECK(t->is_cuda() && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && t->numel() == z.numel(),
                    "act_fwd: z, y and gamma must be dense fp32 CUDA tensors of one size");
    c10::cuda::CUDAGuard guard(z.device());
    cuda_ok(ssb::launch_act_fwd((int)kind, z.data_ptr<float>(), y.data_ptr<float>(), gamma.data_ptr<float>(), z.numel(),
                                cur_stream()), "act_fwd");
}
// g *= gamma (the backward of a smooth activation)
static void gate_mul_(Tensor& g, const Tensor& gamma) {
    check_mat(g, "g"); check_mat(gamma, "gamma");
    TORCH_CHECK(g.size(0) == gamma.size(0) && g.size(1) == gamma.size(1), "gate_mul_: g and gamma differ in shape");
    c10::cuda::CUDAGuard guard(g.device());
    cuda_ok(ssb::launch_gate_mul(g.data_ptr<float>(), ld_of(g), gamma.data_ptr<float>(), ld_of(gamma), g.size(0), g.size(1),
                                 cur_stream()), "gate_mul");
}
static void axpby(const Tensor& x, const Tensor& t, Tensor& y, double a, double b) {
    TORCH_CHECK(x.is_contiguous() && t.is_contiguous() && y.is_contiguous() && x.numel() == y.numel() && t.numel() == y.numel());
    c10::cuda::CUDAGuard guard(x.device());
    cuda_ok(ssb::launch_axpby(x.data_ptr<float>(), t.data_ptr<float>(), y.data_ptr<float>(), (float)a, (float)b, x.numel(), cur_stream()), "axpby");
}
static void sgd_(Tensor& w, const Tensor& g, const py::object& lr) {
    TORCH_CHECK(w.is_contiguous() && g.is_contiguous() && w.numel() == g.numel());
    c10::cuda::CUDAGuard guard(w.device());
    const Tensor lr_dev = lr_scalar(lr, w, "sgd_");
    cuda_ok(ssb::launch_sgd(w.data_ptr<float>(), g.data_ptr<float>(), lr_dev.data_ptr<float>(), w.numel(), cur_stream()), "sgd");
}
static void sgd_momentum_(Tensor& w, const Tensor& g, const c10::optional<Tensor>& v, const py::object& lr, double momentum,
                          double weight_decay, bool nesterov, const c10::optional<Tensor>& e, const py::object& ema_alpha) {
    TORCH_CHECK(w.is_contiguous() && g.is_contiguous() && w.numel() == g.numel());
    TORCH_CHECK(w.scalar_type() == torch::kFloat32 && g.scalar_type() == torch::kFloat32);
    ssb::SgdState opt;
    opt.momentum = (float)momentum; opt.weight_decay = (float)weight_decay; opt.nesterov = nesterov ? 1 : 0;
    if (v.has_value()) {
        TORCH_CHECK(v->is_contiguous() && v->numel() == w.numel() && v->scalar_type() == torch::kFloat32 && v->is_cuda());
        opt.V = v->data_ptr<float>();
    }
    TORCH_CHECK(e.has_value() == !ema_alpha.is_none(), "sgd_momentum_: ema and ema_alpha go together");
    Tensor alpha_dev;
    if (e.has_value()) {
        TORCH_CHECK(e->is_contiguous() && e->numel() == w.numel() && e->scalar_type() == torch::kFloat32 && e->is_cuda());
        alpha_dev = lr_scalar(ema_alpha, w, "sgd_momentum_ (ema_alpha)");
        opt.E = e->data_ptr<float>();
        opt.ema_alpha = alpha_dev.data_ptr<float>();
    }
    const char* err = ssb::sgd_state_check(opt);
    TORCH_CHECK(err == nullptr, "sgd_momentum_: ", err ? err : "");
    c10::cuda::CUDAGuard guard(w.device());
    const Tensor lr_dev = lr_scalar(lr, w, "sgd_momentum_");
    cuda_ok(ssb::launch_sgd_momentum(w.data_ptr<float>(), g.data_ptr<float>(), lr_dev.data_ptr<float>(), opt, w.numel(), cur_stream()),
            "sgd_momentum");
}
static void argmax_correct(const Tensor& pred, const Tensor& target, Tensor& correct) {
    check_mat(pred, "pred"); check_mat(target, "target");
    TORCH_CHECK(correct.scalar_type() == torch::kInt32 && correct.is_cuda());
    c10::cuda::CUDAGuard guard(pred.device());
    cuda_ok(ssb::launch_argmax_correct(pred.data_ptr<float>(), ld_of(pred), target.data_ptr<float>(), ld_of(target),
                                       pred.size(0), pred.size(1), correct.data_ptr<int>(), cur_stream()), "argmax_correct");
}

// the device permutation of the training set (ptx.cuh: shuffle_index) at int64 positions in [0, n)
static Tensor shuffle_index(int64_t n, uint64_t seed, int64_t epoch, const Tensor& positions) {
    TORCH_CHECK(n >= 1 && n < (int64_t(1) << 32), "shuffle_index: n must lie in [1, 2**32)");
    TORCH_CHECK(positions.is_cuda() && positions.scalar_type() == torch::kInt64, "shuffle_index: positions must be int64 CUDA");
    TORCH_CHECK(epoch >= 0, "shuffle_index: the epoch must be >= 0");
    const Tensor q = positions.contiguous();
    if (q.numel() > 0)
        TORCH_CHECK(q.min().item<int64_t>() >= 0 && q.max().item<int64_t>() < n, "shuffle_index: positions must lie in [0, n)");
    c10::cuda::CUDAGuard guard(q.device());
    Tensor out = torch::empty_like(q);
    cuda_ok(ssb::launch_shuffle_index((uint32_t)n, seed, (uint32_t)(epoch & 0xffffffffLL), q.data_ptr<int64_t>(),
                                      out.data_ptr<int64_t>(), (long)q.numel(), cur_stream()), "shuffle_index");
    return out;
}
// the staging gather on its own (launch_gather_rows): rows of global batch `batch` of this rank into x_dst / y_dst, whose
// row pitch is their stride(0); x_src / y_src are the whole dense dataset
static void gather_rows(const c10::optional<Tensor>& x_src, const c10::optional<Tensor>& y_src, uint64_t seed, int64_t epoch,
                        int64_t gbs, int64_t dp, int64_t rank, int64_t batch, const c10::optional<Tensor>& x_dst,
                        const c10::optional<Tensor>& y_dst) {
    TORCH_CHECK(x_src.has_value() == x_dst.has_value() && y_src.has_value() == y_dst.has_value(),
                "gather_rows: every source needs a destination and the reverse");
    TORCH_CHECK(x_src.has_value() || y_src.has_value(), "gather_rows: nothing to gather");
    const Tensor& any_src = x_src.has_value() ? *x_src : *y_src;
    const Tensor& any_dst = x_dst.has_value() ? *x_dst : *y_dst;
    for (const auto* s : {&x_src, &y_src}) {
        if (!s->has_value()) continue;
        const Tensor& t = **s;
        TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.dim() == 2 && t.is_contiguous(),
                    "gather_rows: sources must be dense 2-D fp32 CUDA tensors");
        TORCH_CHECK(t.size(0) == any_src.size(0) && t.device() == any_src.device(), "gather_rows: sources disagree");
    }
    for (const auto* d : {&x_dst, &y_dst}) {
        if (!d->has_value()) continue;
        check_mat(**d, "gather_rows destination");
        TORCH_CHECK((*d)->size(0) == any_dst.size(0) && (*d)->device() == any_src.device(), "gather_rows: destinations disagree");
    }
    if (x_src.has_value()) TORCH_CHECK(x_dst->size(1) == x_src->size(1), "gather_rows: x widths differ");
    if (y_src.has_value()) TORCH_CHECK(y_dst->size(1) == y_src->size(1), "gather_rows: y widths differ");
    TORCH_CHECK(any_src.size(0) < (int64_t(1) << 32) && epoch >= 0 && gbs < (1 << 30) && dp < (1 << 30) && batch < (1 << 30),
                "gather_rows: argument out of range");
    const ssb::ShuffleSpec spec{(uint32_t)any_src.size(0), seed, (uint32_t)(epoch & 0xffffffffLL), (int)gbs, (int)dp, (int)rank};
    const int rows = (int)any_dst.size(0);
    const char* err = ssb::shuffle_spec_check(spec, (int)batch, rows);
    TORCH_CHECK(err == nullptr, "gather_rows: ", err ? err : "");
    c10::cuda::CUDAGuard guard(any_src.device());
    cuda_ok(ssb::launch_gather_rows(x_src ? x_src->data_ptr<float>() : nullptr, y_src ? y_src->data_ptr<float>() : nullptr,
                                    spec, (int)batch, x_dst ? x_dst->data_ptr<float>() : nullptr, x_dst ? ld_of(*x_dst) : 0,
                                    y_dst ? y_dst->data_ptr<float>() : nullptr, y_dst ? ld_of(*y_dst) : 0, rows,
                                    x_src ? (int)x_src->size(1) : 0, y_src ? (int)y_src->size(1) : 0, cur_stream()),
            "gather_rows");
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "shallowspeed_b200 native module: sm_90a kernels + C++ pipeline runtime";
    m.def("linear_fwd", &linear_fwd, py::arg("x"), py::arg("W"), py::arg("bias"), py::arg("bias_stride"), py::arg("relu"),
          py::arg("y"), py::arg("prec") = (int)ssb::PREC_TF32, py::arg("k_splits") = 0, py::arg("act_kind") = (int)ssb::ACT_RELU,
          py::arg("gate") = py::none(), py::arg("drop") = py::none(), py::arg("res") = false, py::arg("skip") = py::none());
    m.def("linear_dgrad", &linear_dgrad, py::arg("dz"), py::arg("W"), py::arg("mask"), py::arg("dx"),
          py::arg("prec") = (int)ssb::PREC_TF32, py::arg("k_splits") = 0, py::arg("act_kind") = (int)ssb::ACT_RELU,
          py::arg("drop") = py::none(), py::arg("res") = false, py::arg("skip") = py::none(), py::arg("gpre") = py::none());
    m.def("linear_wgrad", &linear_wgrad, py::arg("dz"), py::arg("x"), py::arg("G"), py::arg("accumulate"), py::arg("db"),
          py::arg("db_stride"), py::arg("W"), py::arg("lr"), py::arg("fuse_sgd"), py::arg("prec") = (int)ssb::PREC_TF32,
          py::arg("V") = py::none(), py::arg("momentum") = 0.0, py::arg("weight_decay") = 0.0, py::arg("nesterov") = false,
          py::arg("ema") = py::none(), py::arg("ema_alpha") = py::none());
    m.def("loss_head", &loss_head, py::arg("logits"), py::arg("target"), py::arg("probs"), py::arg("dlogits"),
          py::arg("loss_out"), py::arg("inv_batch"), py::arg("loss") = (int)ssb::LOSS_MSE);
    m.def("softmax_grad", &softmax_grad);
    m.def("relu_mask_", &relu_mask_);
    m.def("relu_fwd", &relu_fwd);
    m.def("act_fwd", &act_fwd, py::arg("kind"), py::arg("z"), py::arg("y"), py::arg("gamma"));
    m.def("gate_mul_", &gate_mul_, py::arg("g"), py::arg("gamma"));
    m.def("axpby", &axpby);
    m.def("sgd_", &sgd_);
    m.def("sgd_momentum_", &sgd_momentum_, py::arg("w"), py::arg("g"), py::arg("v"), py::arg("lr"), py::arg("momentum"),
          py::arg("weight_decay"), py::arg("nesterov"), py::arg("ema") = py::none(), py::arg("ema_alpha") = py::none());
    m.def("argmax_correct", &argmax_correct);
    m.def("shuffle_index", &shuffle_index, py::arg("n"), py::arg("seed"), py::arg("epoch"), py::arg("positions"));
    m.def("gather_rows", &gather_rows, py::arg("x_src"), py::arg("y_src"), py::arg("seed"), py::arg("epoch"), py::arg("gbs"),
          py::arg("dp"), py::arg("rank"), py::arg("batch"), py::arg("x_dst"), py::arg("y_dst"));
    m.def("gemm_kernel_count", &ssb::gemm_kernel_count);
    m.def("chain_budget", [](int mb_rows, int prec) {
        int kps = 0, stages = 0, smem = 0;
        const bool ok = ssb::chain_budget(mb_rows, prec, &kps, &stages, &smem);
        return std::make_tuple(ok, kps, stages, smem);
    });
    // tiles of one grouped weight gradient, no GPU needed: ([(m0, n0, rows, cols, owns_bias)], stages, smem bytes per CTA)
    m.def("wgrad_group_tiles", [](int out, int in, int rows) {
        std::vector<ssb::GemmGroupTile> tiles;
        int stages = 0, smem = 0;
        if (const char* e = ssb::gemm_group_tiles(out, in, rows, &tiles, &stages, &smem)) throw std::invalid_argument(e);
        std::vector<std::tuple<int, int, int, int, bool>> list;
        for (const auto& t : tiles) list.emplace_back(t.m0, t.n0, t.rows, t.cols, t.owns_bias);
        return std::make_tuple(list, stages, smem);
    });
    m.def("chain_cluster_budget", [](int mb_rows, int cluster, int prec) {
        int kps = 0, stages = 0, smem = 0;
        const bool ok = ssb::chain_cluster_budget(mb_rows, cluster, prec, &kps, &stages, &smem);
        return std::make_tuple(ok, kps, stages, smem);
    });
    // k-split layer 1, no GPU needed: the k-blocks of a GEMM of nkb k-blocks that part 0 (owner) / 1 (helper) multiplies
    m.def("chain_ksplit_kblocks", [](int nkb, int part) {
        std::vector<int> kb((size_t)std::max(nkb, 0));
        kb.resize((size_t)ssb::chain_ksplit_kblocks(nkb, part, kb.data()));
        return kb;
    });
    m.def("chain_cluster_size", [](const std::vector<std::pair<int, int>>& in_out, bool do_fwd, bool do_loss, bool do_bwd,
                                   bool first_stage, bool gated, bool folded) {
        std::vector<ssb::ChainLayer> ls(in_out.size());
        for (size_t i = 0; i < in_out.size(); ++i) { ls[i] = ssb::ChainLayer{}; ls[i].in = in_out[i].first; ls[i].out = in_out[i].second; }
        return ssb::chain_cluster_size(ls.data(), (int)ls.size(), do_fwd, do_loss, do_bwd, first_stage, gated, folded);
    });
    m.def("chain_eligible", [](const std::vector<std::pair<int, int>>& in_out, int mb_rows, int out_dim, bool has_loss, int prec) {
        std::vector<ssb::ChainLayer> ls(in_out.size());
        for (size_t i = 0; i < in_out.size(); ++i) { ls[i] = ssb::ChainLayer{}; ls[i].in = in_out[i].first; ls[i].out = in_out[i].second; }
        return ssb::chain_eligible(ls.data(), (int)ls.size(), mb_rows, out_dim, has_loss, prec);
    });
    m.def("dp_layer_geometry", [](int in, int out, int dp, bool one_shot) {
        int block_n = 0, tm = 0, tn = 0;
        int64_t slots = 0, slot_floats = 0;
        ssb::dp_layer_geometry(in, out, dp, &block_n, &tm, &tn, &slots, &slot_floats, one_shot ? 1 : 0);
        return std::make_tuple(block_n, tm, tn, slots, slot_floats);
    });
    // host-only planning logic, callable without a GPU (tests/test_planning.py):
    // (k_splits chosen, k-blocks per split, error string of enable() with dummy buffers or "")
    m.def("splitk_plan", [](int m_total, int n_rows, int k_total, int num_sms, int force) {
        ssb::GemmPlan plan{};
        plan.mode = ssb::GEMM_FWD;
        plan.p.m_total = m_total; plan.p.n_total = n_rows; plan.p.k_total = k_total;
        plan.p.block_n = n_rows >= 64 ? 64 : (n_rows + 15) / 16 * 16;   // as gemm_plan_fwd
        plan.grid = dim3((m_total + 127) / 128, (n_rows + plan.p.block_n - 1) / plan.p.block_n, 1);
        int splits = force > 0 ? force : ssb::gemm_splitk_choice(plan, num_sms);
        const int num_kb = (k_total + 31) / 32;
        std::string err;
        if (splits > 1) {
            float dummy_ws;
            unsigned int dummy_ctr;
            const char* e = ssb::gemm_plan_enable_splitk(&plan, splits, &dummy_ws, &dummy_ctr);
            if (e) err = e;
        }
        const int per = splits > 0 ? (num_kb + splits - 1) / splits : num_kb;
        return std::make_tuple(splits, per, (int)plan.grid.z, plan.p.stages, plan.smem_bytes, err);
    });
    // LL data-parallel kernel: host-side geometry (tiles per layer, lines per landing zone), callable without a GPU
    // owner rank of every parameter element of one layer ([out, in + 1], bias last; -1 = every replica), no GPU needed
    m.def("dp_owner_map", [](int proto, int in, int out, int ld, int64_t offset, int dp) {
        torch::Tensor t = torch::empty({out, in + 1}, torch::kInt8);
        auto a = t.accessor<int8_t, 2>();
        for (int mm = 0; mm < out; ++mm)
            for (int nn = 0; nn <= in; ++nn) a[mm][nn] = (int8_t)ssb::dp_element_owner(proto, in, out, ld, offset, dp, mm, nn);
        return t;
    });
    m.attr("DP_PROTO_ALL") = (int)ssb::DP_PROTO_ALL;
    m.attr("DP_PROTO_LL") = (int)ssb::DP_PROTO_LL;
    m.attr("DP_PROTO_TWO_SHOT") = (int)ssb::DP_PROTO_TWO_SHOT;
    m.attr("DP_PROTO_NVLS") = (int)ssb::DP_PROTO_NVLS;
    m.def("dp_ll_tiles", [](int in, int out) { return ssb::dp_ll_tiles(in, out); });
    m.def("dp_ll_zone_lines", [](int dp, int n_tiles) { return (int64_t)ssb::dp_ll_zone_lines(dp, n_tiles); });
    // Exercises the C++ runtime features that break when libstdc++ is linked statically next to torch's dynamic
    // copy (the round-1 GPU-suite segfault): locale-dependent integer / float formatting and an exception that
    // crosses a function boundary.  Callable without a GPU (tests/test_native_linkage.py).
    m.def("selftest_format", [](int v) {
        std::ostringstream os;
        os << "v=" << v << " f=" << 1.5 << " h=" << std::hex << 255;
        try {
            throw std::runtime_error(os.str());
        } catch (const std::exception& e) {
            return std::string(e.what());
        }
    });
    ssb::bind_runtime(m);
}
