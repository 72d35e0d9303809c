#include "runtime/dp_context.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

namespace ssb {

#define CUDA_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t _e = (expr);                                                                           \
        if (_e != cudaSuccess)                                                                             \
            throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr); \
    } while (0)

static int64_t round_up64(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

DpContext::DpContext(int dp, int rank, int64_t arena_numel, const std::vector<std::tuple<int, int, int64_t, int>>& layers,
                     float /*lr: unused, see dp_context.h*/)
    : dp_(dp), rank_(rank), arena_numel_(arena_numel) {
    if (dp < 1 || dp > kMaxDp) throw std::runtime_error("DpContext: dp must be in [1, 8]");
    int64_t stage_off = 0;
    int slot_base = 0, tile_base = 0;
    for (auto& t : layers) {
        DpLayerGeom g{};
        g.in = std::get<0>(t); g.out = std::get<1>(t); g.w_offset = std::get<2>(t); g.ld = std::get<3>(t);
        // latency-bound layers (<= 2 MB of gradient) use the one-shot protocol, big ones two-shot
        g.one_shot = ((int64_t)g.in * g.out * 4 <= (2 << 20)) && !getenv("SSB_DP_TWO_SHOT");
        if (getenv("SSB_DP_ONE_SHOT")) g.one_shot = 1;
        dp_layer_geometry(g.in, g.out, dp, &g.block_n, &g.n_tiles_m, &g.n_tiles_n, &g.slots, &g.slot_floats, g.one_shot);
        total_ctas_ += g.n_tiles_m * g.n_tiles_n;
        g.stage_offset = stage_off;
        g.slot_flag_base = slot_base;
        g.tile_flag_base = tile_base;
        stage_off += g.slots * g.slot_floats;
        slot_base += (int)g.slots;
        tile_base += g.n_tiles_m * g.n_tiles_n;
        geom_.push_back(g);
    }
    stage_parity_stride_ = round_up64(std::max<int64_t>(stage_off, 64), 64);
    stage_src_stride_ = 2 * stage_parity_stride_;        // x2: one-shot slots are double-buffered by epoch parity
    slots_per_src_ = std::max(slot_base, 1);
    tiles_total_ = std::max(tile_base, 1);
    auto alloc = [](void** p, size_t bytes) {
        CUDA_CHECK(cudaMalloc(p, bytes));
        CUDA_CHECK(cudaMemset(*p, 0, bytes));
    };
    alloc((void**)&W_, (size_t)arena_numel_ * 4);
    alloc((void**)&stage_, (size_t)dp_ * stage_src_stride_ * 4);
    alloc((void**)&arrive_, (size_t)dp_ * slots_per_src_ * 4);
    alloc((void**)&done_, (size_t)tiles_total_ * 4);
    alloc((void**)&epoch_, 64);
    // LL landing zones: only for stages whose [128 x 32] tiles all fit on the chip next to the chain kernel
    {
        int tiles = 0;
        for (const auto& g : geom_) tiles += dp_ll_tiles(g.in, g.out);
        const bool ok = tiles > 0 && tiles <= 128 && dp_ >= 2 && (128 % dp_) == 0 && !(getenv("SSB_DP_LL") && atoi(getenv("SSB_DP_LL")) == 0);
        if (ok) {
            ll_tiles_ = tiles;
            const size_t bytes = dp_ll_zone_lines(dp_, tiles) * sizeof(uint4);
            alloc((void**)&llA_, bytes);
            alloc((void**)&llC_, bytes);
            llA_peers_[rank_] = llA_; llC_peers_[rank_] = llC_;
        }
    }
    for (int r = 0; r < kMaxDp; ++r) { peers_.W[r] = nullptr; peers_.stage[r] = nullptr; peers_.arrive[r] = nullptr; peers_.done[r] = nullptr; }
    peers_.W[rank_] = W_; peers_.stage[rank_] = stage_; peers_.arrive[rank_] = arrive_; peers_.done[rank_] = done_;
    CUDA_CHECK(cudaDeviceSynchronize());
}

DpContext::~DpContext() {
    cudaDeviceSynchronize();
    for (void* p : opened_) cudaIpcCloseMemHandle(p);
    cudaFree(W_); cudaFree(stage_); cudaFree(arrive_); cudaFree(done_); cudaFree(epoch_);
    if (llA_) cudaFree(llA_);
    if (llC_) cudaFree(llC_);
}

std::string DpContext::export_handles() const {
    cudaIpcMemHandle_t h[6];
    memset(h, 0, sizeof(h));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[0], W_));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[1], stage_));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[2], arrive_));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[3], done_));
    if (ll_tiles_ > 0) {
        CUDA_CHECK(cudaIpcGetMemHandle(&h[4], llA_));
        CUDA_CHECK(cudaIpcGetMemHandle(&h[5], llC_));
    }
    return std::string(reinterpret_cast<const char*>(h), sizeof(h));
}

void DpContext::open_peers(const std::vector<std::string>& handles) {
    if ((int)handles.size() != dp_) throw std::runtime_error("DpContext::open_peers: need one handle blob per DP rank");
    for (int r = 0; r < dp_; ++r) {
        if (r == rank_) continue;
        if (handles[r].size() != 6 * sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("DpContext: bad handle blob");
        cudaIpcMemHandle_t h[6];
        memcpy(h, handles[r].data(), sizeof(h));
        void* ptr[6] = {};
        const int n = ll_tiles_ > 0 ? 6 : 4;
        for (int i = 0; i < n; ++i) {
            CUDA_CHECK(cudaIpcOpenMemHandle(&ptr[i], h[i], cudaIpcMemLazyEnablePeerAccess));
            opened_.push_back(ptr[i]);
        }
        peers_.W[r] = (float*)ptr[0]; peers_.stage[r] = (float*)ptr[1];
        peers_.arrive[r] = (uint32_t*)ptr[2]; peers_.done[r] = (uint32_t*)ptr[3];
        llA_peers_[r] = (uint4*)ptr[4]; llC_peers_[r] = (uint4*)ptr[5];
    }
}

void DpContext::open_local_peers(const std::vector<const DpContext*>& ctxs) {
    if ((int)ctxs.size() != dp_) throw std::runtime_error("DpContext::open_local_peers: need one context per DP rank");
    for (int r = 0; r < dp_; ++r) {
        if (r == rank_) continue;
        const DpContext* c = ctxs[r];
        if (c == nullptr || c->dp_ != dp_ || c->rank_ != r || c->arena_numel_ != arena_numel_ ||
            c->stage_src_stride_ != stage_src_stride_ || c->slots_per_src_ != slots_per_src_ ||
            c->tiles_total_ != tiles_total_ || c->ll_tiles_ != ll_tiles_)
            throw std::runtime_error("DpContext::open_local_peers: context " + std::to_string(r) +
                                     " is not rank " + std::to_string(r) + " of the same group and geometry");
        peers_.W[r] = c->W_; peers_.stage[r] = c->stage_;
        peers_.arrive[r] = c->arrive_; peers_.done[r] = c->done_;
        llA_peers_[r] = c->llA_; llC_peers_[r] = c->llC_;
    }
}

DpLLParams DpContext::ll_params() const {
    DpLLParams p{};
    p.dp = dp_; p.rank = rank_; p.lr = nullptr;
    p.epoch_ptr = epoch_; p.gate_step = nullptr;
    p.n_tiles = ll_tiles_; p.stages = 2;
    p.W = W_;
    for (int r = 0; r < kMaxDp; ++r) { p.llA[r] = llA_peers_[r]; p.llC[r] = llC_peers_[r]; }
    return p;
}

DpLayerParams DpContext::layer_params(int i) const {
    const DpLayerGeom& g = geom_.at(i);
    DpLayerParams p{};
    p.m_total = g.out; p.n_total = g.in; p.k_total = 0;
    p.block_n = g.block_n; p.stages = 2;
    p.n_tiles_m = g.n_tiles_m; p.n_tiles_n = g.n_tiles_n;
    p.dp = dp_; p.rank = rank_;
    p.w_offset = g.w_offset; p.ldw = g.ld;
    p.stage_offset = g.stage_offset; p.stage_src_stride = stage_src_stride_;
    p.tile_flag_base = g.tile_flag_base; p.slot_flag_base = g.slot_flag_base; p.slots_per_src = slots_per_src_;
    p.lr = nullptr;
    p.epoch_ptr = epoch_;
    p.G = nullptr; p.ldg = g.ld;
    p.one_shot = g.one_shot;
    p.dbg = nullptr;
    p.helpers = 1;
    p.prec = PREC_TF32;
    p.bulk_push = getenv("SSB_DP_BULK") ? atoi(getenv("SSB_DP_BULK")) : 1;   // TMA bulk copies to peer memory (verified on NVLink)
    p.stage_parity_stride = stage_parity_stride_;
    return p;
}

}  // namespace ssb
