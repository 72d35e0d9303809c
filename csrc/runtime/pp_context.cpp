#include "runtime/pp_context.h"

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace ssb {

#define CUDA_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t _e = (expr);                                                                           \
        if (_e != cudaSuccess)                                                                             \
            throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr); \
    } while (0)

PpContext::PpContext(int n_mu, int mb_rows, int ld_in, int ld_out, bool is_first, bool is_last)
    : n_mu_(n_mu), mb_(mb_rows), ld_in_(ld_in), ld_out_(ld_out), first_(is_first), last_(is_last) {
    if (n_mu < 1 || n_mu > kMaxMu) throw std::runtime_error("PpContext: n_mu out of range");
    if (ld_in % 4 != 0 || ld_out % 4 != 0) throw std::runtime_error("PpContext: boundary pitches must be multiples of 4 floats");
    auto alloc = [](void** p, size_t bytes) {
        CUDA_CHECK(cudaMalloc(p, std::max<size_t>(bytes, 256)));
        CUDA_CHECK(cudaMemset(*p, 0, std::max<size_t>(bytes, 256)));
    };
    alloc((void**)&act_in_, (size_t)n_mu * mb_rows * ld_in * sizeof(float));
    alloc((void**)&dz_in_, (size_t)n_mu * mb_rows * ld_out * sizeof(float));
    alloc((void**)&flags_, (size_t)kFlagWords * sizeof(uint32_t));
    alloc((void**)&epoch_, 64);
    alloc((void**)&push_done_, 64);
    CUDA_CHECK(cudaDeviceSynchronize());
}

PpContext::~PpContext() {
    cudaDeviceSynchronize();
    for (void* p : opened_) cudaIpcCloseMemHandle(p);
    cudaFree(act_in_); cudaFree(dz_in_); cudaFree(flags_); cudaFree(epoch_); cudaFree(push_done_);
}

std::string PpContext::export_handles() const {
    cudaIpcMemHandle_t h[3];
    CUDA_CHECK(cudaIpcGetMemHandle(&h[0], act_in_));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[1], dz_in_));
    CUDA_CHECK(cudaIpcGetMemHandle(&h[2], flags_));
    return std::string(reinterpret_cast<const char*>(h), sizeof(h));
}

static void open3(const std::string& blob, void* out[3], std::vector<void*>& opened) {
    if (blob.size() != 3 * sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("PpContext: bad handle blob");
    cudaIpcMemHandle_t h[3];
    memcpy(h, blob.data(), sizeof(h));
    for (int i = 0; i < 3; ++i) {
        CUDA_CHECK(cudaIpcOpenMemHandle(&out[i], h[i], cudaIpcMemLazyEnablePeerAccess));
        opened.push_back(out[i]);
    }
}

void PpContext::open_prev(const std::string& handles) {
    if (first_) throw std::runtime_error("PpContext: the first stage has no predecessor");
    void* p[3];
    open3(handles, p, opened_);
    prev_dz_in_ = (float*)p[1];
    prev_flags_ = (uint32_t*)p[2];
}

void PpContext::open_next(const std::string& handles) {
    if (last_) throw std::runtime_error("PpContext: the last stage has no successor");
    void* p[3];
    open3(handles, p, opened_);
    next_act_in_ = (float*)p[0];
    next_flags_ = (uint32_t*)p[2];
}

void PpContext::open_local(const PpContext* prev, const PpContext* next) {
    if (prev != nullptr) {
        if (first_) throw std::runtime_error("PpContext: the first stage has no predecessor");
        if (prev->ld_out_ != ld_in_ || prev->n_mu_ != n_mu_ || prev->mb_ != mb_)
            throw std::runtime_error("PpContext::open_local: the predecessor's geometry does not match this stage");
        prev_dz_in_ = prev->dz_in_;
        prev_flags_ = prev->flags_;
    }
    if (next != nullptr) {
        if (last_) throw std::runtime_error("PpContext: the last stage has no successor");
        if (next->ld_in_ != ld_out_ || next->n_mu_ != n_mu_ || next->mb_ != mb_)
            throw std::runtime_error("PpContext::open_local: the successor's geometry does not match this stage");
        next_act_in_ = next->act_in_;
        next_flags_ = next->flags_;
    }
}

}  // namespace ssb
