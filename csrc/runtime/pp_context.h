// Peer-memory transport for the pipeline boundaries (opt-in, `--pp-transport peer`): instead of an NCCL send/recv
// pair per micro-batch and direction, the producing stage PUSHES its boundary tile straight into the consuming
// stage's receive slot over NVLink and raises an epoch-valued flag there; the consumer's stream waits on its own
// local flag.  One-sided, so a send never blocks on the peer's schedule position (the NCCL path is a rendezvous).
//
//   act_in  [n_mu][mb x ld_in ]   written by stage s-1 (its layer-L output of micro-batch mu)
//   dz_in   [n_mu][mb x ld_out]   written by stage s+1 (gradient w.r.t. my output)
//   flags   act_arrived[n_mu], dz_arrived[n_mu]   written by the neighbours, polled locally
//           act_credit, dz_credit                  written by the neighbour that CONSUMES what I push: "your slots of
//                                                   step e are free again" (= e), checked by my pushes of step e+1
//   epoch   local step counter, bumped at the start of every step graph (all stages step in lockstep)
//
// Buffers are cudaMalloc'ed and shared with the two neighbours through CUDA IPC handles (same mechanism as DpContext).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

namespace ssb {

class PpContext {
public:
    PpContext(int n_mu, int mb_rows, int ld_in, int ld_out, bool is_first, bool is_last);
    ~PpContext();

    std::string export_handles() const;                        // 3 cudaIpcMemHandle_t: act_in, dz_in, flags
    void open_prev(const std::string& handles);                // stage s-1's export
    void open_next(const std::string& handles);                // stage s+1's export
    // test-facing: neighbours that are contexts of this process (CUDA IPC refuses the caller's own allocations); prev is
    // null on the first stage, next on the last
    void open_local(const PpContext* prev, const PpContext* next);

    // local views
    float* act_in() const { return act_in_; }
    float* dz_in() const { return dz_in_; }
    uint32_t* epoch_ptr() const { return epoch_; }
    uint32_t* push_done_ptr() const { return push_done_; }
    const uint32_t* act_arrived(int mu) const { return flags_ + mu; }
    const uint32_t* dz_arrived(int mu) const { return flags_ + kMaxMu + mu; }
    const uint32_t* act_credit() const { return flags_ + 2 * kMaxMu; }          // written by next: my act pushes may reuse its slots
    const uint32_t* dz_credit() const { return flags_ + 2 * kMaxMu + 32; }      // written by prev
    const uint32_t* flags() const { return flags_; }                            // all kFlagWords words
    // neighbour views (nullptr when there is no such neighbour)
    float* next_act_in(int mu) const { return next_act_in_ ? next_act_in_ + (size_t)mu * mb_ * ld_out_ : nullptr; }
    uint32_t* next_act_arrived(int mu) const { return next_flags_ ? next_flags_ + mu : nullptr; }
    uint32_t* next_dz_credit() const { return next_flags_ ? next_flags_ + 2 * kMaxMu + 32 : nullptr; }
    float* prev_dz_in(int mu) const { return prev_dz_in_ ? prev_dz_in_ + (size_t)mu * mb_ * ld_in_ : nullptr; }
    uint32_t* prev_dz_arrived(int mu) const { return prev_flags_ ? prev_flags_ + kMaxMu + mu : nullptr; }
    uint32_t* prev_act_credit() const { return prev_flags_ ? prev_flags_ + 2 * kMaxMu : nullptr; }

    int n_mu() const { return n_mu_; }
    int mb_rows() const { return mb_; }
    int ld_in() const { return ld_in_; }
    int ld_out() const { return ld_out_; }

    static constexpr int kMaxMu = 256;
    static constexpr int kFlagWords = 2 * kMaxMu + 64;

private:
    int n_mu_, mb_, ld_in_, ld_out_;
    bool first_, last_;
    float *act_in_ = nullptr, *dz_in_ = nullptr;
    uint32_t *flags_ = nullptr, *epoch_ = nullptr, *push_done_ = nullptr;
    float *next_act_in_ = nullptr, *prev_dz_in_ = nullptr;
    uint32_t *next_flags_ = nullptr, *prev_flags_ = nullptr;
    std::vector<void*> opened_;
};

// kernels (csrc/kernels/pp_transport.cu)
// push: wait until credit >= epoch-1, copy n floats (multiple of 4) to the peer slot, fence, raise the peer's flag to epoch
// tiles of at most this many float4 (32 KB) are pushed by ONE CTA without a completion counter: safe to run concurrently
static constexpr int64_t kPpSmallTileF4 = 2048;
cudaError_t launch_pp_push(const float* src, float* dst_peer, int64_t n, uint32_t* flag_peer, const uint32_t* credit_local,
                           const uint32_t* epoch, uint32_t* done_counter, cudaStream_t stream);
// wait: spin (bounded) until *flag_local >= epoch
cudaError_t launch_pp_wait(const uint32_t* flag_local, const uint32_t* epoch, cudaStream_t stream);
// credit: tell the producers of my receive slots that step `epoch` no longer needs them
cudaError_t launch_pp_credit(uint32_t* credit_a, uint32_t* credit_b, const uint32_t* epoch, cudaStream_t stream);

}  // namespace ssb
