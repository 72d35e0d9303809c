// NVLS (NVLink SHARP) symmetric memory: weights + gradients of a stage live in physical memory that every DP
// replica binds into ONE multicast object, so a kernel can
//   * multimem.ld_reduce  a gradient element  -> the NVSwitch sums the dp replicas' copies in flight,
//   * multimem.st         a weight element    -> the switch writes it into every replica,
//   * multimem.red        a flag              -> one instruction bumps the flag on every replica.
// This is the "single-owner reduction inside the switch, multicast of the UPDATED weights" option of the
// design notes (SURVEY.md section 7.5): replicas stay bit-identical because each element is reduced exactly once
// and the result is what gets multicast.  Selected with `--comm nvls`; the peer-memory kernels of fused_dp.cu
// (`--comm fused`) remain the default.
//
// Set-up (driven from Python, parallel/engine.py:make_nvls_context, collective over the DP group):
//   1. every rank: NvlsContext(dp, rank, arena_numel)        -> sizes, granularity, support check
//   2. leader:     export_fd()  (cuMulticastCreate + POSIX fd) -> fd travels over an AF_UNIX socket (SCM_RIGHTS)
//      others:     import_fd(fd)
//   3. every rank: add_device(); barrier; bind_and_map(); barrier
// Layout of the allocation (floats): [ W: numel_pad ][ G: numel_pad ][ flags: 2 x 32 ]
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "kernels/kernels.h"

namespace ssb {

struct NvlsParams {
    float* W_uc;            // this replica's weights (unicast mapping)
    float* G_uc;            // this replica's gradients
    float* W_mc;            // multicast mapping of the same offsets
    float* G_mc;
    uint32_t* flag_in_uc;   // "my gradients are final" arrivals (multimem.red from every replica)
    uint32_t* flag_in_mc;
    uint32_t* flag_out_uc;  // "my share of the new weights is written" arrivals
    uint32_t* flag_out_mc;
    uint32_t* epoch;        // local step counter (plain device memory)
    unsigned int* cta_done; // local counter for the last-CTA election
    int64_t numel;          // floats to reduce / update (multiple of 4)
    int dp, rank;
    const float* lr;        // device float: learning rate of the running step (reduce_sgd only)
    SgdState opt;           // update rule; opt.V = LOCAL momentum arena (unicast), chunk c's entries live at rank c % dp
};

class NvlsContext {
public:
    // lr is not used: the kernel reads the learning rate from NvlsParams::lr, a device slot the caller sets (nullptr in
    // params())
    NvlsContext(int dp, int rank, int64_t arena_numel, float lr);
    ~NvlsContext();

    static bool supported();         // CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED on the current device
    int export_fd();                 // leader only: creates the multicast object, returns a POSIX fd for it
    void import_fd(int fd);          // non-leaders
    void add_device();               // cuMulticastAddDevice (every rank, before anyone binds)
    void bind_and_map();             // cuMemCreate + cuMulticastBindMem + unicast / multicast mappings

    float* weights() const { return reinterpret_cast<float*>(uc_ptr_); }
    float* grads() const { return reinterpret_cast<float*>(uc_ptr_) + numel_pad_; }
    int64_t arena_numel() const { return arena_numel_; }
    int64_t numel_pad() const { return numel_pad_; }
    size_t bytes() const { return size_; }
    int dp() const { return dp_; }
    int rank() const { return rank_; }
    NvlsParams params() const;       // valid after bind_and_map()

private:
    int dp_, rank_, dev_ = 0;
    int64_t arena_numel_, numel_pad_;
    size_t size_ = 0, gran_ = 0;
    CUmemGenericAllocationHandle mc_ = 0, mem_ = 0;
    bool have_mc_ = false, have_mem_ = false, bound_ = false;
    CUdeviceptr uc_ptr_ = 0, mc_ptr_ = 0;
    uint32_t* epoch_ = nullptr;
    unsigned int* cta_done_ = nullptr;
};

// kernels (csrc/kernels/nvls_dp.cu)
//   reduce_sgd: W <- W - *p.lr * sum_replicas(G), every replica ends with the same W (one kernel, whole arena)
//   allreduce : G <- sum_replicas(G) in place (stand-alone collective, used by the NVLS bandwidth benchmark)
cudaError_t launch_nvls_reduce_sgd(const NvlsParams& p, int max_ctas, cudaStream_t stream);
cudaError_t launch_nvls_allreduce(const NvlsParams& p, int max_ctas, cudaStream_t stream);

}  // namespace ssb
