// Symmetric memory for the fused data-parallel path: every DP replica allocates the same
// set of buffers with cudaMalloc, exports them as CUDA IPC handles, and maps the handles of
// its peers (NVLink P2P through NVSwitch).  The resulting pointer tables (`DpPeers`) are
// what the fused kernels dereference.
//
//   W       : the weight arena itself lives in symmetric memory (owners publish new tiles)
//   stage   : [dp src][sum over layers of owned tile slots]  partial-gradient landing zone
//   arrive  : [dp src][slots]   epoch flags "src's partial for slot arrived"
//   done    : [tiles]           epoch flags "new weights of tile arrived"
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "kernels/kernels.h"

namespace ssb {

struct DpLayerGeom {
    int in, out, ld;
    int64_t w_offset;
    int block_n, n_tiles_m, n_tiles_n;
    int64_t slots, slot_floats, stage_offset;
    int tile_flag_base, slot_flag_base;
    int one_shot;
};

class DpContext {
public:
    // layers: (in, out, arena offset, ld)
    DpContext(int dp, int rank, int64_t arena_numel, const std::vector<std::tuple<int, int, int64_t, int>>& layers, float lr);
    ~DpContext();

    std::string export_handles() const;                       // 4 cudaIpcMemHandle_t, concatenated
    void open_peers(const std::vector<std::string>& handles); // index = DP rank (own entry ignored)
    // Peers that are other contexts of this process (index = DP rank, own entry ignored): their buffers enter the
    // pointer tables directly, without IPC.  Lets one GPU run one replica of a dp-way group against peers whose
    // messages a test writes and reads.
    void open_local_peers(const std::vector<const DpContext*>& ctxs);

    DpLayerParams layer_params(int layer_index) const;        // 0-based layer of the stage
    const DpPeers& peers() const { return peers_; }
    float* weights() const { return W_; }
    uint32_t* epoch_ptr() const { return epoch_; }
    int64_t arena_numel() const { return arena_numel_; }
    int dp() const { return dp_; }
    int rank() const { return rank_; }
    int64_t stage_bytes() const { return (int64_t)dp_ * stage_src_stride_ * 4; }
    // raw buffers and the strides that address them (tests)
    float* stage() const { return stage_; }
    uint32_t* arrive() const { return arrive_; }
    uint32_t* done() const { return done_; }
    uint4* ll_a() const { return llA_; }
    uint4* ll_c() const { return llC_; }
    int64_t arrive_bytes() const { return (int64_t)dp_ * slots_per_src_ * 4; }
    int64_t done_bytes() const { return (int64_t)tiles_total_ * 4; }
    int64_t ll_zone_bytes() const { return ll_tiles_ > 0 ? (int64_t)dp_ll_zone_lines(dp_, ll_tiles_) * (int64_t)sizeof(uint4) : 0; }
    int slots_per_src() const { return slots_per_src_; }
    int64_t stage_src_stride() const { return stage_src_stride_; }
    int64_t stage_parity_stride() const { return stage_parity_stride_; }
    const std::vector<DpLayerGeom>& geometry() const { return geom_; }
    int total_ctas() const { return total_ctas_; }   // sum of tiles over layers: all co-resident if <= #SMs
    // LL two-shot path (dp_ll.cu): landing zones exist when every layer is narrow enough for all tiles to be co-resident
    bool ll_enabled() const { return ll_tiles_ > 0; }
    int ll_tiles() const { return ll_tiles_; }
    DpLLParams ll_params() const;

private:
    int dp_, rank_;
    int64_t arena_numel_;
    float lr_;
    std::vector<DpLayerGeom> geom_;
    int64_t stage_src_stride_ = 0, stage_parity_stride_ = 0;
    int total_ctas_ = 0;
    int slots_per_src_ = 0, tiles_total_ = 0;
    float *W_ = nullptr, *stage_ = nullptr;
    uint32_t *arrive_ = nullptr, *done_ = nullptr, *epoch_ = nullptr;
    DpPeers peers_{};
    int ll_tiles_ = 0;
    uint4 *llA_ = nullptr, *llC_ = nullptr;
    uint4 *llA_peers_[kMaxDp] = {}, *llC_peers_[kMaxDp] = {};
    std::vector<void*> opened_;
};

}  // namespace ssb
