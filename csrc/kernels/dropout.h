// Description of the dropout masks a kernel draws (ptx.cuh: dropout_keep), shared by the host API (kernels.h) and the
// device helpers without pulling either into the other.
#pragma once
#include <cstdint>

namespace ssb {

// Inverted dropout of a ReLU'd Linear output (ptx.cuh: dropout_keep).  threshold = floor(p * 2^32) and scale =
// float32(1 / (1 - p)) are formed on the host in fp64 (dropout_spec); threshold == 0 is the dropout-free model.  The
// mask of element (feature f, row n) is a pure function of (seed, layer, f, sample, *step) with sample =
// (row_base + n) * dp + rank: rows are rank-strided shards of the global batch, row_base the DP-local row of the launch's
// row 0.  step: device slot of the optimizer step whose masks are drawn (rewritten between steps without re-planning).
struct DropoutSpec {
    uint32_t threshold;
    float scale;
    uint64_t seed;
    const uint32_t* step;
    int layer;                    // global index of the Linear (chain: of the launch's first layer)
    int row_base, dp, rank;
    bool on() const { return threshold != 0u; }
};

}  // namespace ssb
