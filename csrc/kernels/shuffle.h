// Description of the per-epoch training-set permutation a kernel walks (ptx.cuh: shuffle_index), shared by the host API
// (kernels.h) and the device helpers without pulling either into the other.
#pragma once
#include <cstdint>

namespace ssb {

// Global position q of epoch `epoch` holds dataset row shuffle_index(n, seed, epoch, q), a keyed bijection on [0, n).
// Local row j of DP rank `rank` in global batch b is position q = b * gbs + j * dp + rank (the rank-strided shard of the
// global batch).  n: rows of the dataset (n < 2^32).
struct ShuffleSpec {
    uint32_t n;
    uint64_t seed;
    uint32_t epoch;
    int gbs, dp, rank;
};

}  // namespace ssb
