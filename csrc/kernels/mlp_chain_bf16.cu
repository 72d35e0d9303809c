// The BF16 instantiations of the layer-chain kernel (mlp_chain.cuh), compiled apart from the TF32 / 3xTF32 ones in
// mlp_chain.cu: the build compiles the two translation units in parallel, so a third precision does not lengthen the
// longest compile.
#include "mlp_chain.cuh"

namespace ssb {

cudaError_t chain_configure_bf16() { return chain_configure_prec<PREC_BF16>(); }

cudaError_t chain_launch_bf16(const ChainPlan& plan, int ntw, bool fold, cudaStream_t stream) {
    return chain_launch_prec<PREC_BF16>(plan, ntw, fold, stream);
}

}  // namespace ssb
