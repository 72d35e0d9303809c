// The single-pass TF32 instantiations of the layer-chain kernel (mlp_chain.cuh), compiled apart from the other
// precisions: the build compiles the chain's translation units in parallel, so a precision does not lengthen the
// longest compile.
#include "mlp_chain.cuh"

namespace ssb {

ChainKernel chain_kernel_tf32(ChainForm form, int ntw, bool ce, bool drop, bool gate) {
    return chain_kernel<PREC_TF32, false>(form, ntw, ce, drop, gate);
}

}  // namespace ssb
