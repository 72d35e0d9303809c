// The RES instantiations of the layer-chain kernel (mlp_chain.cuh) in single-pass TF32: residual models, always gated.  Each
// precision's RES forms are compiled apart from everything else, in parallel, so that they do not lengthen the longest
// compile.
#include "mlp_chain.cuh"

namespace ssb {

ChainKernel chain_kernel_res_tf32(ChainForm form, int ntw, bool ce, bool drop, bool gate) {
    return chain_kernel<PREC_TF32, true>(form, ntw, ce, drop, gate);
}

}  // namespace ssb
