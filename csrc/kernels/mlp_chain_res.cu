// The RES instantiations of the layer-chain kernel (mlp_chain.cuh) for every precision: residual models, always gated.
// Compiled apart from mlp_chain.cu and mlp_chain_bf16.cu, in parallel with them, so that the residual forms do not
// lengthen the longest compile.
#include "mlp_chain.cuh"

namespace ssb {

ChainKernel chain_kernel_res(int prec, ChainForm form, int ntw, bool ce, bool drop, bool gate) {
    switch (prec) {
        case PREC_TF32: return chain_kernel<PREC_TF32, true>(form, ntw, ce, drop, gate);
        case PREC_3XTF32: return chain_kernel<PREC_3XTF32, true>(form, ntw, ce, drop, gate);
        case PREC_BF16: return chain_kernel<PREC_BF16, true>(form, ntw, ce, drop, gate);
    }
    return nullptr;
}

}  // namespace ssb
