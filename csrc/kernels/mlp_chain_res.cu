// The RES instantiations of the layer-chain kernel (mlp_chain.cuh) for every precision: residual models, always gated.
// Compiled apart from mlp_chain.cu and mlp_chain_bf16.cu, in parallel with them, so that the residual forms do not
// lengthen the longest compile.
#include "mlp_chain.cuh"

namespace ssb {

template <int PREC>
static cudaError_t configure_res() {
    cudaError_t e;
    if ((e = chain_configure_kind<PREC, false, true, true>()) != cudaSuccess) return e;
    return chain_configure_kind<PREC, true, true, true>();
}

template <int PREC>
static cudaError_t launch_res(const ChainPlan& plan, int ntw, bool fold, cudaStream_t stream) {
    const bool ce = plan.p.loss_kind == LOSS_CROSS_ENTROPY;
    if (plan.p.drop.on()) return chain_launch_kind<PREC, true, true, true>(plan, ntw, ce, fold, stream);
    return chain_launch_kind<PREC, false, true, true>(plan, ntw, ce, fold, stream);
}

cudaError_t chain_configure_res(int prec) {
    if (prec == PREC_TF32) return configure_res<PREC_TF32>();
    if (prec == PREC_3XTF32) return configure_res<PREC_3XTF32>();
    if (prec == PREC_BF16) return configure_res<PREC_BF16>();
    return cudaErrorInvalidValue;
}

cudaError_t chain_launch_res(const ChainPlan& plan, int ntw, bool fold, cudaStream_t stream) {
    if (plan.p.prec == PREC_TF32) return launch_res<PREC_TF32>(plan, ntw, fold, stream);
    if (plan.p.prec == PREC_3XTF32) return launch_res<PREC_3XTF32>(plan, ntw, fold, stream);
    if (plan.p.prec == PREC_BF16) return launch_res<PREC_BF16>(plan, ntw, fold, stream);
    return cudaErrorInvalidValue;
}

}  // namespace ssb
