// Tensor-core precision of the GEMMs, shared by the host API (kernels.h) and the device helpers (ptx.cuh: warp_mma_kblock).
#pragma once

namespace ssb {

// Operands and results stay fp32 in memory in every mode; only the products differ.  PREC_TF32: one TF32 MMA per k8.
// PREC_3XTF32: three (fp32-equivalent products).  PREC_BF16: each operand rounded to bf16 (nearest even) in registers,
// one BF16 MMA per k16, fp32 accumulation.  0 and 1 are what the former boolean `split` meant, so a bool that still
// arrives as the precision selects the same products.  ops/cuda.py: PRECISION_CODES holds the same numbers.
enum Precision : int { PREC_TF32 = 0, PREC_3XTF32 = 1, PREC_BF16 = 2 };

inline bool prec_valid(int prec) { return prec >= PREC_TF32 && prec <= PREC_BF16; }

}  // namespace ssb
