// Hidden-layer activations, shared by the host API (kernels.h) and the device helpers (ptx.cuh: act_fwd).
#pragma once

namespace ssb {

// The activation of every hidden Linear.  ACT_RELU is the model whose stored output is its own backward mask; the
// smooth ones (act_smooth) store the gate gamma = f'(z) * keep * s next to the output, and every backward site
// multiplies by it.  ops/functional.py: ACTIVATION_CODES holds the same numbers.
enum ActKind : int { ACT_RELU = 0, ACT_GELU = 1, ACT_SILU = 2, ACT_TANH = 3 };

inline bool act_valid(int kind) { return kind >= ACT_RELU && kind <= ACT_TANH; }
inline bool act_smooth(int kind) { return kind == ACT_GELU || kind == ACT_SILU || kind == ACT_TANH; }
inline const char* act_name(int kind) {
    return kind == ACT_GELU ? "gelu" : kind == ACT_SILU ? "silu" : kind == ACT_TANH ? "tanh" : "relu";
}

}  // namespace ssb
