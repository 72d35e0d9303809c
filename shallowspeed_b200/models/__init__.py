from .layers import (LD_ALIGN, CrossEntropyLoss, Linear, Module, MSELoss, ParamArena, Parameter, ReLU,
                     Sequential, Softmax, param_ld, round_up)
from .mlp import (DEFAULT_LAYER_SIZES, MLP, mlp_sizes, stage_layer_specs, stage_sizes)

__all__ = [
    "LD_ALIGN", "CrossEntropyLoss", "Linear", "Module", "MSELoss", "ParamArena", "Parameter", "ReLU", "Sequential",
    "Softmax", "param_ld", "round_up", "DEFAULT_LAYER_SIZES", "MLP", "mlp_sizes",
    "stage_layer_specs", "stage_sizes",
]
