"""``shallowspeed_b200.layers`` - same module name/surface as the reference's
``shallowspeed/layers.py``; implementation lives in ``models``."""
from .models.layers import (CrossEntropyLoss, Linear, Module, MSELoss, ParamArena, Parameter, ReLU,  # noqa: F401
                            Sequential, Softmax)
from .models.mlp import MLP, mlp_sizes, stage_layer_specs, stage_sizes  # noqa: F401
