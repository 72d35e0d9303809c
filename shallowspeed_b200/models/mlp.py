"""MLP model family + pipeline-stage partitioner.

Parity with the reference's ``MLP(sizes, stage_idx, n_stages, batch_size)``
(``shallowspeed/layers.py:236-270``): ``len(sizes) % n_stages == 0``; stage *s* owns
``sizes[s*k : s*k+k+1]`` (k = len(sizes)//n_stages), i.e. k Linears, the last stage
k-1 Linears + Softmax + MSELoss (or, with ``loss="cross_entropy"``, + CrossEntropyLoss); the final Linear carries no ReLU only when it sits on
the last stage; ``in_dim`` / ``out_dim`` are exposed for buffer allocation.

All Linears of a stage share one ``ParamArena`` (flat weights + flat grads).
"""
from __future__ import annotations

from typing import Optional, Sequence, Union

import torch

from ..ops.functional import check_activation, check_dropout, check_loss, dropout_scale
from .layers import CrossEntropyLoss, Linear, MSELoss, ParamArena, Sequential, Softmax

DEFAULT_LAYER_SIZES = [784, 128, 127, 126, 125, 124, 123, 10]  # reference train.py:98


def stage_sizes(sizes: Sequence[int], stage_idx: int, n_stages: int):
    """The slice of ``sizes`` owned by ``stage_idx`` (reference layers.py:242-250)."""
    assert len(sizes) % n_stages == 0, (
        f"len(sizes)={len(sizes)} must be divisible by the number of pipeline stages {n_stages}"
    )
    assert 0 <= stage_idx < n_stages
    k = len(sizes) // n_stages
    return list(sizes[stage_idx * k : min(len(sizes), k * stage_idx + k + 1)])


def stage_layer_specs(sizes: Sequence[int], stage_idx: int, n_stages: int):
    """[(in, out, relu, global_layer_index)] for the Linears of a stage."""
    local = stage_sizes(sizes, stage_idx, n_stages)
    is_last = stage_idx == n_stages - 1
    k = len(sizes) // n_stages
    specs = []
    for i in range(len(local) - 1):
        relu = not (i == len(local) - 2 and is_last)
        specs.append((local[i], local[i + 1], relu, stage_idx * k + i))
    return specs


def residual_layers(sizes: Sequence[int], n_stages: int = 1):
    """Global indices of the Linears a residual model wraps in a skip: those with an activation (stage_layer_specs) and
    equal widths.  The same set for every stage of a layout."""
    return [g for s in range(n_stages) for i, o, relu, g in stage_layer_specs(sizes, s, n_stages) if relu and i == o]


def mlp_sizes(hidden: int, n_layers: int, in_dim: int = 784, out_dim: int = 10):
    """``n_layers`` Linears: in_dim -> hidden x (n_layers-1) -> out_dim."""
    assert n_layers >= 1
    return [in_dim] + [hidden] * (n_layers - 1) + [out_dim]


class MLP(Sequential):
    def __init__(self, sizes: Sequence[int], stage_idx: int, n_stages: int, batch_size: int,
                 device="cpu", seed_mode: str = "shape", verbose: bool = False, loss: str = "mse",
                 dropout: float = 0.0, dropout_seed: int = 0, activation: str = "relu", residual: bool = False):
        """
        :param batch_size: the GLOBAL batch size - the loss gradient is scaled by
            1/batch_size so that summing over micro-batches and DP replicas reproduces
            sequential training (reference layers.py:237-241).
        :param seed_mode: "shape" = reference-identical shape-seeded init;
            "index" = additionally mixes the global layer index into the seed.
        :param loss: "mse" = the reference's Softmax + MSELoss head; "cross_entropy" =
            CrossEntropyLoss on the logits.  Every stage records it (the native engine reads it).
        :param dropout: inverted dropout with this drop probability on the output of every Linear that has a ReLU (every
            hidden layer, never the logits), in training only.  The mask of an element is a pure function of
            (dropout_seed, global layer index, feature, the sample's position in the global batch, dropout_step)
            (ops.functional.dropout_mask), so every DP x PP layout draws the same masks.  Under pp=8 the default model's
            stage 6 ends in a 123->10 Linear that carries a ReLU (the stage rule above); it is dropped like any other.
        :param activation: the activation of every Linear that has one (every hidden layer, never the logits): "relu"
            (the reference's), "gelu" (erf form), "silu" or "tanh".  The pp=8 stage-6 Linear above carries it as well.
        :param residual: an identity skip around every Linear that has an activation and as many outputs as inputs,
            a = x + drop(f(x W^T + b)) (models.layers.Linear).  ValueError when no Linear of the whole model (all stages
            of the layout) qualifies, e.g. the reference's 784-128-127-...-10.
        """
        if not isinstance(residual, bool):
            raise ValueError(f"residual must be a bool, got {residual!r}")
        res_layers = set(residual_layers(sizes, n_stages)) if residual else set()
        if residual and not res_layers:
            raise ValueError(f"residual=True, but no Linear of the model {list(sizes)} has an activation and equal input and "
                             "output widths")
        self.residual = residual
        assert seed_mode in ("shape", "index")
        self.loss = check_loss(loss)
        self.activation = check_activation(activation)
        self.dropout, self.dropout_seed = check_dropout(dropout, dropout_seed)
        self._dropout_step = 0
        self.dropout_shard = (0, 1)   # (DP rank, DP size) of the rows this replica forwards (set by the pipeline VM)
        self.sizes = list(sizes)
        self.stage_idx, self.n_stages, self.batch_size = stage_idx, n_stages, batch_size
        specs = stage_layer_specs(sizes, stage_idx, n_stages)
        local = stage_sizes(sizes, stage_idx, n_stages)
        self.is_last_stage = stage_idx == n_stages - 1
        self.arena = ParamArena([(o, i) for i, o, _, _ in specs], device=device)
        layers = [
            Linear(i, o, activation=self.activation if relu else None, arena=self.arena, block_index=bi,
                   layer_index=gidx if seed_mode == "index" else None, residual=gidx in res_layers)
            for bi, (i, o, relu, gidx) in enumerate(specs)
        ]
        self.linears = list(layers)
        self.layer_base = specs[0][3] if specs else 0   # global index of this stage's first Linear
        if self.dropout > 0.0:
            scale = dropout_scale(self.dropout)
            for lin, (_, _, relu, gidx) in zip(layers, specs):
                if relu:
                    lin.dropout = (self.dropout, self.dropout_seed, gidx, scale)
                    lin.activation.dropout_scale = scale
        if self.is_last_stage and self.loss == "cross_entropy":
            layers.append(CrossEntropyLoss(batch_size=batch_size))
        elif self.is_last_stage:
            layers.append(Softmax())
            layers.append(MSELoss(batch_size=batch_size))
        super().__init__(layers)
        if verbose:
            print(layers)
        self.in_dim = local[0]
        self.out_dim = local[-1]  # softmax & loss keep the width

    def to(self, device):
        self.arena.to(device)
        return self

    @property
    def dropout_step(self) -> int:
        """The optimizer step (0-based, global) whose dropout masks the next training step draws."""
        return self._dropout_step

    @dropout_step.setter
    def dropout_step(self, step):
        if isinstance(step, bool) or not isinstance(step, int) or step < 0:
            raise ValueError(f"dropout_step must be an integer >= 0, got {step!r}")
        self._dropout_step = int(step)

    def forward(self, inputs, mubatch_id=0):
        if self._training and self.dropout > 0.0:
            # row n of micro-batch mu of the DP-local batch on replica r of dp is sample (mu * rows + n) * dp + r
            rank, dp = self.dropout_shard
            n = inputs.shape[0]
            samples = (mubatch_id * n + torch.arange(n, dtype=torch.int64)) * dp + rank
            for lin in self.linears:
                lin.dropout_rows = (samples, self._dropout_step)
        return super().forward(inputs, mubatch_id)

    @property
    def loss_layer(self) -> Optional[Union[MSELoss, CrossEntropyLoss]]:
        return self.layers[-1] if self.is_last_stage else None
