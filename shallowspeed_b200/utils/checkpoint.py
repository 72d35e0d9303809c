"""Per-stage checkpoint / resume.  The reference package has none (only the side script
pickles a state_dict, scripts/DDP_PyTorch_MNIST.py:157); SURVEY.md section 5 lists it as an
auxiliary subsystem.  Format: ``stage{S}of{P}.pt`` holding the flat weight arena plus
the layer dims, so a checkpoint can only be loaded into the same DP x PP layout's stage.
Runs with SGD momentum add the flat momentum arena (same layout as the weights) under
``"momentum"``; momentum-free checkpoints are unchanged."""
from __future__ import annotations

from pathlib import Path

import torch

# settings a checkpoint without them was written under (plain SGD, the MSE loss, a constant learning rate)
_HPARAM_DEFAULTS = {"momentum": 0.0, "weight_decay": 0.0, "nesterov": False, "loss": "mse",
                    "lr_schedule": {"kind": "constant"}}


def _path(directory, stage, n_stages):
    return Path(directory) / f"stage{stage}of{n_stages}.pt"


def save_stage(model, directory, stage, n_stages, step=0, hparams=None, momentum=None):
    """``hparams`` (lr, global batch, seed mode, schedule ...) travel with the weights so that a resume can refuse to
    continue a run under different settings.  ``momentum``: the stage's full momentum arena (None without momentum)."""
    Path(directory).mkdir(parents=True, exist_ok=True)
    ck = {"blocks": model.arena.blocks, "weights": model.arena.weights.detach().cpu().clone(),
          "sizes": model.sizes, "step": step, "hparams": dict(hparams or {})}
    if momentum is not None:
        ck["momentum"] = momentum.detach().cpu().clone()
    torch.save(ck, _path(directory, stage, n_stages))


def load_stage(model, directory, stage, n_stages, expect_hparams=None):
    """Load this stage's weights (and its momentum arena into ``model.arena.momentum`` when both exist); returns the
    global step the checkpoint was taken at.  Every key of ``expect_hparams`` that the checkpoint also recorded must
    match (a resumed run continues the SAME run); a checkpoint that predates the momentum settings counts as plain SGD."""
    ck = torch.load(_path(directory, stage, n_stages), map_location="cpu")
    assert [tuple(b) for b in ck["blocks"]] == [tuple(b) for b in model.arena.blocks], "checkpoint/model layout mismatch"
    saved = {**_HPARAM_DEFAULTS, **(ck.get("hparams", {}) or {})}
    for k, v in (expect_hparams or {}).items():
        if k in saved and saved[k] != v:
            raise ValueError(f"checkpoint was written with {k}={saved[k]!r}, this run uses {k}={v!r}")
    model.arena.weights.copy_(ck["weights"].to(model.arena.weights.device))
    if "momentum" in ck and model.arena.momentum is not None:
        n = ck["momentum"].numel()
        model.arena.momentum[:n].copy_(ck["momentum"].to(model.arena.momentum.device))
    return int(ck.get("step", 0))
