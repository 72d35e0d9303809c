"""Learning-rate schedules: linear warmup followed by a constant, step, cosine or linear decay.

``LRSchedule(base_lr, kind, ...)(i)`` is the learning rate of optimizer step ``i`` (0-based, global: it keeps counting
across a resume).  The rate is evaluated in fp64 from a closed form and rounded to fp32 once, so every replica, every
pipeline stage and the CPU oracle use the same bits.  With ``W = warmup_steps``, ``f = warmup_start_factor``,
``j = i - W`` and the horizon ``H = total_steps - W``:

    i < W      base * (f + (1 - f) * i / W)                      torch LinearLR(start_factor=f, total_iters=W)
    constant   base
    step       base * gamma ** (j // step_size)                  torch StepLR
    cosine     min_lr + (base - min_lr) * (1 + cos(pi * j / H)) / 2, held at min_lr for j >= H
                                                                 torch CosineAnnealingLR(T_max=H, eta_min=min_lr)
    linear     base + (min_lr - base) * min(j, H) / H            torch LinearLR(end_factor=min_lr / base, total_iters=H)

Warmup followed by a decay is ``torch.optim.lr_scheduler.SequentialLR([LinearLR(...), <decay>], milestones=[W])``.
One deliberate difference: torch's cosine schedule is periodic past ``T_max``; this one holds ``min_lr``.

Anything that takes a schedule (``Trainer(lr_schedule=...)``) also takes any callable ``step -> lr``.
"""
from __future__ import annotations

import math
import struct

from .optimizer import check_hparams

KINDS = ("constant", "step", "cosine", "linear")
DEFAULT_WARMUP_START_FACTOR = 1.0 / 3.0   # torch LinearLR's default start_factor


def to_fp32(x: float) -> float:
    """``x`` rounded to the nearest fp32 value (returned as a Python float)."""
    return struct.unpack("f", struct.pack("f", x))[0]


def _is_int(v) -> bool:
    return isinstance(v, int) and not isinstance(v, bool)


class LRSchedule:
    def __init__(self, base_lr, kind="constant", total_steps=None, warmup_steps=0,
                 warmup_start_factor=DEFAULT_WARMUP_START_FACTOR, min_lr=0.0, step_size=None, gamma=0.1):
        try:
            check_hparams(float(base_lr), 0.0, 0.0, False)
        except (TypeError, ValueError) as e:
            raise ValueError(f"LRSchedule: base_lr: {e}") from None
        if not math.isfinite(float(base_lr)):
            raise ValueError(f"LRSchedule: base_lr must be finite, got {base_lr}")
        if kind not in KINDS:
            raise ValueError(f"LRSchedule: kind must be one of {KINDS}, got {kind!r}")
        if not _is_int(warmup_steps) or warmup_steps < 0:
            raise ValueError(f"LRSchedule: warmup_steps must be an integer >= 0, got {warmup_steps!r}")
        if not 0.0 < float(warmup_start_factor) <= 1.0:
            raise ValueError(f"LRSchedule: warmup_start_factor must be in (0, 1], got {warmup_start_factor}")
        if total_steps is not None and (not _is_int(total_steps) or total_steps < 0):
            raise ValueError(f"LRSchedule: total_steps must be an integer >= 0, got {total_steps!r}")
        if kind in ("cosine", "linear"):
            if total_steps is None or total_steps <= warmup_steps:
                raise ValueError(f"LRSchedule: {kind} decay needs total_steps > warmup_steps, got total_steps="
                                 f"{total_steps!r}, warmup_steps={warmup_steps}")
            if not 0.0 <= float(min_lr) <= float(base_lr):
                raise ValueError(f"LRSchedule: min_lr must be in [0, base_lr], got {min_lr}")
        if kind == "step":
            if not _is_int(step_size) or step_size < 1:
                raise ValueError(f"LRSchedule: step decay needs an integer step_size >= 1, got {step_size!r}")
            if not 0.0 < float(gamma) <= 1.0:
                raise ValueError(f"LRSchedule: gamma must be in (0, 1], got {gamma}")
        self.base_lr, self.kind = float(base_lr), kind
        self.total_steps, self.warmup_steps = total_steps, int(warmup_steps)
        self.warmup_start_factor = float(warmup_start_factor)
        self.min_lr, self.step_size, self.gamma = float(min_lr), step_size, float(gamma)

    def exact(self, i: int) -> float:
        """The fp64 rate of step ``i`` before the one rounding to fp32."""
        if not _is_int(i) or i < 0:
            raise ValueError(f"LRSchedule: step must be an integer >= 0, got {i!r}")
        base, W = self.base_lr, self.warmup_steps
        if i < W:
            f = self.warmup_start_factor
            return base * (f + (1.0 - f) * i / W)
        j = i - W
        if self.kind == "constant":
            return base
        if self.kind == "step":
            return base * self.gamma ** (j // self.step_size)
        H = self.total_steps - W
        if j >= H:
            return self.min_lr
        if self.kind == "cosine":
            return self.min_lr + (base - self.min_lr) * (1.0 + math.cos(math.pi * j / H)) / 2.0
        return base + (self.min_lr - base) * j / H

    def schedule(self, i: int) -> float:
        """The learning rate of optimizer step ``i`` (0-based, global), an fp32 value."""
        return to_fp32(self.exact(i))

    __call__ = schedule

    def spec(self) -> dict:
        """The settings that define the schedule besides ``base_lr``, as a plain dict (checkpoints record it next to
        ``lr``).  A constant schedule without warmup is ``{"kind": "constant"}``."""
        d = {"kind": self.kind}
        if self.warmup_steps:
            d.update(warmup_steps=self.warmup_steps, warmup_start_factor=self.warmup_start_factor)
        if self.kind == "step":
            d.update(step_size=self.step_size, gamma=self.gamma)
        if self.kind in ("cosine", "linear"):
            d.update(total_steps=self.total_steps, min_lr=self.min_lr)
        return d

    def __repr__(self):
        return f"LRSchedule(base_lr={self.base_lr!r}, {', '.join(f'{k}={v!r}' for k, v in self.spec().items())})"
