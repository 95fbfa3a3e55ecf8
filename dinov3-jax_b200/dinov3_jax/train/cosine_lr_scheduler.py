"""Warm-up + cosine schedules with the reference's class interface (dinov3_jax/train/cosine_lr_scheduler.py:14-52).

Layout of the array: [zeros(freeze_iters) | linspace(start_warmup_value, base_value, warmup_iters) | cosine tail].
The reference's `trunc_extra != 0` branch reads `iters` before assigning it (:35); only trunc_extra == 0 is defined.
"""
from __future__ import annotations

import numpy as np


class CosineScheduler:
    def __init__(self, base_value, final_value, total_iters, warmup_iters=0, start_warmup_value=0, freeze_iters=0,
                 trunc_extra=0.0):
        if trunc_extra != 0:
            raise NotImplementedError("trunc_extra != 0 is undefined in the reference (cosine_lr_scheduler.py:35)")
        self.final_value = np.float64(final_value)
        self.total_iters = total_iters
        n_cos = total_iters - warmup_iters - freeze_iters
        steps = np.arange(n_cos)
        tail = final_value + 0.5 * (base_value - final_value) * (1 + np.cos(np.pi * steps / len(steps)))
        head = [np.zeros((freeze_iters,)), np.linspace(start_warmup_value, base_value, warmup_iters)]
        self.schedule = np.concatenate(head + [tail], dtype=np.float64)
        assert len(self.schedule) == self.total_iters

    def gen(self):
        return self.schedule

    def __getitem__(self, it):
        return self.final_value if it >= self.total_iters else self.schedule[it]


class linear_warmup_cosine_decay:
    """Upstream DINOv3's loss-weight (and v2) schedule (cosine_lr_scheduler.py:54-79; the reference passes
    `endpoit=False` to np.linspace, so it does not run; parity unpinned):
    [linspace(start, peak, warmup, endpoint=False) | end + (peak - end)(1 + cos(linspace(0, pi, cosine)))/2 | end ...],
    cosine_iterations defaulting to total - warmup."""

    def __init__(self, start, peak, end, warmup_iterations, total_iterations, cosine_iterations=None):
        warmup_iterations, total_iterations = int(warmup_iterations), int(total_iterations)
        if cosine_iterations is None:
            cosine_iterations = total_iterations - warmup_iterations
        cosine_iterations = int(cosine_iterations)
        remaining = total_iterations - cosine_iterations - warmup_iterations
        if warmup_iterations < 0 or cosine_iterations < 0 or remaining < 0:
            raise ValueError(f"linear_warmup_cosine_decay: warmup {warmup_iterations} + cosine {cosine_iterations} "
                             f"iterations exceed the total {total_iterations}")
        linear = np.linspace(start, peak, warmup_iterations, endpoint=False)
        cosine = (peak - end) * (np.cos(np.linspace(0, np.pi, cosine_iterations)) + 1) / 2 + end
        self.schedule = np.concatenate([linear, cosine, np.full((remaining,), fill_value=end)]).astype(np.float64)

    def gen(self):
        return self.schedule

    def __getitem__(self, idx):
        return self.schedule[idx]
