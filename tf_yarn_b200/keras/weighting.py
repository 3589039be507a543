"""Keras sample weighting (``sample_weight`` / ``class_weight``) for the autograd and eager engines.

The weight of sample i is ``sample_weight[i] * class_weight[class(y_i)]``; a missing factor, or a label outside
the class table, counts as 1.  ``class(y)`` is the integer label of sparse labels, the argmax of one-hot labels and
``round(y)`` of binary targets.  The loss is ``sum(w * l) / B`` (Keras' SUM_OVER_BATCH_SIZE), not the mean over
the weights.  Everything stays on the device: no host copy inside a CUDA-graph capture.
(The fused classifier head of the fast path does the same inside its kernel.)"""
from __future__ import annotations

from typing import Callable, Optional

import torch


def class_index(y: torch.Tensor) -> torch.Tensor:
    if torch.is_floating_point(y):
        if y.dim() >= 2 and y.shape[-1] > 1:
            return y.argmax(dim=-1).reshape(-1)
        return torch.round(y).long().reshape(-1)
    return y.long().reshape(-1)


def sample_weights(y, sample_weight: Optional[torch.Tensor],
                   class_table: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Per-sample weights ``[B]`` (fp32), or None when neither factor is given."""
    w = None
    if class_table is not None:
        if not torch.is_tensor(y):
            raise ValueError("class_weight needs a single label tensor per batch")
        cls = class_index(y)
        n = class_table.numel()
        w = class_table[cls.clamp(0, n - 1)].masked_fill((cls < 0) | (cls >= n), 1.0)
    if sample_weight is not None:
        sw = sample_weight.reshape(-1).float()
        w = sw if w is None else sw * w
    return w


def weighted_loss(per_sample_loss: Callable, y, out, w: torch.Tensor) -> torch.Tensor:
    """``sum(w * l) / B``."""
    per = per_sample_loss(y, out)
    return (per * w.reshape(-1)).sum() / per.shape[0]
