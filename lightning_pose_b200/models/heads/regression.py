"""Linear regression head (mirror of ``lightning_pose/models/heads/regression.py``).

The reference's backbone ends in torchvision's ``avgpool`` for regression models, so its head receives
``(B, C, 1, 1)`` and is ``features.reshape(B, C)`` -> ``nn.Linear(C, 2K)``.  Here the pool is folded into the head: the
trackers cut the backbone before ``avgpool`` and the head averages the ``(B, C, h, w)`` map itself, reading every feature
byte once, in one autograd node whose forward and backward are ``lpb_regression_head_fwd/_bwd``.  With ``h = w = 1``
(a caller's own backbone that keeps its pool) this is the reference's head exactly.  ``avgpool`` has no parameters, so
the state-dict keys stay the reference's: ``linear_layer.weight`` / ``linear_layer.bias``.
"""
from __future__ import annotations

import torch
from torch import nn

from lightning_pose_b200 import ops

__all__: list[str] = []


class LinearRegressionHead(nn.Module):
    """``(B, C, h, w)`` features -> ``(B, num_targets)`` coordinates: spatial mean, then ``linear_layer``."""

    def __init__(self, in_channels: int, num_targets: int) -> None:
        super().__init__()
        self.linear_layer = nn.Linear(in_channels, num_targets)

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        if features.dim() == 2:  # already pooled (B, C): the reference's reshape accepts it too
            features = features[:, :, None, None]
        return ops.regression_head(features, self.linear_layer.weight, self.linear_layer.bias)
