"""Return-type contracts of the tracker loss-input methods (mirror of ``lightning_pose/models/datatypes.py``).

The reference validates loss/model compatibility by reading these TypedDict annotations
(``lightning_pose/models/factory.py:139-192``), so key names are load-bearing.
"""
from __future__ import annotations

from typing import TypedDict

import torch

__all__ = ["HeatmapTrackerLabeledOutputsDict", "HeatmapTrackerUnlabeledOutputsDict", "RegressionTrackerLabeledOutputsDict",
           "RegressionTrackerUnlabeledOutputsDict"]


class HeatmapTrackerLabeledOutputsDict(TypedDict):
    heatmaps_targ: torch.Tensor  # (batch, K, h, w)
    heatmaps_pred: torch.Tensor  # (batch, K, h, w)
    keypoints_targ: torch.Tensor  # (batch, 2K)
    keypoints_pred: torch.Tensor  # (batch, 2K)
    confidences: torch.Tensor  # (batch, K)


class HeatmapTrackerUnlabeledOutputsDict(TypedDict):
    heatmaps_pred: torch.Tensor  # (seq, K, h, w)
    keypoints_pred: torch.Tensor  # (seq, 2K) in frame coordinates, augmentation undone
    keypoints_pred_augmented: torch.Tensor  # (seq, 2K) matching heatmaps_pred
    confidences: torch.Tensor  # (seq, K)


class RegressionTrackerLabeledOutputsDict(TypedDict):
    keypoints_targ: torch.Tensor  # (batch, 2K) model pixels
    keypoints_pred: torch.Tensor  # (batch, 2K) model pixels


class RegressionTrackerUnlabeledOutputsDict(TypedDict):
    keypoints_pred: torch.Tensor  # (seq, 2K), augmentation undone
