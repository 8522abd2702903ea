"""Detector predictions -> per-frame crop boxes on the device: the numerical part of ``lightning_pose.utils.cropzoom``.

``compute_bboxes`` replaces ``_compute_bbox_df`` + ``_calculate_bbox_size`` (reference ``utils/cropzoom.py:31-143``) and
``smooth_bboxes`` the rolling median of ``smooth_bbox`` (:355-402).  Both take and return device tensors; CSV files,
cropped videos and labeled-frame crops are host I/O and out of scope.  The boxes feed
``BatchedPredictor(..., bboxes=...)`` or ``frames_to_unlabeled_batch(..., bbox=...)`` directly.
"""
from __future__ import annotations

from typing import Sequence

import torch

from lightning_pose_b200 import ops

__all__ = ["anchor_indices", "compute_bboxes", "smooth_bboxes"]


def anchor_indices(keypoint_names: Sequence[str], anchor_keypoints: Sequence[str]) -> list[int]:
    """Indices of ``anchor_keypoints`` among ``keypoint_names`` (the names a ``PredictionHandler`` labels its table
    with), in keypoint order, as the reference selects its DataFrame columns; an empty list means all keypoints."""
    names = list(keypoint_names)
    invalid = set(anchor_keypoints) - set(names)
    if invalid:
        raise ValueError(f"Anchor keypoints not found in DataFrame: {invalid}")
    wanted = set(anchor_keypoints)
    return [i for i, n in enumerate(names) if n in wanted]


def compute_bboxes(keypoints: torch.Tensor, anchor_indices: Sequence[int] = (), crop_ratio: float | None = None,
                   crop_height: int | None = None, crop_width: int | None = None) -> torch.Tensor:
    """One box per frame around the anchor keypoints: (N, 4) fp32 [x, y, h, w] holding integers.

    ``keypoints``: (N, K, 2) frame-pixel keypoints, or a ``BatchedPredictor`` (N, 3K) prediction table, read in place.
    ``crop_ratio`` mode: a square of side ceil(crop_ratio * the larger of the x and y spans), bumped to even; fixed mode:
    ``crop_height`` x ``crop_width``, each bumped to even.  The box is centred on the anchors' mean; as in the
    reference, its x is the centroid's x minus h // 2 and its y the centroid's y minus w // 2.  Frames whose anchors
    hold a NaN get a NaN row (the reference casts NaN to an undefined integer).
    """
    fixed_size_mode = crop_height is not None and crop_width is not None
    if fixed_size_mode and crop_ratio is not None:
        raise ValueError('provide either crop_ratio or (crop_height, crop_width), not both.')
    if not fixed_size_mode and crop_ratio is None:
        raise ValueError('one of crop_ratio or (crop_height, crop_width) must be provided.')
    if crop_ratio is not None and not crop_ratio > 0:
        raise ValueError(f'crop_ratio must be positive; got {crop_ratio}')
    if fixed_size_mode and not (int(crop_height) > 0 and int(crop_width) > 0):
        raise ValueError(f'crop_height and crop_width must be positive; got {crop_height}, {crop_width}')
    return ops.bboxes_from_keypoints(keypoints, sorted(set(int(i) for i in anchor_indices)), crop_ratio, crop_height, crop_width)


def smooth_bboxes(bboxes: torch.Tensor, method: str = "median", window: int = 5) -> torch.Tensor:
    """Centred rolling median of each box column over ``window`` frames, rounded half to even: what ``smooth_bbox``
    writes (pandas ``rolling(window, center=True, min_periods=1).median().round(0)``).  NaN entries are skipped; a
    window holding only NaN stays NaN."""
    supported_methods = ('median',)
    if method not in supported_methods:
        raise ValueError(
            f'unsupported method {method!r}; choose one of {supported_methods}.'
        )
    if int(window) < 1:
        raise ValueError(f'window must be >= 1; got {window}')
    return ops.bboxes_rolling_median(bboxes, int(window))
