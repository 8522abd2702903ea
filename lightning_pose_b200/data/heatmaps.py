"""Gaussian target generation and windowed evaluation: drop-in for ``lightning_pose.data.heatmaps``.

``generate_heatmaps`` (reference ``lightning_pose/data/heatmaps.py:11-87``) and
``evaluate_heatmaps_at_location`` (:90-142) with the reference's signatures; both run as CUDA
kernels (``csrc/targets.cu``).  The DataLoader-worker call site of the reference
(``lightning_pose/data/datasets.py:516``, CPU tensors, no CUDA context) is data-layer and stays with
the reference; these functions serve the GPU side (tracker / losses).
"""
from __future__ import annotations

import math

import torch

from lightning_pose_b200 import ops

__all__: list[str] = []


def generate_heatmaps(
    keypoints: torch.Tensor,
    height: int,
    width: int,
    output_shape: tuple[int, int],
    sigma: float = 1.25,
    keep_gradients: bool = False,
    visibility: torch.Tensor | None = None,
) -> torch.Tensor:
    """(batch, num_keypoints, 2) image-pixel keypoints -> normalised Gaussian heatmaps.

    NaN / out-of-bounds keypoints give all-zero planes; with ``visibility``: 0 -> zeros,
    1 -> uniform, 2 -> Gaussian (zeros if also out of bounds), any other value (3, -1, ...) ->
    the clamped Gaussian, as the reference's masks leave it.  ``keep_gradients=True`` makes the
    result differentiable with respect to ``keypoints``.
    """
    return ops.generate_heatmaps(keypoints, height, width, output_shape, sigma, keep_gradients, visibility)


def evaluate_heatmaps_at_location(
    heatmaps: torch.Tensor, locs: torch.Tensor, sigma: float = 1.25, num_stds: int = 2
) -> torch.Tensor:
    """Sum of the (2r+1)^2 window (r = floor(sigma * num_stds)) around trunc(locs), zero outside."""
    return ops.evaluate_heatmaps_at_location(heatmaps, locs, int(math.floor(sigma * num_stds)))


class GaussianTargets:
    """Lazy Gaussian targets: what a labeled batch carries when the targets are generated on the GPU (SURVEY 8f-2).

    The reference's DataLoader workers render ``(K, h, w)`` target planes on the CPU
    (``data/datasets.py:486-525``) and ship 627 KB per frame to the device.  Here the batch ships only
    ``(keypoints, visibility)``; the supervised loss consumes this object: ``HeatmapMSELoss``, ``HeatmapKLLoss``,
    ``HeatmapJSLoss`` and ``ReprojectionHeatmapLoss`` evaluate targets and loss in one kernel without ever writing the
    planes (``ops.heatmap_loss_from_keypoints``); ``materialize()`` renders them for any other consumer.  ``keypoints``
    are model-image pixels AFTER augmentation; the out-of-frame -> NaN rule of ``compute_heatmap`` (:496-508) is applied
    on the device at construction unless ``ignore_nans`` (the reference's flag: calibrated multi-view validation
    batches skip the rule, ``datasets.py:1161-1164``).
    """

    def __init__(self, keypoints: torch.Tensor, height: int, width: int, output_shape: tuple[int, int], sigma: float = 1.25,
                 visibility: torch.Tensor | None = None, ignore_nans: bool = False) -> None:
        kp = keypoints.reshape(keypoints.shape[0], -1, 2)
        self.keypoints = kp if ignore_nans else ops.keypoints_mask_oob(kp, height, width)
        self.height, self.width, self.output_shape, self.sigma = int(height), int(width), (int(output_shape[0]), int(output_shape[1])), float(sigma)
        self.visibility = visibility if (visibility is not None and visibility.numel() > 0) else None

    @property
    def shape(self) -> tuple[int, int, int, int]:
        return (self.keypoints.shape[0], self.keypoints.shape[1], *self.output_shape)

    @property
    def device(self) -> torch.device:
        return self.keypoints.device

    def materialize(self) -> torch.Tensor:
        return generate_heatmaps(self.keypoints, self.height, self.width, self.output_shape, self.sigma, visibility=self.visibility)
