"""Camera geometry of the calibrated multi-view losses: the training-step part of ``lightning_pose.data.cameras``.

``project_camera_pairs_to_3d`` (reference ``data/cameras.py:22-83``) and ``project_3d_to_2d`` (:86-171) with the
reference's parameter names, shapes and NaN behaviour, each one CUDA launch forward and one backward
(``csrc/cameras.cu``), with no host sync.  Camera tensors are batch data: they get no gradient.  ``CameraGroup`` and
``triangulate_fast`` belong to the data layer (NumPy / OpenCV in DataLoader workers) and are not mirrored.
"""
from __future__ import annotations

import torch

from lightning_pose_b200 import ops

__all__: list[str] = []


def project_camera_pairs_to_3d(
    points: torch.Tensor,
    intrinsics: torch.Tensor,
    extrinsics: torch.Tensor,
    dist: torch.Tensor,
) -> torch.Tensor:
    """(batch, num_views, num_keypoints, 2) frame pixels -> (batch, cam_pair, num_keypoints, 3) world points.

    Each view is undistorted, then every camera pair (``itertools.combinations`` order) is triangulated by the DLT.
    A keypoint that is NaN in either view of a pair is NaN in that pair's output."""
    return ops.triangulate_pairs(points, intrinsics, extrinsics, dist)


def project_3d_to_2d(
    points_3d: torch.Tensor,
    intrinsics: torch.Tensor,
    extrinsics: torch.Tensor,
    dist: torch.Tensor,
) -> torch.Tensor:
    """(batch, num_keypoints, 3) world points -> (batch, num_views, num_keypoints, 2) frame pixels.

    Pinhole projection, then distortion for every (batch, view) whose ``dist`` row is not all zero.  A NaN point is
    NaN in every view."""
    return ops.project_points(points_3d, intrinsics, extrinsics, dist)
