"""Model -> frame coordinate transform: the hot-path part of ``lightning_pose.data.bboxes``.

``model_to_frame_batch`` (reference ``data/bboxes.py:222-288``), ``norm_to_frame`` (:74-105) and, for the calibrated
multi-view losses, ``frame_to_model_batch`` (:194-219).
Like the reference, ``in_place=True`` writes the result through the caller's tensor.
"""
from __future__ import annotations

import torch

from lightning_pose_b200 import ops

__all__: list[str] = []


def norm_to_frame(keypoints: torch.Tensor, bbox: torch.Tensor) -> torch.Tensor:
    """(batch, K, 2) normalised coords * bbox (x, y, h, w) -> frame pixels; modifies ``keypoints``."""
    n, k, _ = keypoints.shape
    flat = keypoints.reshape(n, 2 * k)
    ops.remap_keypoints(flat, None, bbox, 1.0, 1.0, out=flat if flat.is_contiguous() else None)
    return keypoints


def model_to_frame_batch(batch_dict: dict, model_keypoints: torch.Tensor, in_place: bool = True) -> torch.Tensor:
    """(batch, 2K) model-pixel keypoints -> original-frame pixels using ``batch_dict['bbox']``.

    Image size comes from ``images`` / ``frames``; multiview batches (``num_views`` > 1 or
    ``is_multiview``) apply the v-th bbox quadruple to the v-th block of keypoints.
    """
    img = batch_dict["images"] if "images" in batch_dict else batch_dict["frames"]
    model_height, model_width = img.shape[-2], img.shape[-1]
    bbox = batch_dict["bbox"]
    num_views = 1
    if "num_views" in batch_dict and int(batch_dict["num_views"].max()) > 1:
        unique = batch_dict["num_views"].unique()
        if len(unique) != 1:
            raise ValueError(f"each batch element must contain the same number of views; found elements with {unique} views")
        num_views = int(unique)
    elif batch_dict.get("is_multiview", False):
        num_views = bbox.shape[1] // 4
    kp = model_keypoints
    if not (kp.is_cuda and kp.dtype == torch.float32 and kp.is_contiguous()):
        in_place = False
    out = ops.remap_keypoints(kp, None, bbox, model_height, model_width, num_views=num_views, out=kp if in_place else None)
    return out.reshape(-1, model_keypoints.shape[1])


def frame_to_model_batch(batch_dict: dict, frame_keypoints: torch.Tensor) -> torch.Tensor:
    """(batch, num_views, num_keypoints, 2) frame pixels -> model-input pixels (reference ``data/bboxes.py:194-219``).

    The v-th bbox quadruple [x, y, h, w] of ``batch_dict['bbox']`` maps view v; the model size is that of
    ``batch_dict['images']``.  Returns a new tensor, differentiable in ``frame_keypoints``."""
    img = batch_dict["images"]
    return ops.frame_to_model(frame_keypoints, batch_dict["bbox"], img.shape[-2], img.shape[-1])
