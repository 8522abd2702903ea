"""Model -> frame coordinate transform: the hot-path part of ``lightning_pose.data.bboxes``.

``model_to_frame_batch`` (reference ``data/bboxes.py:222-288``), ``norm_to_frame`` (:74-105), for the calibrated
multi-view losses ``frame_to_model_batch`` (:194-219), and for crop-zoom pose models ``crop_and_resize_frames`` (:291-343).
Like the reference, ``in_place=True`` writes the result through the caller's tensor.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

from lightning_pose_b200 import ops

__all__: list[str] = []


def norm_to_frame(keypoints: torch.Tensor, bbox: torch.Tensor) -> torch.Tensor:
    """(batch, K, 2) normalised coords * bbox (x, y, h, w) -> frame pixels; modifies ``keypoints``."""
    n, k, _ = keypoints.shape
    flat = keypoints.reshape(n, 2 * k)
    ops.remap_keypoints(flat, None, bbox, 1.0, 1.0, out=flat if flat.is_contiguous() else None)
    return keypoints


def crop_and_resize_frames(frames: torch.Tensor, bbox_rows, resize_dims: Sequence[int]) -> tuple[torch.Tensor, torch.Tensor]:
    """Crop each frame to its box and resize the crops to ``resize_dims`` (reference ``data/bboxes.py:291-343``), in one
    launch (``lpb_frames_crop_normalize``).

    ``frames``: (seq, 3, H, W) fp32 on the device, already normalised; ``bbox_rows``: DataFrame with columns
    ``x, y, h, w``, or a (rows, 4) tensor, with at least ``seq`` rows (row i crops frame i).  Returns (frames
    (seq, 3, h, w), the boxes actually used (seq, 4) [x1, y1, y2 - y1, x2 - x1], clamped to the frame).  Boxes the
    reference rejects (origin past the far edge, NaN) give a one-pixel crop and the whole frame (DESIGN.md §2).
    """
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda:
        raise RuntimeError("lpb200: `frames` must be a CUDA tensor (this package has no CPU fallback)")
    if isinstance(bbox_rows, torch.Tensor):
        rows = bbox_rows.to(device=frames.device, dtype=torch.float32)
    else:
        rows = torch.as_tensor(bbox_rows[["x", "y", "h", "w"]].to_numpy(dtype=np.float64, copy=True), dtype=torch.float32, device=frames.device)
    if rows.dim() != 2 or rows.shape[0] < frames.shape[0]:
        raise ValueError(f"need one bbox row per frame: {frames.shape[0]} frames, bbox rows {tuple(rows.shape)}")
    return ops.frames_crop_normalize(frames.float(), rows, resize_dims)


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
