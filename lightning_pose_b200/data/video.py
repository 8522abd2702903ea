"""Video-ingest boundary: decoded frames -> ``UnlabeledBatchDict`` (SURVEY 8f-4).

Mirror of what ``LitDaliWrapper._dali_output_to_tensors`` hands the trackers
(``lightning_pose/data/video/dali.py:265-327``): ``frames`` (seq, 3, H, W) normalised with the ImageNet statistics,
``transforms`` (a lone ``[-1]`` when no geometric augmentation ran, :175-178), ``bbox`` = ``[0, 0, height, width]`` of the
ORIGINAL frame repeated per frame, ``is_multiview``.  Video decoding itself (NVDEC / DALI readers, :133-156) is host/driver
I/O and out of scope: the entry point takes decoded uint8 RGB surfaces already on the device and fuses resize + /255 +
normalise + layout change into one kernel (``csrc/ingest.cu``).
"""
from __future__ import annotations

from typing import Sequence

import torch

from lightning_pose_b200 import ops

__all__ = ["frames_to_unlabeled_batch", "context_windows_step"]


AUGMENTED_IMGAUG = ("dlc", "dlc-top-down")  # training.imgaug values whose unlabeled frames are augmented (dali.py:156)


def frames_to_unlabeled_batch(frames_u8: torch.Tensor | Sequence[torch.Tensor], resize_dims: Sequence[int] | None = None,
                              dtype: torch.dtype = torch.float32, channels_last: bool = False, bbox: torch.Tensor | None = None,
                              bbox_row0: int = 0, imgaug: str | None = "default", generator: torch.Generator | None = None) -> dict:
    """uint8 (seq, H, W, 3) frames of one view - or a list of them, one per view - to the batch dict of the trackers.

    Single view -> ``UnlabeledBatchDict``; several views -> ``MultiviewUnlabeledBatchDict`` with frames
    (seq, views, 3, H, W), transforms (views, 1), bbox (seq, 4 * views) (reference :289-327).

    Crop-zoom pose models (reference ``LitDaliWrapper._apply_bbox_crop``, :332-380): ``bbox`` is the video's (N, 4)
    [x, y, h, w] device table and frame i is cropped to row ``min(bbox_row0 + i, N - 1)``, resized to ``resize_dims``
    (required) and normalised, in one launch; the returned ``bbox`` holds the clamped boxes the remap needs.  Single
    view only, as in the reference.

    Augmentation (``imgaug`` "dlc" or "dlc-top-down", the reference's ``training.imgaug`` values that augment the
    unlabeled branch, dali.py:156-178): each view draws its own rotation, scale, brightness, contrast and shot-noise
    factor (``ops.draw_dlc_params``: one draw per call, shared by the call's frames) and is resized, warped, changed
    and normalised in one launch (``ops.frames_augment_normalize``).  ``transforms`` is then the warp's source ->
    destination matrix, (2, 3) for one view and (V, 1, 2, 3) for V views, which the trackers undo on their predictions.
    ``resize_dims`` is required, and crop mode (``bbox``) is not augmented, as in the reference.  ``generator`` is the
    torch generator the draw uses (default: the device's default generator, which a captured CUDA graph replays with
    fresh draws); for per-rank streams under DDP seed one per rank, as the reference does with ``seed + device_id``.
    Every other ``imgaug`` value, ``None`` included, leaves the frames unaugmented.
    """
    views = [frames_u8] if isinstance(frames_u8, torch.Tensor) else list(frames_u8)
    if imgaug in AUGMENTED_IMGAUG:
        if bbox is not None:
            raise ValueError("unlabeled augmentation is not supported with bounding-box crops (crop mode is prediction-only)")
        if resize_dims is None:
            raise ValueError(f"resize_dims is required with imgaug={imgaug!r}")
        return _augmented_batch(views, resize_dims, dtype, channels_last, generator)
    if bbox is not None:
        if len(views) > 1:
            raise ValueError("bbox_file is not supported for multiview prediction")
        if resize_dims is None:
            raise ValueError("resize_dims is required when frames are cropped to bounding boxes")
        frames, boxes = ops.frames_crop_normalize(views[0], bbox, resize_dims, row0=bbox_row0, channels_last=channels_last, dtype=dtype)
        return {"frames": frames, "transforms": torch.tensor([-1.0], device=frames.device), "bbox": boxes, "is_multiview": False}
    boxes = torch.tensor([[0.0, 0.0, float(v.shape[1]), float(v.shape[2])] for v in views], device=views[0].device).reshape(1, -1)
    seq = views[0].shape[0]
    if len(views) == 1:
        frames = ops.frames_normalize(views[0], size=resize_dims, channels_last=channels_last, dtype=dtype)
        return {"frames": frames, "transforms": torch.tensor([-1.0], device=frames.device), "bbox": boxes.repeat(seq, 1), "is_multiview": False}
    if resize_dims is None:  # each view at its own size: they can only be stacked when the sizes agree
        if len({tuple(v.shape[1:3]) for v in views}) > 1:
            raise ValueError("views of different sizes need resize_dims to be stacked")
        resize_dims = tuple(views[0].shape[1:3])
    return {
        "frames": ops.frames_normalize_views(views, resize_dims, channels_last=channels_last, dtype=dtype),
        "transforms": torch.full((len(views), 1), -1.0, device=views[0].device),
        "bbox": boxes.repeat(seq, 1),
        "is_multiview": True,
    }


def _augmented_batch(views, resize_dims, dtype, channels_last, generator) -> dict:
    dev = views[0].device
    params, seeds = ops.draw_dlc_params(len(views), dev, generator=generator)
    transforms = torch.empty((len(views), 1, 2, 3), device=dev, dtype=torch.float32)
    bbox = torch.zeros((views[0].shape[0], 4 * len(views)), device=dev)  # filled in place: no host copy, capturable
    outs = []
    for i, v in enumerate(views):
        frames, _ = ops.frames_augment_normalize(v, resize_dims, params[i], seeds[i : i + 1], channels_last=channels_last,
                                                 dtype=dtype, transform_out=transforms[i, 0])
        outs.append(frames)
        bbox[:, 4 * i + 2].fill_(float(v.shape[1]))
        bbox[:, 4 * i + 3].fill_(float(v.shape[2]))
    if len(views) == 1:
        return {"frames": outs[0], "transforms": transforms[0, 0], "bbox": bbox, "is_multiview": False}
    return {"frames": torch.stack(outs, dim=1), "transforms": transforms, "bbox": bbox, "is_multiview": True}


def context_windows_step(sequence_length: int) -> int:
    """Reader step of context (MHCRNN) prediction: consecutive sequences overlap by 4 frames (dali.py:214-216)."""
    return int(sequence_length) - 4
