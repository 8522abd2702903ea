"""float64 CPU restatement of the unlabeled-video augmentation (reference ``lightning_pose/data/video/dali.py:154-192``,
``training.imgaug`` "dlc").  TEST INFRASTRUCTURE ONLY: nothing under ``lightning_pose_b200/`` imports this module.

Steps, per view and per draw (``include/lpb200.h``, ``lpb_frames_augment_normalize``):
  1. resize uint8 (F, H, W, 3) to (h, w): bilinear, half-pixel centres, no antialiasing (the plain ingest's resize);
  2. params = angle (degrees), sx, sy, brightness, contrast, factor;
  3. M = S_c R_c in (x, y), c = (h / 2, w / 2) taken as (x, y);
  4. warp: destination (x, y) samples the resized image bilinearly at M^-1 (x + 0.5, y + 0.5) - 0.5, zero outside;
  5. brightness * (0.5 + contrast * (v - 0.5));
  6. shot noise Poisson(max(0, v / factor)) * factor (numpy's generator here: the kernel's stream differs);
  7. / 255 and ImageNet normalisation, FCHW.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])


def resize(u8: np.ndarray, size) -> np.ndarray:
    """uint8 (F, H, W, 3) -> float64 (F, h, w, 3) in 0..255: bilinear, half-pixel centres, edge-clamped taps."""
    f, H, W, _ = u8.shape
    h, w = int(size[0]), int(size[1])
    x = u8.astype(np.float64)

    def axis(n_out, n_in):
        s = np.maximum((np.arange(n_out) + 0.5) * (n_in / n_out) - 0.5, 0.0)
        i0 = np.minimum(np.floor(s).astype(np.int64), n_in - 1)
        return i0, np.minimum(i0 + 1, n_in - 1), s - i0

    y0, y1, wy = axis(h, H)
    x0, x1, wx = axis(w, W)
    wx = wx[None, None, :, None]
    top = x[:, y0][:, :, x0] * (1 - wx) + x[:, y0][:, :, x1] * wx
    bot = x[:, y1][:, :, x0] * (1 - wx) + x[:, y1][:, :, x1] * wx
    wy = wy[None, :, None, None]
    return top * (1 - wy) + bot * wy


def dlc_matrix(params, size) -> np.ndarray:
    """(2, 3) source -> destination M = S_c R_c of fn.transforms.rotation(angle, center=c) followed by
    fn.transforms.scale(scale, center=c), in (x, y), with c = (h / 2, w / 2) as the reference passes it."""
    angle, sx, sy = float(params[0]), float(params[1]), float(params[2])
    cx, cy = size[0] / 2.0, size[1] / 2.0
    th = np.deg2rad(angle)

    def about_centre(lin):
        t = np.eye(3)
        t[:2, 2] = (cx, cy)
        m = np.eye(3)
        m[:2, :2] = lin
        back = np.eye(3)
        back[:2, 2] = (-cx, -cy)
        return t @ m @ back

    r = about_centre(np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]))
    s = about_centre(np.diag([sx, sy]))
    return (s @ r)[:2]


def invert(m: np.ndarray) -> np.ndarray:
    a_inv = np.linalg.inv(m[:, :2])
    return np.concatenate([a_inv, -a_inv @ m[:, 2:]], axis=1)


def warp(img: np.ndarray, m: np.ndarray) -> np.ndarray:
    """float64 (F, h, w, 3) warped by source -> destination M, output size = input size, zero fill."""
    f, h, w, _ = img.shape
    mi = invert(m)
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    u = mi[0, 0] * (xx + 0.5) + mi[0, 1] * (yy + 0.5) + mi[0, 2] - 0.5
    v = mi[1, 0] * (xx + 0.5) + mi[1, 1] * (yy + 0.5) + mi[1, 2] - 0.5
    x0, y0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    fx, fy = (u - x0)[None, :, :, None], (v - y0)[None, :, :, None]
    out = np.zeros_like(img)
    for dy in (0, 1):
        for dx in (0, 1):
            tx, ty = x0 + dx, y0 + dy
            ok = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
            tap = img[:, np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)] * ok[None, :, :, None]
            out += tap * (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
    return out


def brightness_contrast(x: np.ndarray, brightness: float, contrast: float) -> np.ndarray:
    return brightness * (0.5 + contrast * (x - 0.5))


def shot_noise(x: np.ndarray, factor: float, rng: np.random.Generator) -> np.ndarray:
    if factor == 0:
        return x
    return rng.poisson(np.maximum(0.0, x / factor)) * factor


def normalise(x: np.ndarray) -> np.ndarray:
    """float64 (F, h, w, 3) in 0..255 -> (F, 3, h, w), (x / 255 - mean) / std."""
    return ((x / 255.0 - MEAN) / STD).transpose(0, 3, 1, 2)


def augment(u8: np.ndarray, size, params, rng: np.random.Generator | None = None):
    """Steps 1 to 7: (frames (F, 3, h, w) float64, M (2, 3))."""
    m = dlc_matrix(params, size)
    x = warp(resize(u8, size), m)
    x = brightness_contrast(x, float(params[3]), float(params[4]))
    x = shot_noise(x, float(params[5]), rng or np.random.default_rng(0))
    return normalise(x), m


def undo_then_model_to_frame(kp: np.ndarray, m: np.ndarray, bbox: np.ndarray, model_h: int, model_w: int) -> np.ndarray:
    """float64 (n, K, 2) augmented model coordinates -> frame coordinates: the reference's undo_affine_transform
    (M^-1 applied to the raw coordinates, no half-pixel shift) then model_to_frame (x / w * bbox_w + bbox_x, likewise y)
    with bbox (n, 4) [x, y, h, w]."""
    mi = invert(m)
    p = kp @ mi[:, :2].T + mi[:, 2]
    x = p[..., 0] / model_w * bbox[:, None, 3] + bbox[:, None, 0]
    y = p[..., 1] / model_h * bbox[:, None, 2] + bbox[:, None, 1]
    return np.stack([x, y], axis=-1)


def reference_tree_available() -> bool:
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return os.path.isfile(os.path.join(R.REF_ROOT, "lightning_pose", "data", "utils.py"))


def load_reference_utils():
    """The reference's ``lightning_pose/data/utils.py``, unmodified (``undo_affine_transform`` and its batch form)."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return R.load("lightning_pose.data.utils")
