"""numpy restatement of OpenCV 4.x ``cv2.resize(..., interpolation=INTER_LINEAR)`` on uint8 HWC images (the fixed-point
path of imgproc/src/resize.cpp with its vectorised vertical pass), and the fp32 normalisation of the reference's
``Model.predict_frame`` (lightning_pose/api/model.py:423-430).  It is what ``lpb_frames_crop_resize_cv2`` computes.

Per output axis, with ``scale = 1.0 / ((double)dst / src)``:

    f  = (float)((d + 0.5) * scale - 0.5)         computed in double, then rounded to float
    s  = floor(f);  f -= s
    s0 = clamp(s, 0, src - 1);  s1 = clamp(s + 1, 0, src - 1)
    a1 = rint(f * 2048);  a0 = rint((1 - f) * 2048)

then, per channel, ``S(y, x) = a0[x] img[y, x0] + a1[x] img[y, x1]`` (int32) and
``out = clamp((((b0 (S(y0) >> 4)) >> 16) + ((b1 (S(y1) >> 4)) >> 16) + 2) >> 2, 0, 255)``.

The ``wrong`` switches give the rules a careless port would use; each must change at least one byte on the test shapes:
``double_f`` keeps f in double, ``zero_vertical`` zeroes the vertical weights where a row index is clamped (OpenCV's
horizontal rule), ``no_preshift`` drops the ``>> 4``, ``scalar`` uses the scalar tail ``(b0 S0 + b1 S1 + 2^21) >> 22``.
"""
from __future__ import annotations

import numpy as np

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
WRONG_RULES = ("double_f", "zero_vertical", "no_preshift", "scalar")


def axis_taps(src: int, dst: int, wrong: str | None = None, vertical: bool = False):
    """(i0, i1, w0, w1) int64 arrays of length dst: the two source indices and their 11-bit weights."""
    scale = 1.0 / (float(dst) / float(src))
    d = np.arange(dst, dtype=np.float64)
    fd = (d + 0.5) * scale - 0.5
    if wrong == "double_f":
        s = np.floor(fd)
        f = fd - s
        w1 = np.rint(f * 2048.0)
        w0 = np.rint((1.0 - f) * 2048.0)
    else:
        f = fd.astype(np.float32)
        s = np.floor(f)
        f = (f - s).astype(np.float32)
        w1 = np.rint(f * np.float32(2048.0))
        w0 = np.rint((np.float32(1.0) - f) * np.float32(2048.0))
    s = s.astype(np.int64)
    i0, i1 = np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1)
    w0, w1 = w0.astype(np.int64), w1.astype(np.int64)
    if vertical and wrong == "zero_vertical":
        lo, hi = s < 0, s + 1 >= src
        w0 = np.where(lo | hi, 2048, w0)
        w1 = np.where(lo | hi, 0, w1)
        i0 = np.where(hi, src - 1, i0)
    return i0, i1, w0, w1


def resize_linear_u8(img: np.ndarray, out_h: int, out_w: int, wrong: str | None = None) -> np.ndarray:
    """uint8 (H, W, C) -> uint8 (out_h, out_w, C), cv2.resize INTER_LINEAR."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3
    h, w, _ = img.shape
    x0, x1, a0, a1 = axis_taps(w, out_w, wrong)
    y0, y1, b0, b1 = axis_taps(h, out_h, wrong, vertical=True)
    src = img.astype(np.int64)
    rows = a0[None, :, None] * src[:, x0] + a1[None, :, None] * src[:, x1]  # S(y, x): (H, out_w, C)
    s0, s1 = rows[y0], rows[y1]
    bb0, bb1 = b0[:, None, None], b1[:, None, None]
    if wrong == "scalar":
        out = (bb0 * s0 + bb1 * s1 + (1 << 21)) >> 22
    elif wrong == "no_preshift":
        out = (((bb0 * s0) >> 20) + ((bb1 * s1) >> 20) + 2) >> 2
    else:
        out = (((bb0 * (s0 >> 4)) >> 16) + ((bb1 * (s1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def normalize(u8: np.ndarray, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> np.ndarray:
    """uint8 (..., 3) -> fp32 ``(u8 / 255 - mean) / std`` as numpy evaluates it in the reference (HWC kept)."""
    t = u8.astype(np.float32) / np.float32(255.0)
    return (t - np.asarray(mean, dtype=np.float32)) / np.asarray(std, dtype=np.float32)


def crop(frame: np.ndarray, box) -> tuple[np.ndarray, list[int]]:
    """numpy-slice crop of the reference: (x, y, w, h) -> (crop, [x, y, actual_h, actual_w]); None is the whole frame."""
    if box is None:
        return frame, [0, 0, frame.shape[-3], frame.shape[-2]]
    x, y, w, h = (int(v) for v in box)
    c = frame[..., y : y + h, x : x + w, :]
    return c, [x, y, c.shape[-3], c.shape[-2]]


def crop_resize_normalize(frames: np.ndarray, box, out_h: int, out_w: int, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """uint8 (F, H, W, 3) -> (uint8 (F, out_h, out_w, 3), fp32 (F, 3, out_h, out_w), bbox row [x, y, h, w])."""
    c, row = crop(frames, box)
    u8 = np.stack([resize_linear_u8(f, out_h, out_w) for f in c])
    return u8, np.ascontiguousarray(normalize(u8, mean, std).transpose(0, 3, 1, 2)), row
