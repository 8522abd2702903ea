"""Write tests/golden/frame_resize.npz: the single-frame ingest's cases computed by OpenCV itself.

    python scripts/gen_frame_resize_golden.py        (needs cv2; the GPU tests then need neither cv2 nor this script)

Each case is the reference's ``Model.predict_frame`` preprocessing (lightning_pose/api/model.py:388-430) on seeded
uint8 frames: the numpy-slice crop ``frame[y:y+h, x:x+w]``, ``cv2.resize(INTER_LINEAR)``, then ``(u8 / 255 - mean) / std``
in fp32 numpy.  Stored per case: ``<name>_frames`` (F, H, W, 3) uint8, ``<name>_box`` [x, y, w, h] int32 (all -1: no box),
``<name>_u8`` (F, h, w, 3) the cv2 output, ``<name>_f32`` (F, 3, h, w) the normalised fp32 images, ``<name>_bbox``
[x, y, actual_h, actual_w].  The script also asserts that tests/frame_resize_oracle.py reproduces every byte.
"""
from __future__ import annotations

import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import frame_resize_oracle as O  # noqa: E402

# name: (frames (F, H, W), box [x, y, w, h] or None, out (h, w))
CASES = {
    "whole_down": ((1, 90, 130), None, (64, 56)),
    "interior_up": ((1, 90, 130), (17, 9, 41, 33), (100, 72)),
    "clipped_right_bottom": ((1, 90, 130), (100, 70, 80, 50), (48, 40)),
    "one_pixel": ((1, 90, 130), (5, 7, 1, 1), (16, 24)),
    "one_row": ((1, 90, 130), (3, 60, 77, 1), (20, 36)),
    "context5": ((5, 40, 60), (3, 4, 50, 30), (32, 48)),
    "exact_2x": ((1, 64, 96), None, (32, 48)),
    "identity": ((1, 37, 53), None, (37, 53)),
}


def main() -> None:
    rng = np.random.default_rng(20261017)
    mean = np.array(O.IMAGENET_MEAN, dtype=np.float32)
    std = np.array(O.IMAGENET_STD, dtype=np.float32)
    out = {}
    for name, ((f, h, w), box, (oh, ow)) in CASES.items():
        frames = rng.integers(0, 256, (f, h, w, 3), dtype=np.uint8)
        crop, row = O.crop(frames, box)
        u8 = np.stack([cv2.resize(c, (ow, oh), interpolation=cv2.INTER_LINEAR) for c in crop])
        f32 = ((u8.astype(np.float32) / 255.0 - mean) / std).transpose(0, 3, 1, 2)
        ref_u8, ref_f32, ref_row = O.crop_resize_normalize(frames, box, oh, ow)
        assert np.array_equal(ref_u8, u8) and np.array_equal(ref_f32.view(np.uint32), np.ascontiguousarray(f32).view(np.uint32)), name
        assert ref_row == row, name
        out[f"{name}_frames"] = frames
        out[f"{name}_box"] = np.array(box if box is not None else (-1, -1, -1, -1), dtype=np.int32)
        out[f"{name}_u8"] = u8
        out[f"{name}_f32"] = np.ascontiguousarray(f32)
        out[f"{name}_bbox"] = np.array(row, dtype=np.float32)
        print(f"{name:22s} frames {frames.shape} box {box} -> {u8.shape}  bbox {row}")
    path = os.path.join(ROOT, "tests", "golden", "frame_resize.npz")
    np.savez_compressed(path, cv2_version=np.array(cv2.__version__), **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
