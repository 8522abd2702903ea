"""Golden generator for crop-zoom inference.  TEST INFRASTRUCTURE ONLY.

``python tests/cropzoom_oracle.py`` writes ``tests/golden/cropzoom.npz`` by running the reference's own, unmodified code:
``crop_and_resize_frames`` (``lightning_pose/data/bboxes.py:291-343``, loaded through ``oracle/ref_loader.py``) and
``_compute_bbox_df`` / ``smooth_bbox`` (``lightning_pose/utils/cropzoom.py``), loaded with placeholder modules for
``moviepy``, ``tqdm`` and ``lightning_pose.utils.io``, which those two functions do not use.  ``smooth_bbox`` runs on
temporary CSV files, as in the reference.  Inputs are stored next to the outputs; every input is fp32-representable.
Needs the full reference tree; the GPU tests only read the committed npz.  Nothing under ``lightning_pose_b200/``
imports this module.

Cases
  crop_<name>:  uint8 frames (F, H, W, 3), their normalised fp32 form (F, 3, H, W) ((u8 / 255 - mean) / std, the
                DALI pipeline's normalisation), bbox rows (F, 4) x y h w, output size; the reference's cropped frames
                (from the fp32 form) and clamped boxes.
  bbox_<name>:  a prediction table (N, 3K) (x, y, likelihood per keypoint, a PredictionHandler's column order), anchor
                indices (empty: all), crop_ratio or (crop_height, crop_width); the reference's boxes.
  smooth_<name>: integer boxes (N, 4) and a window; the reference's smoothed boxes.
"""
from __future__ import annotations

import importlib
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "cropzoom.npz")
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def normalise(u8: torch.Tensor) -> torch.Tensor:
    """uint8 (F, H, W, 3) -> fp32 (F, 3, H, W), (x / 255 - mean) / std."""
    x = u8.permute(0, 3, 1, 2).float() / 255.0
    return (x - torch.tensor(MEAN)[:, None, None]) / torch.tensor(STD)[:, None, None]


# (name, frames (F, H, W), rows, (out_h, out_w)); F = len(rows)
CROP_CASES = [
    # the reference's own known answers (tests/data/test_bboxes.py:636-700): 50 x 50 frames
    ("known", (50, 50), [[10, 10, 20, 20], [-5, -5, 20, 20], [40, 40, 30, 30]], (32, 32)),
    # in bounds, negative origins, past the far edges, one pixel, the whole frame, fractional values (truncated)
    ("mixed_square", (32, 40), [[10, 5, 20, 30], [-5, -7, 20, 25], [35, 28, 30, 30], [3, 4, 1, 1], [0, 0, 32, 40],
                                [20, 10, 5, 7], [10.75, 5.5, 20.25, 30.5], [-3.75, -0.5, 12.5, 9.75]], (32, 32)),
    ("mixed_odd", (32, 40), [[10, 5, 20, 30], [-5, -7, 20, 25], [35, 28, 30, 30], [3, 4, 1, 1], [0, 0, 32, 40],
                             [39, 31, 9, 9]], (17, 23)),
    ("upscale", (40, 36), [[4, 6, 9, 7], [30, 30, 20, 20], [0, 0, 2, 3], [-2, 5, 11, 13]], (64, 56)),
    ("downscale", (72, 60), [[0, 0, 72, 60], [7, 11, 50, 40], [-20, -10, 60, 50], [40, 30, 200, 200]], (20, 18)),
]

# (name, anchors (names; empty = all), kwargs)
BBOX_CASES = [
    ("ratio_all", [], {"crop_ratio": 1.0}),
    ("ratio_subset", ["kp4", "kp1", "kp2"], {"crop_ratio": 1.35}),
    ("fixed_hw", [], {"crop_height": 101, "crop_width": 64}),
    ("fixed_subset", ["kp0", "kp3"], {"crop_height": 80, "crop_width": 80}),
    ("fixed_tall", ["kp2", "kp5"], {"crop_height": 30, "crop_width": 121}),
]
N_KP = 6

# (name, n frames, window)
SMOOTH_CASES = [("w1", 23, 1), ("w4", 23, 4), ("w5", 23, 5), ("w7", 23, 7), ("short_w5", 3, 5), ("short_w7", 4, 7)]


def _predictions(n: int, seed: int) -> np.ndarray:
    """(n, 3K) prediction table: keypoints around a drifting centre, some near the frame's origin (negative top-left
    corners), fp32-representable."""
    g = np.random.default_rng(seed)
    centre = np.cumsum(g.normal(0, 6, size=(n, 2)), axis=0) + np.array([120.0, 90.0])
    centre[: n // 4] = g.uniform(2, 15, size=(n // 4, 2))
    kp = centre[:, None, :] + g.normal(0, 18, size=(n, N_KP, 2))
    tab = np.zeros((n, 3 * N_KP), np.float32)
    tab[:, 0::3], tab[:, 1::3], tab[:, 2::3] = kp[..., 0], kp[..., 1], g.uniform(0, 1, size=(n, N_KP))
    return tab


def load_reference():
    """(reference data/bboxes.py, reference utils/cropzoom.py), loaded unmodified."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    R.install()
    for name in ("moviepy", "tqdm"):
        mod = types.ModuleType(name)
        mod.VideoFileClip = type("VideoFileClip", (), {})
        sys.modules[name] = mod
    io = types.ModuleType("lightning_pose.utils.io")
    sys.modules["lightning_pose.utils.io"] = io
    sys.modules["lightning_pose.utils"].io = io  # type: ignore[attr-defined]
    return importlib.import_module("lightning_pose.data.bboxes"), importlib.import_module("lightning_pose.utils.cropzoom")


def reference_tree_available() -> bool:
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return os.path.isfile(os.path.join(R.REF_ROOT, "lightning_pose", "utils", "cropzoom.py"))


def gen_crop(db) -> dict:
    import pandas as pd

    g = {}
    for i, (name, (h, w), rows, size) in enumerate(CROP_CASES):
        gen = torch.Generator().manual_seed(100 + i)
        u8 = torch.randint(0, 256, (len(rows), h, w, 3), dtype=torch.uint8, generator=gen)
        f32 = normalise(u8)
        rows_np = np.asarray(rows, np.float32)
        df = pd.DataFrame(rows_np.astype(np.float64), columns=["x", "y", "h", "w"])
        out, boxes = db.crop_and_resize_frames(f32, df, list(size))
        g[f"crop_{name}_in_u8"], g[f"crop_{name}_in_f32"] = u8.numpy(), f32.numpy()
        g[f"crop_{name}_in_rows"], g[f"crop_{name}_in_size"] = rows_np, np.asarray(size, np.int64)
        g[f"crop_{name}_out_frames"], g[f"crop_{name}_out_boxes"] = out.numpy(), boxes.numpy()
    return g


def _pred_df(tab: np.ndarray):
    import pandas as pd

    names = [f"kp{k}" for k in range(N_KP)]
    cols = pd.MultiIndex.from_product([["heatmap_tracker"], names, ["x", "y", "likelihood"]], names=["scorer", "bodyparts", "coords"])
    return pd.DataFrame(tab.astype(np.float64), columns=cols), names


def gen_bbox(cz) -> dict:
    g = {}
    for i, (name, anchors, kw) in enumerate(BBOX_CASES):
        tab = _predictions(37, 200 + i)
        df, names = _pred_df(tab)
        out = cz._compute_bbox_df(df, list(anchors), **kw)
        g[f"bbox_{name}_in_table"] = tab
        g[f"bbox_{name}_in_anchors"] = np.asarray([names.index(a) for a in anchors], np.int32)
        g[f"bbox_{name}_in_ratio"] = np.asarray(kw.get("crop_ratio", 0.0), np.float64)
        g[f"bbox_{name}_in_hw"] = np.asarray([kw.get("crop_height", 0), kw.get("crop_width", 0)], np.int64)
        g[f"bbox_{name}_out"] = out[["x", "y", "h", "w"]].to_numpy().astype(np.int64)
    return g


def gen_smooth(cz, db_boxes: np.ndarray) -> dict:
    import pandas as pd

    g = {}
    for i, (name, n, window) in enumerate(SMOOTH_CASES):
        rng = np.random.default_rng(300 + i)
        base = db_boxes[np.arange(n) % len(db_boxes)]
        boxes = (base + rng.integers(-6, 7, size=base.shape) * (rng.uniform(size=base.shape) < 0.5)).astype(np.int64)
        with tempfile.TemporaryDirectory() as tmp:
            src, dst = Path(tmp) / "in", Path(tmp) / "out"
            src.mkdir()
            pd.DataFrame(boxes, columns=["x", "y", "h", "w"]).to_csv(src / "vid_bbox.csv")
            cz.smooth_bbox(src, dst, method="median", window=window)
            out = pd.read_csv(dst / "vid_bbox.csv", index_col=0)[["x", "y", "h", "w"]].to_numpy().astype(np.int64)
        g[f"smooth_{name}_in_boxes"], g[f"smooth_{name}_in_window"] = boxes, np.asarray(window, np.int64)
        g[f"smooth_{name}_out"] = out
    return g


def main(path: str = GOLDEN_PATH) -> None:
    assert reference_tree_available(), "needs the full reference tree (lightning_pose/utils/cropzoom.py)"
    db, cz = load_reference()
    with torch.no_grad():
        arrays = gen_crop(db)
    arrays.update(gen_bbox(cz))
    arrays.update(gen_smooth(cz, arrays["bbox_ratio_all_out"]))
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(arrays)} arrays, {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main(*sys.argv[1:])
