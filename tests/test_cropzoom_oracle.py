"""CPU: tests/golden/cropzoom.npz against the reference's known answers, plain restatements of the box, smoothing and
crop-clamp rules (the arithmetic the kernels in csrc/cropzoom.cu implement) against the goldens, the new ABI entries'
argument checks and the Python surface without a GPU."""
import ast
import ctypes
import filecmp
import inspect
import math
import os

import numpy as np
import pandas as pd
import pytest
import torch

import cropzoom_oracle as O
from oracle import ref_loader as R

BBOX = [c[0] for c in O.BBOX_CASES]
SMOOTH = [c[0] for c in O.SMOOTH_CASES]
CROP = [c[0] for c in O.CROP_CASES]


# ---- restatements of the kernels' rules ---------------------------------------------------------------------------
def boxes_rule(table, anchors, ratio, hw):
    """bboxes_kernel: fp64, centroid summed in keypoint order, h subtracted from x and w from y."""
    k = table.shape[1] // 3
    idx = list(anchors) if len(anchors) else list(range(k))
    out = []
    for row in table.astype(np.float64):
        xs, ys = [row[3 * i] for i in idx], [row[3 * i + 1] for i in idx]
        if ratio > 0:
            s = int(math.ceil(max(max(xs) - min(xs), max(ys) - min(ys)) * ratio))
            h = w = s + s % 2
        else:
            h, w = int(hw[0]) + int(hw[0]) % 2, int(hw[1]) + int(hw[1]) % 2
        sx = sy = 0.0
        for x, y in zip(xs, ys):
            sx, sy = sx + x, sy + y
        out.append([int(sx / len(idx) - h // 2), int(sy / len(idx) - w // 2), h, w])
    return np.asarray(out, np.int64)


def median_rule(boxes, window):
    """rolling_median_kernel: window [i + 1 + (w - 1) // 2 - w, i + 1 + (w - 1) // 2) clipped, NaN skipped, round half
    to even."""
    n = boxes.shape[0]
    out = np.full(boxes.shape, np.nan)
    for i in range(n):
        end = min(n, i + 1 + (window - 1) // 2)
        lo = max(0, i + 1 + (window - 1) // 2 - window)
        for c in range(4):
            v = sorted(x for x in boxes[lo:end, c].astype(np.float64) if not np.isnan(x))
            if v:
                m = v[len(v) // 2] if len(v) % 2 else (v[len(v) // 2 - 1] + v[len(v) // 2]) / 2.0
                out[i, c] = np.rint(m)
    return out


def clamp_rule(row, h, w):
    """crop_box: the reference's clamp, plus the two divergences (origin past the far edge, NaN / inf rows)."""
    if not all(math.isfinite(v) for v in row):
        return [0, 0, h, w]
    xi, yi = int(row[0]), int(row[1])
    x1, y1 = min(max(0, xi), w - 1), min(max(0, yi), h - 1)
    x2, y2 = max(x1 + 1, min(w, xi + int(row[3]))), max(y1 + 1, min(h, yi + int(row[2])))
    return [x1, y1, y2 - y1, x2 - x1]


# ---- goldens --------------------------------------------------------------------------------------------------------
def test_crop_golden_holds_the_reference_known_answers(golden):
    g = golden("cropzoom")
    # tests/data/test_bboxes.py:636-700
    assert g["crop_known_out_boxes"].tolist() == [[10, 10, 20, 20], [0, 0, 15, 15], [40, 40, 10, 10]]
    for name in CROP:
        f, h, w, _ = g[f"crop_{name}_in_u8"].shape
        assert g[f"crop_{name}_out_frames"].shape == (f, 3, *g[f"crop_{name}_in_size"])
        np.testing.assert_allclose(g[f"crop_{name}_in_f32"], O.normalise(torch.from_numpy(g[f"crop_{name}_in_u8"])).numpy(), rtol=0, atol=0)
        want = [clamp_rule(r, h, w) for r in g[f"crop_{name}_in_rows"].astype(np.float64)]
        assert g[f"crop_{name}_out_boxes"].tolist() == want, name


def test_crop_golden_covers_the_issue_cases(golden):
    g = golden("cropzoom")
    rows = np.concatenate([g[f"crop_{n}_in_rows"] for n in CROP])
    assert (rows[:, :2] < 0).any() and (rows[:, 2:] == 1).all(1).any() and (rows != np.trunc(rows)).any()
    sizes = {tuple(g[f"crop_{n}_in_size"]) for n in CROP}
    assert (17, 23) in sizes and any(a != b for a, b in sizes)
    past = [(r[0] + r[3] > g[f"crop_{n}_in_u8"].shape[2]) for n in CROP for r in g[f"crop_{n}_in_rows"]]
    assert any(past)
    up = g["crop_upscale_in_rows"][:, 2:] < g["crop_upscale_in_size"]
    assert up.all() and (g["crop_downscale_in_rows"][:2, 2:] > g["crop_downscale_in_size"]).all()


@pytest.mark.parametrize("name", BBOX)
def test_box_rule_matches_golden(golden, name):
    g = golden("cropzoom")
    out = g[f"bbox_{name}_out"]
    np.testing.assert_array_equal(boxes_rule(g[f"bbox_{name}_in_table"], g[f"bbox_{name}_in_anchors"], float(g[f"bbox_{name}_in_ratio"]),
                                             g[f"bbox_{name}_in_hw"]), out)
    assert (out[:, 2:] % 2 == 0).all()
    if float(g[f"bbox_{name}_in_ratio"]) == 0:  # tests/utils/test_cropzoom.py: fixed sizes are the requested (even) ones
        assert (out[:, 2:] == g[f"bbox_{name}_in_hw"] + g[f"bbox_{name}_in_hw"] % 2).all()
    else:
        assert (out[:, 2] == out[:, 3]).all()


def test_box_golden_pins_the_h_from_x_quirk(golden):
    """cropzoom.py:135 subtracts h // 2 from x and w // 2 from y; with h != w, the swapped form gives other boxes."""
    g = golden("cropzoom")
    tab, anchors, hw = g["bbox_fixed_tall_in_table"], g["bbox_fixed_tall_in_anchors"], g["bbox_fixed_tall_in_hw"]
    assert hw[0] != hw[1]
    swapped = boxes_rule(tab, anchors, 0.0, hw[::-1])[:, :2]
    assert not np.array_equal(swapped, g["bbox_fixed_tall_out"][:, :2])
    assert (g["bbox_ratio_all_out"][:, :2] < 0).any()  # negative top-left corners (truncation toward zero)
    assert list(g["bbox_ratio_subset_in_anchors"]) == [4, 1, 2]  # given out of keypoint order


@pytest.mark.parametrize("name", SMOOTH)
def test_median_rule_matches_golden(golden, name):
    g = golden("cropzoom")
    boxes, window = g[f"smooth_{name}_in_boxes"], int(g[f"smooth_{name}_in_window"])
    np.testing.assert_array_equal(median_rule(boxes, window), g[f"smooth_{name}_out"])
    if window == 1:
        np.testing.assert_array_equal(g[f"smooth_{name}_out"], boxes)


def test_median_rule_edges():
    b = np.array([[1, 0, 0, 0], [2, 0, 0, 0], [np.nan, 0, 0, 0], [4, 0, 0, 0], [np.nan] * 4, [np.nan] * 4, [np.nan] * 4], np.float64)
    want = pd.DataFrame(b).rolling(window=4, center=True, min_periods=1).median().round(0).to_numpy()
    np.testing.assert_array_equal(median_rule(b, 4), want)
    assert np.isnan(median_rule(b, 2)[5:, 0]).all()


# ---- goldens are reproducible -----------------------------------------------------------------------------------------
@pytest.mark.skipif(not O.reference_tree_available(), reason="needs the reference tree to regenerate the goldens")
def test_regenerating_cropzoom_golden_is_byte_identical(tmp_path):
    O.main(str(tmp_path / "cropzoom.npz"))
    assert filecmp.cmp(O.GOLDEN_PATH, str(tmp_path / "cropzoom.npz"), shallow=False)


# ---- ABI, no GPU --------------------------------------------------------------------------------------------------------
def test_cropzoom_entry_points_validate_without_gpu():
    from lightning_pose_b200 import _lib

    L, p = _lib.lib, ctypes.c_void_p(16)
    m3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    crop = lambda **kw: L.lpb_frames_crop_normalize(*[kw.get(k, v) for k, v in (
        ("frames", p), ("in_f32", 0), ("F", 2), ("H", 8), ("W", 8), ("boxes", p), ("n_boxes", 2), ("cursor", None), ("row0", 0),
        ("oh", 4), ("ow", 4), ("mean", m3), ("std", m3), ("layout", 0), ("bf16", 0), ("out", p), ("boxes_out", p), ("stream", None))])
    for kw in ({"frames": None}, {"boxes": None}, {"out": None}, {"boxes_out": None}, {"mean": None}):
        assert crop(**kw) == -1 and b"null pointer" in L.lpb_last_error(), kw
    for kw in ({"n_boxes": 0}, {"F": -1}, {"F": 65536}, {"H": 0}, {"oh": 0}, {"layout": 2}, {"row0": -1}):
        assert crop(**kw) == -1 and b"bad shape" in L.lpb_last_error(), kw
    assert crop(std=(ctypes.c_float * 3)(0.5, 0.0, 0.5)) == -1 and b"std" in L.lpb_last_error()
    assert crop(F=0) == 0 and crop(F=0, in_f32=1, mean=None, std=None) == 0  # nothing to do: no launch

    anchors = (ctypes.c_int32 * 2)(0, 1)
    box = lambda **kw: L.lpb_bboxes_from_keypoints(*[kw.get(k, v) for k, v in (
        ("kp", p), ("n", 3), ("K", 4), ("row_stride", 12), ("point_stride", 3), ("anchors", anchors), ("n_anchors", 2),
        ("ratio", 1.5), ("ch", 0), ("cw", 0), ("out", p), ("stream", None))])
    for kw in ({"kp": None}, {"out": None}, {"anchors": None}):
        assert box(**kw) == -1 and b"null pointer" in L.lpb_last_error(), kw
    assert box(K=0, n_anchors=0) == -1 and b"bad shape" in L.lpb_last_error()  # "all keypoints" of none
    for kw in ({"point_stride": 1}, {"row_stride": 11}, {"n_anchors": 257}, {"n": -1}):
        assert box(**kw) == -1 and b"bad shape" in L.lpb_last_error(), kw
    for kw in ({"ch": 10, "cw": 10}, {"ratio": 0.0}, {"ratio": 0.0, "ch": 10}, {"ratio": float("nan")}, {"ratio": -1.0}):
        assert box(**kw) == -1 and b"not both" in L.lpb_last_error(), kw
    assert box(anchors=(ctypes.c_int32 * 2)(0, 4)) == -1 and b"anchor index" in L.lpb_last_error()
    assert box(n=0) == 0 and box(n=0, ratio=0.0, ch=7, cw=9, n_anchors=0) == 0

    assert L.lpb_bboxes_rolling_median(None, 3, 5, p, None) == -1 and b"null pointer" in L.lpb_last_error()
    assert L.lpb_bboxes_rolling_median(p, 3, 5, p, None) == -1 and b"alias" in L.lpb_last_error()
    assert L.lpb_bboxes_rolling_median(p, 3, 0, ctypes.c_void_p(32), None) == -1 and b"bad shape" in L.lpb_last_error()
    assert L.lpb_bboxes_rolling_median(p, 0, 5, ctypes.c_void_p(32), None) == 0


# ---- Python surface, no GPU ----------------------------------------------------------------------------------------------
def test_cropzoom_surface_refuses_cpu_tensors():
    from lightning_pose_b200.data.bboxes import crop_and_resize_frames
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch
    from lightning_pose_b200.utils.cropzoom import compute_bboxes, smooth_bboxes

    rows = pd.DataFrame({"x": [0], "y": [0], "h": [4], "w": [4]})
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crop_and_resize_frames(torch.rand(1, 3, 8, 8), rows, [4, 4])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        frames_to_unlabeled_batch(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), resize_dims=(4, 4), bbox=torch.ones(1, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        compute_bboxes(torch.rand(2, 3, 2), crop_ratio=1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        smooth_bboxes(torch.rand(5, 4))


def test_cropzoom_surface_raises_like_the_reference():
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch
    from lightning_pose_b200.utils.cropzoom import anchor_indices, compute_bboxes, smooth_bboxes

    kp = torch.rand(2, 3, 2)
    with pytest.raises(ValueError, match="not both"):  # tests/utils/test_cropzoom.py:95-104
        compute_bboxes(kp, crop_ratio=2.0, crop_height=100, crop_width=100)
    with pytest.raises(ValueError, match="must be provided"):
        compute_bboxes(kp)
    with pytest.raises(ValueError, match="must be provided"):
        compute_bboxes(kp, crop_height=100)
    with pytest.raises(ValueError, match="unsupported method 'foo'"):
        smooth_bboxes(torch.rand(5, 4), method="foo")
    u8 = torch.zeros(2, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="not supported for multiview"):  # utils/predictions.py:461-462
        frames_to_unlabeled_batch([u8, u8], resize_dims=(4, 4), bbox=torch.ones(2, 4))
    with pytest.raises(ValueError, match="resize_dims"):
        frames_to_unlabeled_batch(u8, bbox=torch.ones(2, 4))
    names = ["nose", "ear_l", "ear_r", "tail"]
    assert anchor_indices(names, ["tail", "nose"]) == [0, 3]  # keypoint (column) order, as the reference selects them
    assert anchor_indices(names, []) == []
    with pytest.raises(ValueError, match="not found"):
        anchor_indices(names, ["paw"])


def test_cropzoom_parameter_names_match_reference():
    from lightning_pose_b200.data import bboxes
    from lightning_pose_b200.utils import cropzoom

    sig = lambda f: list(inspect.signature(f).parameters)
    assert sig(bboxes.crop_and_resize_frames) == ["frames", "bbox_rows", "resize_dims"]
    assert sig(cropzoom.compute_bboxes)[1:] == ["anchor_indices", "crop_ratio", "crop_height", "crop_width"]
    assert sig(cropzoom.smooth_bboxes)[1:] == ["method", "window"]
    assert inspect.signature(cropzoom.smooth_bboxes).parameters["window"].default == 5
    path = os.path.join(R.REF_ROOT, "lightning_pose", "data", "bboxes.py")
    if os.path.isfile(path):
        fn = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == "crop_and_resize_frames"][0]
        assert [a.arg for a in fn.args.args] == sig(bboxes.crop_and_resize_frames)
    path = os.path.join(R.REF_ROOT, "lightning_pose", "utils", "cropzoom.py")
    if os.path.isfile(path):
        fns = {n.name: n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef)}
        assert [a.arg for a in fns["_compute_bbox_df"].args.args][2:] == sig(cropzoom.compute_bboxes)[2:]
        assert [a.arg for a in fns["smooth_bbox"].args.args][2:] == sig(cropzoom.smooth_bboxes)[1:]


def test_batched_predictor_crop_mode_arguments():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = torch.nn.Linear(1, 1)
    with pytest.raises(ValueError, match="frame_hw"):
        BatchedPredictor(head, 3, 10, 4, (64, 64), features_of=lambda x: x, bboxes=torch.ones(10, 4))
    with pytest.raises(ValueError, match="features_of"):
        BatchedPredictor(head, 3, 10, 4, (64, 64), bboxes=torch.ones(10, 4), frame_hw=(128, 128))
