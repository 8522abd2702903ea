"""CPU: tests/frame_resize_oracle.py (the rule of lpb_frames_crop_resize_cv2) equals cv2.resize(INTER_LINEAR) byte for
byte, equals the committed OpenCV golden set, and each wrong rule a port could take changes at least one byte."""
import os

import numpy as np
import pytest

import frame_resize_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame_resize.npz")

# (source (h, w), output (h, w)): downscales, the exact 2x downscales where OpenCV switches to INTER_AREA, upscales,
# identity, one-pixel and one-line crops, and output sizes that are not multiples of 8
SHAPES = [
    ((1024, 1280), (384, 384)), ((406, 396), (256, 256)), ((720, 1280), (384, 384)), ((1000, 37), (256, 256)),
    ((512, 512), (256, 256)), ((1024, 1024), (512, 512)),
    ((100, 90), (384, 384)), ((37, 53), (256, 256)), ((37, 1000), (384, 384)), ((300, 200), (384, 384)), ((250, 250), (384, 384)),
    ((64, 64), (64, 64)),
    ((1, 1), (384, 384)), ((1, 57), (256, 256)), ((57, 1), (130, 250)),
    ((200, 300), (123, 77)), ((33, 47), (61, 93)), ((90, 130), (13, 201)),
]


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("src,dst", SHAPES, ids=[f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in SHAPES])
def test_oracle_equals_cv2(src, dst):
    cv2 = pytest.importorskip("cv2")
    img = _image(*src, seed=src[0] * 7 + src[1])
    ref = cv2.resize(img, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(O.resize_linear_u8(img, *dst), ref)


@pytest.mark.parametrize("rule", O.WRONG_RULES)
def test_each_wrong_rule_changes_a_byte(rule):
    """f kept in double, vertical weights zeroed where the row index is clamped, no >> 4 pre-shift, the scalar
    rounding: each gives at least one different byte on the shapes above (which the right rule gets exactly)."""
    changed = 0
    for src, dst in SHAPES:
        img = _image(*src, seed=src[0] * 7 + src[1])
        changed += int((O.resize_linear_u8(img, *dst, wrong=rule) != O.resize_linear_u8(img, *dst)).sum())
    assert changed > 0


def test_normalize_is_numpy_fp32():
    """(u8 / 255 - mean) / std in fp32, each step rounded: not a fused or reassociated form."""
    u8 = np.arange(256, dtype=np.uint8).reshape(-1, 1).repeat(3, axis=1)
    got = O.normalize(u8)
    want = (u8.astype(np.float32) / np.float32(255.0) - np.array(O.IMAGENET_MEAN, np.float32)) / np.array(O.IMAGENET_STD, np.float32)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    fused = (u8.astype(np.float32) * np.float32(1 / 255.0) - np.array(O.IMAGENET_MEAN, np.float32)) * (1 / np.array(O.IMAGENET_STD, np.float32))
    assert not np.array_equal(got, fused.astype(np.float32))


def test_crop_is_a_numpy_slice():
    frames = np.zeros((2, 10, 20, 3), dtype=np.uint8)
    assert O.crop(frames, None)[1] == [0, 0, 10, 20]
    assert O.crop(frames, (15, 7, 100, 100))[1] == [15, 7, 3, 5]   # the far edges clip
    assert O.crop(frames, (0, 0, 1, 1))[1] == [0, 0, 1, 1]


def test_golden_is_cv2_and_the_oracle():
    """tests/golden/frame_resize.npz was written by cv2 (scripts/gen_frame_resize_golden.py); the oracle reproduces
    every byte of it, so the GPU tests compare with OpenCV without importing it."""
    g = np.load(GOLDEN)
    names = sorted({k[: -len("_frames")] for k in g.files if k.endswith("_frames")})
    assert len(names) >= 8
    for name in names:
        box = g[f"{name}_box"]
        box = None if box[0] < 0 else tuple(int(v) for v in box)
        oh, ow = g[f"{name}_u8"].shape[1:3]
        u8, f32, row = O.crop_resize_normalize(g[f"{name}_frames"], box, oh, ow)
        assert np.array_equal(u8, g[f"{name}_u8"]), name
        assert np.array_equal(f32.view(np.uint32), g[f"{name}_f32"].view(np.uint32)), name
        assert np.array_equal(np.array(row, np.float32), g[f"{name}_bbox"]), name
