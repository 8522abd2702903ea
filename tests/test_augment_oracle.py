"""CPU: the float64 augmentation oracle (tests/augment_oracle.py) against the reference's own undo and an independent
torch composition, the ABI's argument checks and the Python surface's validation."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import augment_oracle as O

RNG = np.random.default_rng(7)


def random_params(n):
    lo, hi = np.array([-10, 0.8, 0.8, 0.75, 0.75, 0.0]), np.array([10, 1.2, 1.2, 1.25, 1.25, 10.0])
    return lo + (hi - lo) * RNG.random((n, 6))


@pytest.mark.skipif(not O.reference_tree_available(), reason="needs the reference tree (lightning_pose/data/utils.py)")
def test_matrix_is_what_the_reference_undo_inverts():
    ref = O.load_reference_utils()
    size = (64, 96)
    params = random_params(2)
    ms = [O.dlc_matrix(p, size) for p in params]
    pts = RNG.uniform(-20, 120, size=(6, 5, 2))  # (seq, K, 2) in (x, y)
    warped = [pts @ m[:, :2].T + m[:, 2] for m in ms]
    # single view: one (2, 3) transform for the whole sequence (dali.py:286)
    got = ref.undo_affine_transform(torch.from_numpy(warped[0]), torch.from_numpy(ms[0])).detach().numpy()
    np.testing.assert_allclose(got, pts, atol=1e-9, rtol=0)
    # two views: (V, 1, 2, 3), keypoints of view v in columns [v K, (v + 1) K) (tests/data/test_datamodules.py:348,430)
    kp = torch.from_numpy(np.concatenate(warped, axis=1).reshape(6, -1))
    tf = torch.from_numpy(np.stack(ms)[:, None])
    got = ref.undo_affine_transform_batch(kp, tf, is_multiview=True).detach().numpy().reshape(6, -1, 2)
    np.testing.assert_allclose(got, np.concatenate([pts, pts], axis=1), atol=1e-9, rtol=0)


@pytest.mark.parametrize("src,size", [((100, 140), (64, 96)), ((50, 70), (64, 64)), ((40, 40), (48, 30))])
def test_warp_matches_grid_sample(src, size):
    u8 = RNG.integers(0, 256, size=(2, *src, 3), dtype=np.uint8)
    img = O.resize(u8, size)
    for p in random_params(3):
        m = O.dlc_matrix(p, size)
        got = O.warp(img, m)
        # grid_sample on the same float64 image: theta maps destination to source in [-1, 1] units (align_corners=False)
        h, w = size
        a_inv = np.linalg.inv(m[:, :2])
        to_norm = np.array([[2.0 / w, 0, -1], [0, 2.0 / h, -1], [0, 0, 1]])
        inv = np.eye(3)
        inv[:2] = np.concatenate([a_inv, -a_inv @ m[:, 2:]], axis=1)
        theta = (to_norm @ inv @ np.linalg.inv(to_norm))[:2]
        x = torch.from_numpy(img).permute(0, 3, 1, 2)
        grid = F.affine_grid(torch.from_numpy(theta)[None].expand(2, 2, 3), list(x.shape), align_corners=False)
        want = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False).permute(0, 2, 3, 1)
        np.testing.assert_allclose(got, want.numpy(), atol=1e-9, rtol=0)


def test_resize_matches_interpolate():
    u8 = RNG.integers(0, 256, size=(2, 100, 140, 3), dtype=np.uint8)
    for size in [(64, 96), (50, 70), (128, 160)]:
        want = F.interpolate(torch.from_numpy(u8).permute(0, 3, 1, 2).double(), size=size, mode="bilinear", align_corners=False)
        np.testing.assert_allclose(O.resize(u8, size), want.permute(0, 2, 3, 1).numpy(), atol=1e-9)


def test_identity_parameters_reproduce_the_plain_resize():
    u8 = RNG.integers(0, 256, size=(3, 100, 140, 3), dtype=np.uint8)
    frames, m = O.augment(u8, (64, 96), [0.0, 1.0, 1.0, 1.0, 1.0, 0.0])
    np.testing.assert_array_equal(m, [[1, 0, 0], [0, 1, 0]])
    np.testing.assert_allclose(frames, O.normalise(O.resize(u8, (64, 96))), atol=1e-12)


def test_non_square_centre_is_h_half_w_half_as_x_y():
    """The reference passes (h / 2, w / 2) as the (x, y) centre: that point is fixed, the image centre is not."""
    size = (64, 96)
    m = O.dlc_matrix([7.0, 1.1, 0.9, 1, 1, 0], size)
    np.testing.assert_allclose(m[:, :2] @ [32.0, 48.0] + m[:, 2], [32.0, 48.0], atol=1e-12)
    assert np.abs(m[:, :2] @ [48.0, 32.0] + m[:, 2] - [48.0, 32.0]).max() > 1.0
    # A = diag(sx, sy) R, t = c - A c
    th = np.deg2rad(7.0)
    a = np.diag([1.1, 0.9]) @ np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    np.testing.assert_allclose(m[:, :2], a, atol=1e-15)
    np.testing.assert_allclose(m[:, 2], np.array([32.0, 48.0]) - a @ [32.0, 48.0], atol=1e-12)


def test_abi_argument_validation():
    from lightning_pose_b200 import _lib

    L = _lib.lib
    p = C.c_void_p(16)
    m3, s3 = (C.c_float * 3)(0.5, 0.5, 0.5), (C.c_float * 3)(0.2, 0.2, 0.2)
    bad = (C.c_float * 3)(0.2, 0.0, 0.2)
    for args, msg in (
        ((None, 1, 8, 8, 4, 4, p, p, m3, s3, 0, 0, p, p, None), b"null pointer"),
        ((p, 1, 8, 8, 4, 4, None, p, m3, s3, 0, 0, p, p, None), b"null pointer"),
        ((p, 1, 8, 8, 4, 4, p, None, m3, s3, 0, 0, p, p, None), b"null pointer"),
        ((p, 1, 8, 8, 4, 4, p, p, m3, s3, 0, 0, p, None, None), b"null pointer"),
        ((p, -1, 8, 8, 4, 4, p, p, m3, s3, 0, 0, p, p, None), b"bad shape"),
        ((p, 1, 0, 8, 4, 4, p, p, m3, s3, 0, 0, p, p, None), b"bad shape"),
        ((p, 1, 8, 8, 4, 0, p, p, m3, s3, 0, 0, p, p, None), b"bad shape"),
        ((p, 1, 8, 8, 4, 4, p, p, m3, s3, 2, 0, p, p, None), b"bad shape"),
        ((p, 1, 8, 8, 4, 4, p, p, m3, bad, 0, 0, p, p, None), b"std must be positive"),
    ):
        assert L.lpb_frames_augment_normalize(*args) == -1
        assert msg in L.lpb_last_error()
    assert L.lpb_frames_augment_normalize(p, 0, 8, 8, 4, 4, p, p, m3, s3, 1, 1, p, p, None) == 0  # F = 0: nothing to do


def test_surface_validation_without_gpu():
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.video import AUGMENTED_IMGAUG, frames_to_unlabeled_batch

    assert AUGMENTED_IMGAUG == ("dlc", "dlc-top-down")
    u8 = torch.zeros((2, 8, 8, 3), dtype=torch.uint8)
    for imgaug in AUGMENTED_IMGAUG:
        with pytest.raises(ValueError, match="resize_dims"):
            frames_to_unlabeled_batch(u8, None, imgaug=imgaug)
        with pytest.raises(ValueError, match="bounding-box"):
            frames_to_unlabeled_batch(u8, (8, 8), imgaug=imgaug, bbox=torch.zeros(2, 4))
    # every other value takes the plain path, which refuses CPU tensors (no CPU fallback) but needs no resize_dims
    for imgaug in ("default", None, "dlc-lr", "imgaug"):
        with pytest.raises(RuntimeError, match="CUDA"):
            frames_to_unlabeled_batch(u8, None, imgaug=imgaug)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.frames_augment_normalize(u8, (8, 8), torch.zeros(6), torch.zeros(1, dtype=torch.int64))
    assert [(c.start, c.stop, lo, hi) for c, lo, hi in ops.DLC_PARAM_RANGES] == [
        (0, 1, -10.0, 10.0), (1, 3, 0.8, 1.2), (3, 5, 0.75, 1.25), (5, 6, 0.0, 10.0)]
    params, seeds = ops.draw_dlc_params(5, "cpu", generator=torch.Generator().manual_seed(0))
    assert params.shape == (5, 6) and params.dtype == torch.float32 and seeds.shape == (5,) and seeds.dtype == torch.int64
    for c, lo, hi in ops.DLC_PARAM_RANGES:
        assert bool((params[:, c] >= lo).all() and (params[:, c] <= hi).all())
