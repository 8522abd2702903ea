"""CPU: the camera-geometry restatements in tests/cameras_oracle.py (kornia undistort_points / distort_points /
PinholeCamera.project / triangulate_points) against OpenCV, the reference's known answers
(tests/data/test_cameras.py) and tests/golden/cameras.npz; the new ABI entries and Python mirror without a GPU."""
import ctypes
import filecmp
import inspect
import math
import os

import cv2
import numpy as np
import pytest
import torch

import cameras_oracle as O
from oracle import ref_loader as R

T = torch.from_numpy
RIGS = ("fly", "ring2", "ring3", "ring4", "ring6")


def close(a, b, atol=1e-6, rtol=1e-5):
    a = a.detach().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    np.testing.assert_allclose(a, np.asarray(b), atol=atol, rtol=rtol, equal_nan=True)


def rig(g, name):
    """float64 copies of a rig's fp32 inputs: points, K, E, dist, bbox, (model h, w), points3d"""
    d = lambda k: T(g[f"{name}_in_{k}"]).double()
    return d("points"), d("K"), d("E"), d("dist"), d("bbox"), tuple(int(x) for x in g[f"{name}_in_model_hw"]), d("points3d")


def _seeded_camera(seed, p):
    gen = np.random.default_rng(seed)
    K = np.array([[820.0, 0.0, 190.0], [0.0, 790.0, 200.0], [0.0, 0.0, 1.0]])
    rvec = gen.normal(size=3) * 0.3
    R_, _ = cv2.Rodrigues(rvec)
    t = np.array([0.1, -0.2, 3.0]) + gen.normal(size=3) * 0.1
    dist = gen.normal(size=p) * 0.05
    return K, rvec, R_, t, dist


# ---- OpenCV cross-checks -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [4, 5, 8, 12])
def test_undistort_points_matches_opencv(p):
    K, _, _, _, dist = _seeded_camera(p, p)
    pts = np.random.default_rng(1).uniform(20, 360, size=(40, 2))
    crit = (cv2.TERM_CRITERIA_COUNT, 5, 0.0)
    ref = cv2.undistortPointsIter(pts[:, None, :], K, dist, None, None, crit)[:, 0, :]
    mine = O.undistort_points(T(pts), T(K), T(dist), new_K=torch.eye(3, dtype=torch.float64))
    assert mine.dtype == torch.float64
    close(mine, ref, atol=1e-12, rtol=1e-10)


@pytest.mark.parametrize("p", [4, 5, 8, 12])
def test_projection_and_distortion_match_opencv(p):
    K, rvec, R_, t, dist = _seeded_camera(10 + p, p)
    X = np.random.default_rng(2).normal(size=(30, 3)) * 0.4
    ref = cv2.projectPoints(X, rvec, t, K, dist)[0][:, 0, :]
    k4, e4 = torch.eye(4, dtype=torch.float64)[None], torch.eye(4, dtype=torch.float64)[None]
    k4[0, :3, :3], e4[0, :3, :3], e4[0, :3, 3] = T(K), T(R_), T(t)
    proj = O.PinholeCamera(k4, e4, None, None).project(T(X)[None])
    mine = O.distort_points(proj, T(K)[None], T(dist)[None])[0]
    assert mine.dtype == torch.float64
    close(mine, ref, atol=1e-6, rtol=1e-8)  # kornia's +1e-8 in the dehomogenisation


def test_triangulate_points_matches_opencv():
    _, _, R1, t1, _ = _seeded_camera(20, 5)
    _, _, R2, t2, _ = _seeded_camera(21, 5)
    P1, P2 = np.hstack([R1, t1[:, None]]), np.hstack([R2, t2[:, None]])
    X = np.random.default_rng(3).normal(size=(25, 3)) * 0.4
    x1 = (X @ R1.T + t1)[:, :2] / (X @ R1.T + t1)[:, 2:]
    x2 = (X @ R2.T + t2)[:, :2] / (X @ R2.T + t2)[:, 2:]
    x1 += np.random.default_rng(4).normal(size=x1.shape) * 1e-3  # inconsistent rays: the SVD's least-squares answer
    h = cv2.triangulatePoints(P1, P2, x1.T, x2.T)
    ref = (h[:3] / h[3]).T
    mine = O.triangulate_points(T(P1), T(P2), T(x1), T(x2))
    assert mine.dtype == torch.float64
    close(mine, ref, atol=1e-9, rtol=1e-7)


# ---- the reference's known answers (tests/data/test_cameras.py), fly rig ---------------------------------------------
def test_reference_known_answers_fly(golden):
    g = golden("cameras")
    pts, K, E, D, bbox, hw, p3 = [t.float() if isinstance(t, torch.Tensor) else t for t in rig(g, "fly")]
    p3d = O.project_camera_pairs_to_3d(pts, K, E, D)
    assert p3d.shape == (2, 3, 2, 3)
    assert torch.allclose(p3d[0], p3[0][None].expand(3, 2, 3), rtol=1e-2)
    # keypoint 0 NaN in view 0: pairs (0,1), (0,2) NaN for it, pair (1,2) unaffected
    assert torch.isnan(p3d[1, 0, 0]).all() and torch.isnan(p3d[1, 1, 0]).all()
    assert torch.allclose(p3d[1, :, 1], p3[0, 1].expand(3, 3), rtol=1e-2) and torch.allclose(p3d[1, 2], p3d[0, 2], rtol=1e-3)
    p2d = O.project_3d_to_2d(p3, K, E, D)
    assert torch.allclose(p2d[0], pts[0], rtol=1e-4)
    pn = p3.clone()
    pn[0, 0] = float("nan")
    out = O.project_3d_to_2d(pn, K, E, D)
    assert torch.isnan(out[0, :, 0]).all() and torch.allclose(out[0, :, 1], pts[0, :, 1], rtol=1e-4)
    assert torch.isnan(O.project_3d_to_2d(torch.full_like(p3, float("nan")), K, E, D)).all()
    back = O.project_3d_to_2d(p3d[:1].mean(1), K[:1], E[:1], D[:1])
    assert float(torch.norm(back - pts[:1], dim=-1).max()) < 1.0  # round trip under 1 px


@pytest.mark.parametrize("name", RIGS)
def test_oracle_matches_cameras_golden(golden, name):
    g = golden("cameras")
    pts, K, E, D, bbox, hw, p3n = rig(g, name)
    close(O.project_camera_pairs_to_3d(pts, K, E, D), g[f"{name}_out_p3d"], atol=1e-9, rtol=1e-7)
    close(O.project_3d_to_2d(p3n, K, E, D), g[f"{name}_out_p2d"], atol=1e-9, rtol=1e-9)
    close(O.frame_to_model_batch(pts, bbox, *hw), g[f"{name}_out_frame_to_model"], atol=1e-9, rtol=1e-12)
    x = pts.clone().requires_grad_(True)
    rep = O.frame_to_model_batch(O.project_3d_to_2d(O.project_camera_pairs_to_3d(x, K, E, D).mean(1), K, E, D), bbox, *hw)
    close(rep, g[f"{name}_out_reproj"], atol=1e-9, rtol=1e-7)
    (rep * T(g[f"{name}_in_g2"]).double()).sum().backward()
    ref = g[f"{name}_out_grad_points_reproj"]
    fin = np.isfinite(ref)
    close(x.grad.numpy()[fin], ref[fin], atol=1e-9 * np.abs(ref[fin]).max(), rtol=1e-6)


def test_golden_rigs_cover_the_issue_cases(golden):
    g = golden("cameras")
    assert sorted({g[f"{n}_in_dist"].shape[-1] for n in RIGS}) == [4, 5, 8, 12]
    assert sorted(g[f"{n}_in_points"].shape[1] for n in RIGS if n != "fly") == [2, 3, 4, 6]
    for n in RIGS[1:]:
        d = g[f"{n}_in_dist"]
        assert (np.abs(d).reshape(-1, d.shape[-1]).max(-1) == 0).any()  # a view without distortion
        p = g[f"{n}_in_points"]
        nan_kp = np.isnan(p).any(-1)  # (B, V, K)
        assert (nan_kp.any(1) & ~nan_kp.all(1)).any() and nan_kp.all(1).any()  # NaN in one view; NaN in every view


# ---- goldens are reproducible ----------------------------------------------------------------------------------------
@pytest.mark.skipif(not O.reference_tree_available(), reason="needs the full reference tree (sources and tests) to regenerate the goldens")
def test_regenerating_goldens_is_byte_identical(tmp_path, monkeypatch):
    from oracle import gen_golden

    committed = gen_golden.GOLDEN_DIR
    monkeypatch.setattr(gen_golden, "GOLDEN_DIR", str(tmp_path))
    gen_golden.main()
    O.main(str(tmp_path / "cameras.npz"))
    for name in ("decode", "targets", "head", "remap", "losses", "mhcrnn", "cameras"):
        assert filecmp.cmp(os.path.join(committed, f"{name}.npz"), str(tmp_path / f"{name}.npz"), shallow=False), name


# ---- ABI and mirror, no GPU ----------------------------------------------------------------------------------------
def test_camera_entry_points_validate_without_gpu():
    from lightning_pose_b200 import _lib

    L, p = _lib.lib, ctypes.c_void_p(16)
    for rc in (
        L.lpb_triangulate_pairs_fwd(None, p, p, p, 1, 3, 2, 5, p, None),
        L.lpb_triangulate_pairs_bwd(p, p, p, p, None, 1, 3, 2, 5, p, None),
        L.lpb_project_points_fwd(p, 0, None, p, p, None, 0.0, 0.0, 1, 3, 2, 5, p, None),
        L.lpb_project_points_bwd(p, 0, p, p, p, None, 0.0, 0.0, p, 1, 3, 2, 5, None, None),
        L.lpb_frame_to_model(p, 1, 3, 2, None, 256.0, 256.0, 0, p, None),
        L.lpb_pairwise_projections_loss_fwd(p, None, 1, 3, 2, p, None),
        L.lpb_pairwise_projections_loss_bwd(p, p, 1, 3, 2, None, p, p, None),
    ):
        assert rc == -1 and b"null pointer" in L.lpb_last_error()
    for P in (0, 3, 6, 14):
        assert L.lpb_triangulate_pairs_fwd(p, p, p, p, 1, 3, 2, P, p, None) == -1 and b"bad P" in L.lpb_last_error()
        assert L.lpb_project_points_bwd(p, 0, p, p, p, None, 0.0, 0.0, p, 1, 3, 2, P, p, None) == -1 and b"bad P" in L.lpb_last_error()
    for V in (0, 1, 65):
        assert L.lpb_triangulate_pairs_bwd(p, p, p, p, p, 1, V, 2, 5, p, None) == -1 and b"bad V" in L.lpb_last_error()
    assert L.lpb_project_points_fwd(p, 0, p, p, p, None, 0.0, 0.0, 1, 0, 2, 5, p, None) == -1 and b"bad V" in L.lpb_last_error()
    assert L.lpb_project_points_fwd(p, 0, p, p, p, p, 0.0, 0.0, 1, 2, 2, 5, p, None) == -1  # bbox without a model size


def test_camera_mirror_refuses_cpu_tensors():
    from lightning_pose_b200.data.bboxes import frame_to_model_batch
    from lightning_pose_b200.data.cameras import project_3d_to_2d, project_camera_pairs_to_3d
    from lightning_pose_b200.losses.losses import PairwiseProjectionsLoss

    K, E, D = torch.eye(3).expand(1, 2, 3, 3), torch.zeros(1, 2, 3, 4), torch.zeros(1, 2, 5)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        project_camera_pairs_to_3d(torch.rand(1, 2, 3, 2), K, E, D)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        project_3d_to_2d(torch.rand(1, 3, 3), K, E, D)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        frame_to_model_batch({"images": torch.zeros(1, 2, 3, 64, 64), "bbox": torch.ones(1, 8)}, torch.rand(1, 2, 3, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        PairwiseProjectionsLoss()(keypoints_targ_3d=torch.rand(1, 3, 3), keypoints_pred_3d=torch.rand(1, 1, 3, 3))


def test_camera_mirror_parameter_names_match_reference():
    from lightning_pose_b200.data import bboxes, cameras

    want = {
        (cameras, "project_camera_pairs_to_3d"): ["points", "intrinsics", "extrinsics", "dist"],
        (cameras, "project_3d_to_2d"): ["points_3d", "intrinsics", "extrinsics", "dist"],
        (bboxes, "frame_to_model_batch"): ["batch_dict", "frame_keypoints"],
    }
    for (mod, fn), names in want.items():
        assert list(inspect.signature(getattr(mod, fn)).parameters) == names, fn
    if R.reference_available():
        import ast

        for rel, mod in (("data/cameras.py", cameras), ("data/bboxes.py", bboxes)):
            path = os.path.join(R.REF_ROOT, "lightning_pose", rel)
            if not os.path.isfile(path):  # the staged copy holds the hot-path files only
                continue
            tree = ast.parse(open(path).read())
            for node in tree.body:
                if isinstance(node, ast.FunctionDef) and (mod, node.name) in want:
                    assert [a.arg for a in node.args.args] == want[(mod, node.name)], node.name


def test_ring_rig_geometry_is_sane(golden):
    """Ring cameras look at the origin from radius 2: every finite golden 3-D point lies in front of every camera."""
    g = golden("cameras")
    for n in RIGS[1:]:
        E = g[f"{n}_in_E"].astype(np.float64)
        p3d = g[f"{n}_out_p3d"]
        pts = p3d[np.isfinite(p3d).all(-1)]
        z = np.einsum("bvj,nj->bvn", E[:, :, 2, :3], pts) + E[:, :, 2, 3:4]
        assert (z > 0.5).all() and math.isfinite(float(np.abs(pts).max()))
