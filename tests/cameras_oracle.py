"""CPU oracle and golden generator for the calibrated multi-view geometry.  TEST INFRASTRUCTURE ONLY.

Restates, in plain torch on the CPU, the four kornia functions the reference's ``lightning_pose/data/cameras.py`` calls
(``kornia.geometry.calibration.undistort_points`` / ``distort_points``, ``kornia.geometry.camera.PinholeCamera.project``,
``kornia.geometry.epipolar.triangulate_points``) and the compositions the multi-view tracker builds from them
(``project_camera_pairs_to_3d`` :22-83, ``project_3d_to_2d`` :86-171, ``frame_to_model_batch`` ``data/bboxes.py:194-219``).
Every function keeps the dtype of its inputs: float64 in, float64 out.  kornia is not installed here, so the restatements
are pinned against OpenCV and the reference's known answers (``tests/test_cameras_oracle.py``).

``python tests/cameras_oracle.py`` writes ``tests/golden/cameras.npz``: with these restatements registered as the kornia
modules (and a placeholder ``aniposelib.cameras.CameraGroup``), the reference's own ``data/cameras.py`` loads unmodified
through ``oracle/ref_loader.py`` and is run in float64 on fp32-representable inputs; its outputs and float64 autograd
gradients are stored, and the restatements are checked against them.  Needs the full reference tree (sources and
tests); the GPU tests only read the committed npz and use the restatements.  Nothing under ``lightning_pose_b200/``
imports this module.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "cameras.npz")


# --------------------------------------------------------------------------------------
# kornia restatements
# --------------------------------------------------------------------------------------


def _pad_dist(dist: torch.Tensor) -> torch.Tensor:
    if dist.shape[-1] not in (4, 5, 8, 12, 14):
        raise ValueError(f"dist must have 4, 5, 8, 12 or 14 coefficients; got {dist.shape[-1]}")
    if dist.shape[-1] < 14:
        dist = F.pad(dist, [0, 14 - dist.shape[-1]])
    if bool(torch.any(dist[..., 12] != 0)) or bool(torch.any(dist[..., 13] != 0)):
        raise NotImplementedError("tilt distortion (coefficients 13, 14) is not restated")
    return dist


def undistort_points(points: torch.Tensor, K: torch.Tensor, dist: torch.Tensor, new_K: torch.Tensor | None = None,
                     num_iters: int = 5) -> torch.Tensor:
    """kornia.geometry.calibration.undistort_points: OpenCV's fixed-point undistortion in normalised coordinates
    (fx, fy, cx, cy of K; skew ignored), ``num_iters`` iterations, then back to pixels with ``new_K`` (default K).
    points (..., N, 2), K (..., 3, 3), dist (..., P)."""
    if new_K is None:
        new_K = K
    d = _pad_dist(dist)
    cx, cy, fx, fy = K[..., 0:1, 2], K[..., 1:2, 2], K[..., 0:1, 0], K[..., 1:2, 1]
    x = (points[..., 0] - cx) / fx
    y = (points[..., 1] - cy) / fy
    x0, y0 = x, y
    for _ in range(num_iters):
        r2 = x * x + y * y
        inv_rad = (1 + d[..., 5:6] * r2 + d[..., 6:7] * r2 * r2 + d[..., 7:8] * r2**3) / (
            1 + d[..., 0:1] * r2 + d[..., 1:2] * r2 * r2 + d[..., 4:5] * r2**3)
        dx = 2 * d[..., 2:3] * x * y + d[..., 3:4] * (r2 + 2 * x * x) + d[..., 8:9] * r2 + d[..., 9:10] * r2 * r2
        dy = d[..., 2:3] * (r2 + 2 * y * y) + 2 * d[..., 3:4] * x * y + d[..., 10:11] * r2 + d[..., 11:12] * r2 * r2
        x = (x0 - dx) * inv_rad
        y = (y0 - dy) * inv_rad
    x = new_K[..., 0:1, 0] * x + new_K[..., 0:1, 2]
    y = new_K[..., 1:2, 1] * y + new_K[..., 1:2, 2]
    return torch.stack([x, y], -1)


def distort_points(points: torch.Tensor, K: torch.Tensor, dist: torch.Tensor, new_K: torch.Tensor | None = None) -> torch.Tensor:
    """kornia.geometry.calibration.distort_points: OpenCV's distortion model applied to pixel points
    (normalised with ``new_K``, default K; back to pixels with the same)."""
    if new_K is None:
        new_K = K
    d = _pad_dist(dist)
    cx, cy, fx, fy = new_K[..., 0:1, 2], new_K[..., 1:2, 2], new_K[..., 0:1, 0], new_K[..., 1:2, 1]
    x = (points[..., 0] - cx) / fx
    y = (points[..., 1] - cy) / fy
    r2 = x * x + y * y
    rad = (1 + d[..., 0:1] * r2 + d[..., 1:2] * r2 * r2 + d[..., 4:5] * r2**3) / (
        1 + d[..., 5:6] * r2 + d[..., 6:7] * r2 * r2 + d[..., 7:8] * r2**3)
    xd = x * rad + 2 * d[..., 2:3] * x * y + d[..., 3:4] * (r2 + 2 * x * x) + d[..., 8:9] * r2 + d[..., 9:10] * r2 * r2
    yd = y * rad + d[..., 2:3] * (r2 + 2 * y * y) + 2 * d[..., 3:4] * x * y + d[..., 10:11] * r2 + d[..., 11:12] * r2 * r2
    return torch.stack([fx * xd + cx, fy * yd + cy], -1)


def convert_points_from_homogeneous(points: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """kornia.geometry.conversions.convert_points_from_homogeneous: divide by the last coordinate + eps where it
    exceeds eps in magnitude, else by 1."""
    z = points[..., -1:]
    scale = torch.where(torch.abs(z) > eps, 1.0 / (z + eps), torch.ones_like(z))
    return scale * points[..., :-1]


class PinholeCamera:
    """kornia.geometry.camera.PinholeCamera, the part cameras.py uses: ``project`` = dehomogenise((K E) [X; 1]) then
    dehomogenise again (4x4 intrinsics / extrinsics per batch element; height / width are not read)."""

    def __init__(self, intrinsics: torch.Tensor, extrinsics: torch.Tensor, height: torch.Tensor, width: torch.Tensor) -> None:
        self.intrinsics, self.extrinsics, self.height, self.width = intrinsics, extrinsics, height, width

    def project(self, point_3d: torch.Tensor) -> torch.Tensor:
        P = self.intrinsics @ self.extrinsics  # (B, 4, 4)
        ph = torch.cat([point_3d, torch.ones_like(point_3d[..., :1])], -1) @ P.transpose(-2, -1)
        return convert_points_from_homogeneous(convert_points_from_homogeneous(ph))


def triangulate_points(P1: torch.Tensor, P2: torch.Tensor, points1: torch.Tensor, points2: torch.Tensor) -> torch.Tensor:
    """kornia.geometry.epipolar.triangulate_points: DLT rows x P[2] - P[0], y P[2] - P[1] of both cameras; the 3-D point
    is the right singular vector of the smallest singular value, dehomogenised."""
    shape = torch.broadcast_shapes(points1.shape, points2.shape)[:-1] + (4, 4)
    X = torch.zeros(shape, dtype=points1.dtype, device=points1.device)
    for i in range(4):
        X[..., 0, i] = points1[..., 0] * P1[..., 2:3, i] - P1[..., 0:1, i]
        X[..., 1, i] = points1[..., 1] * P1[..., 2:3, i] - P1[..., 1:2, i]
        X[..., 2, i] = points2[..., 0] * P2[..., 2:3, i] - P2[..., 0:1, i]
        X[..., 3, i] = points2[..., 1] * P2[..., 2:3, i] - P2[..., 1:2, i]
    _, _, Vh = torch.linalg.svd(X)
    return convert_points_from_homogeneous(Vh.transpose(-2, -1)[..., -1])


def project_camera_pairs_to_3d(points, intrinsics, extrinsics, dist):
    """lightning_pose/data/cameras.py:22-83 without the per-batch boolean gathers: (B, V, K, 2) -> (B, V(V-1)/2, K, 3),
    NaN where the keypoint is NaN in either view of the pair."""
    b, v = points.shape[:2]
    eye = torch.eye(3, dtype=points.dtype).expand(b, v, 3, 3)
    und = undistort_points(points, intrinsics, dist, new_K=eye)
    out = []
    for j1 in range(v):
        for j2 in range(j1 + 1, v):
            p1, p2 = und[:, j1], und[:, j2]
            bad = torch.isnan(p1).any(-1) | torch.isnan(p2).any(-1)
            tri = triangulate_points(extrinsics[:, j1], extrinsics[:, j2],
                                     torch.where(bad[..., None], 0.0, p1), torch.where(bad[..., None], 0.0, p2))
            out.append(torch.where(bad[..., None], torch.full_like(tri, float("nan")), tri))
    return torch.stack(out, 1)


def project_3d_to_2d(points_3d, intrinsics, extrinsics, dist):
    """lightning_pose/data/cameras.py:86-171: (B, K, 3) -> (B, V, K, 2); distortion for the (b, v) whose dist row is not
    all zero."""
    b, v = intrinsics.shape[:2]
    k4 = torch.eye(4, dtype=points_3d.dtype).repeat(b, v, 1, 1)
    k4[:, :, :3, :3] = intrinsics
    e4 = torch.eye(4, dtype=points_3d.dtype).repeat(b, v, 1, 1)
    e4[:, :, :3, :4] = extrinsics
    out = []
    for j in range(v):
        p = PinholeCamera(k4[:, j], e4[:, j], None, None).project(points_3d)
        has = torch.any(dist[:, j] != 0, dim=-1)
        out.append(torch.where(has[:, None, None], distort_points(p, intrinsics[:, j], dist[:, j]), p))
    return torch.stack(out, 1)


def frame_to_model_batch(keypoints: torch.Tensor, bbox: torch.Tensor, model_height: int, model_width: int) -> torch.Tensor:
    """lightning_pose/data/bboxes.py:194-219: (B, V, K, 2) frame pixels -> model pixels, bbox (B, 4V) = [x, y, h, w]
    per view."""
    bb = bbox.reshape(bbox.shape[0], -1, 1, 4)
    x = (keypoints[..., 0] - bb[..., 0]) / bb[..., 3] * model_width
    y = (keypoints[..., 1] - bb[..., 1]) / bb[..., 2] * model_height
    return torch.stack([x, y], -1)


# --------------------------------------------------------------------------------------
# golden generation (runs the reference)
# --------------------------------------------------------------------------------------


def _ref_root():
    from oracle import ref_loader as R

    return R.REF_ROOT


def _fly_rig():
    """The anipose-fly calibration of the reference's tests/data/test_cameras.py:11-89 (3 views, 2 keypoints, 5 params;
    focal lengths up to 1e5, k1 = -1906), read from that file's fixtures; batch 2: the fixture, then the same with
    keypoint 0 NaN in view 0."""
    import ast

    path = os.path.join(_ref_root(), "tests", "data", "test_cameras.py")
    tree = ast.parse(open(path).read())
    fx = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("points_2d", "points_3d_single", "intrinsics", "extrinsics", "distortions"):
            ns = {"torch": torch}
            body = node.body[-1]
            assert isinstance(body, ast.Return)
            fx[node.name] = eval(compile(ast.Expression(body.value), path, "eval"), ns)
    pts = fx["points_2d"][None].repeat(2, 1, 1, 1)
    pts[1, 0, 0] = float("nan")
    gen = torch.Generator().manual_seed(60)
    bbox = torch.cat([torch.rand(2, 3, 2, generator=gen) * 200, 500 + torch.rand(2, 3, 2, generator=gen) * 200], -1).reshape(2, 12)
    rep = lambda t: t[None].repeat(2, *([1] * t.dim()))
    return pts, rep(fx["intrinsics"]), rep(fx["extrinsics"]), rep(fx["distortions"]), bbox, (256, 256), rep(fx["points_3d_single"])


def _ring_rig(cam, v, p, seed, b=2, k=5, img=384):
    """V cameras on a circle of radius 2 around the origin looking inward, intrinsics and distortion drawn as in
    tests/models/test_heatmap_tracker_multiview.py:205-246 (whose extrinsics put every camera at the same centre, which
    leaves nothing to triangulate; here the centres are spread over the circle), P distortion coefficients (view 1 without distortion), keypoints = projections of random 3-D points plus
    0.5 px noise; keypoint 1 NaN in view 0 of example 0, keypoint 2 NaN everywhere in example 1."""
    gen = torch.Generator().manual_seed(seed)
    K = torch.zeros(b, v, 3, 3)
    E = torch.zeros(b, v, 3, 4)
    for j in range(v):
        f = 800.0 + torch.randn(b, generator=gen) * 50
        K[:, j, 0, 0], K[:, j, 1, 1] = f, f
        K[:, j, 0, 2] = img / 2 + torch.randn(b, generator=gen) * 10
        K[:, j, 1, 2] = img / 2 + torch.randn(b, generator=gen) * 10
        K[:, j, 2, 2] = 1.0
        # centre C = 2 (-sin a, 0, -cos a), optical axis towards the origin: R = rot_y(-a), t = -R C = (0, 0, 2)
        a = j / v * 2 * math.pi
        E[:, j] = torch.tensor([[math.cos(a), 0.0, -math.sin(a), 0.0], [0.0, 1.0, 0.0, 0.0],
                                [math.sin(a), 0.0, math.cos(a), 2.0]])
    D = torch.randn(b, v, p, generator=gen) * 0.1
    if p > 5:
        D[..., 5:] *= 0.1
    D[:, 1] = 0.0
    p3 = torch.randn(b, k, 3, generator=gen) * 0.3  # well inside the rig: 5 undistortion iterations converge
    pts = cam.project_3d_to_2d(p3.double(), K.double(), E.double(), D.double()).float()
    pts = pts + torch.randn(pts.shape, generator=gen) * 0.5
    pts[0, 0, 1] = float("nan")
    pts[1, :, 2] = float("nan")
    p3n = torch.randn(b, k, 3, generator=gen) * 0.5
    p3n[0, 3] = float("nan")
    bbox = torch.cat([torch.rand(b, v, 2, generator=gen) * 40, 300 + torch.rand(b, v, 2, generator=gen) * 100], -1).reshape(b, 4 * v)
    return pts, K, E, D, bbox, (img, img), p3n


def gen_cameras(cam, db):
    """project_camera_pairs_to_3d / project_3d_to_2d (data/cameras.py) and frame_to_model_batch (data/bboxes.py) in float64
    on fp32-representable inputs, with float64 autograd gradients for seeded upstream gradients."""
    g = {}
    rigs = {"fly": _fly_rig()}
    for v, p, seed in ((2, 4, 61), (3, 8, 62), (4, 5, 63), (6, 12, 64)):
        rigs[f"ring{v}"] = _ring_rig(cam, v, p, seed)
    for name, (pts, K, E, D, bbox, hw, p3n) in rigs.items():
        b, v, k, _ = pts.shape
        gen = torch.Generator().manual_seed(70 + v)
        g3 = torch.randn(b, v * (v - 1) // 2, k, 3, generator=gen)
        g2 = torch.randn(b, v, k, 2, generator=gen)
        for key, t in (("points", pts), ("K", K), ("E", E), ("dist", D), ("bbox", bbox), ("points3d", p3n), ("g3", g3), ("g2", g2)):
            g[f"{name}_in_{key}"] = _np(t.float())
        g[f"{name}_in_model_hw"] = np.array(hw, np.int64)
        K, E, D, bbox = (t.float().double() for t in (K, E, D, bbox))
        bd = {"images": torch.zeros(b, v, 3, *hw), "bbox": bbox}
        with torch.enable_grad():
            x = pts.float().double().requires_grad_(True)
            p3d = cam.project_camera_pairs_to_3d(x, K, E, D)
            (p3d * g3.double()).sum().backward()
            g[f"{name}_out_p3d"], g[f"{name}_out_grad_points_tri"] = _np(p3d), _np(x.grad)
            _check(f"cameras {name} pairs -> 3d", p3d, project_camera_pairs_to_3d(x.detach(), K, E, D), atol=1e-9, rtol=1e-7)

            y = p3n.float().double().requires_grad_(True)
            p2d = cam.project_3d_to_2d(y, K, E, D)
            (p2d * g2.double()).sum().backward()
            g[f"{name}_out_p2d"], g[f"{name}_out_grad_points3d"] = _np(p2d), _np(y.grad)
            _check(f"cameras {name} 3d -> 2d", p2d, project_3d_to_2d(y.detach(), K, E, D), atol=1e-9, rtol=1e-9)

            x = pts.float().double().requires_grad_(True)
            p3d = cam.project_camera_pairs_to_3d(x, K, E, D)
            rep = db.frame_to_model_batch(bd, cam.project_3d_to_2d(torch.mean(p3d, dim=1), K, E, D))
            (rep * g2.double()).sum().backward()
            g[f"{name}_out_reproj"], g[f"{name}_out_grad_points_reproj"] = _np(rep), _np(x.grad)
            mine = frame_to_model_batch(project_3d_to_2d(project_camera_pairs_to_3d(x.detach(), K, E, D).mean(1), K, E, D), bbox, *hw)
            _check(f"cameras {name} reprojection (model coords)", rep, mine, atol=1e-9, rtol=1e-7)

        f2m = db.frame_to_model_batch(bd, pts.float().double())
        g[f"{name}_out_frame_to_model"] = _np(f2m)
        _check(f"cameras {name} frame_to_model", f2m, frame_to_model_batch(pts.float().double(), bbox, *hw), atol=1e-9, rtol=1e-12)
    return g


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _check(name, ref, mine, atol=1e-6, rtol=1e-5):
    ref, mine = _np(ref), _np(mine)
    assert ref.shape == mine.shape, (name, ref.shape, mine.shape)
    ok = np.allclose(ref, mine, atol=atol, rtol=rtol, equal_nan=True)
    err = float(np.nanmax(np.abs(ref - mine))) if ref.size else 0.0
    print(f"  oracle-vs-reference {name:45s} max|diff| = {err:.3e} {'OK' if ok else 'MISMATCH'}")
    assert ok, name


def load_reference():
    """(reference data/cameras.py, reference data/bboxes.py), loaded unmodified with the kornia calls bound to the
    restatements above."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import importlib
    import types

    from oracle import ref_loader as R

    R.install()
    for name, attrs in (("kornia.geometry.calibration", {"undistort_points": undistort_points, "distort_points": distort_points}),
                        ("kornia.geometry.camera", {"PinholeCamera": PinholeCamera}),
                        ("kornia.geometry.epipolar", {"triangulate_points": triangulate_points}),
                        ("aniposelib", {}),
                        ("aniposelib.cameras", {"CameraGroup": type("CameraGroup", (), {})})):  # data-layer base class
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        sys.modules[name] = mod
    return importlib.import_module("lightning_pose.data.cameras"), importlib.import_module("lightning_pose.data.bboxes")


def reference_tree_available() -> bool:
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return os.path.isfile(os.path.join(R.REF_ROOT, "tests", "data", "test_cameras.py"))


def main(path: str = GOLDEN_PATH) -> None:
    assert reference_tree_available(), "needs the full reference tree (sources and tests)"
    cam, db = load_reference()
    with torch.no_grad():
        arrays = gen_cameras(cam, db)
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(arrays)} arrays, {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main(*sys.argv[1:])
