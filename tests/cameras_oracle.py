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
# the kernels' conventions, rigs and cases at the edges (tests/test_cameras_edges_*.py)
# --------------------------------------------------------------------------------------


def camera_pairs(v: int):
    """the pair order of the pair axis: itertools.combinations(range(v), 2)"""
    return [(i, j) for i in range(v) for j in range(i + 1, v)]


def triangulate_points_v3_nonneg(P1, P2, points1, points2, eps=1e-8, dlt_dtype=None):
    """triangulate_points with the kernels' sign convention: the singular vector is negated when its last coordinate
    is negative.  LAPACK's sign is arbitrary, and 1 / (z + eps) is not odd in z, so without the convention a far point
    (|v3| below ~2e-2) dehomogenises differently for the two signs.  ``dlt_dtype``: build and solve the DLT in that
    dtype (float32 is a mutant).  P1, P2 (B, 3, 4), points (B, K, 2) normalised."""
    rows = [points1[..., 0:1] * P1[:, None, 2] - P1[:, None, 0], points1[..., 1:2] * P1[:, None, 2] - P1[:, None, 1],
            points2[..., 0:1] * P2[:, None, 2] - P2[:, None, 0], points2[..., 1:2] * P2[:, None, 2] - P2[:, None, 1]]
    A = torch.stack(rows, -2)
    if dlt_dtype is not None:
        A = A.to(dlt_dtype)
    v = torch.linalg.svd(A)[2][..., -1, :].to(points1.dtype)
    v = torch.where(v[..., 3:] < 0, -v, v)
    return convert_points_from_homogeneous(v, eps)


def triangulate_pairs_ref(points, intrinsics, extrinsics, dist, num_iters=5, eps=1e-8, dlt_dtype=None, pairs=None):
    """project_camera_pairs_to_3d with the v3 >= 0 convention; the keyword arguments other than the defaults are
    mutants (undistortion iterations, dehomogenisation eps, DLT dtype, pair order)."""
    b, v = points.shape[:2]
    eye = torch.eye(3, dtype=points.dtype).expand(b, v, 3, 3)
    und = undistort_points(points, intrinsics, dist, new_K=eye, num_iters=num_iters)
    out = []
    for j1, j2 in pairs or camera_pairs(v):
        p1, p2 = und[:, j1], und[:, j2]
        bad = torch.isnan(p1).any(-1) | torch.isnan(p2).any(-1)
        tri = triangulate_points_v3_nonneg(extrinsics[:, j1], extrinsics[:, j2], torch.where(bad[..., None], 0.0, p1),
                                           torch.where(bad[..., None], 0.0, p2), eps, dlt_dtype)
        out.append(torch.where(bad[..., None], torch.full_like(tri, float("nan")), tri))
    return torch.stack(out, 1)


def project_points_ref(points_3d, intrinsics, extrinsics, dist, mean_over_pairs=False, bbox=None, model_size=None, eps=1e-8,
                       pair_mean_grad_scaled=True):
    """ops.project_points: the optional NaN-propagating mean over the pair axis, PinholeCamera.project (both
    dehomogenisations with ``eps``), distortion where a view's row is not all zero, optional frame_to_model_batch.
    ``eps`` != 1e-8 and ``pair_mean_grad_scaled=False`` (the mean's value with a sum's gradient) are mutants."""
    X = points_3d
    if mean_over_pairs:
        X = points_3d.mean(1)
        if not pair_mean_grad_scaled:
            s = points_3d.sum(1)
            X = X.detach() + (s - s.detach())
    b, v = intrinsics.shape[:2]
    k4 = torch.eye(4, dtype=X.dtype).repeat(b, v, 1, 1)
    k4[:, :, :3, :3] = intrinsics
    e4 = torch.eye(4, dtype=X.dtype).repeat(b, v, 1, 1)
    e4[:, :, :3, :4] = extrinsics
    out = []
    for j in range(v):
        ph = torch.cat([X, torch.ones_like(X[..., :1])], -1) @ (k4[:, j] @ e4[:, j]).transpose(-2, -1)
        p = convert_points_from_homogeneous(convert_points_from_homogeneous(ph, eps), eps)
        has = torch.any(dist[:, j] != 0, dim=-1)
        out.append(torch.where(has[:, None, None], distort_points(p, intrinsics[:, j], dist[:, j]), p))
    out = torch.stack(out, 1)
    return out if bbox is None else frame_to_model_batch(out, bbox, *model_size)


def pairwise_projections_loss_ref(targets, preds):
    """(loss, count): the mean L2 distance between preds (B, pairs, K, 3) and targets (B, K, 3) over the entries with
    neither side NaN, 0 when there is none (the package's rule: nothing to average gives 0 with a zero gradient)."""
    diff = preds - targets[:, None]
    keep = ~torch.isnan(diff).any(-1)
    d = torch.linalg.vector_norm(torch.where(keep[..., None], diff, 0.0), dim=-1)
    n = keep.sum()
    return (d * keep).sum() / n.clamp(min=1), n


def rot_y(a: float) -> torch.Tensor:
    """world -> camera rotation of a camera turned by ``a`` about y: its optical axis is (sin a, 0, cos a)"""
    c, s = math.cos(a), math.sin(a)
    return torch.tensor([[c, 0.0, -s], [0.0, 1.0, 0.0], [s, 0.0, c]], dtype=torch.float64)


def arc_rig(b, v, k, p, seed, step=0.5, depth=2.0, focal=800.0, target=(0.0, 0.0, 0.0), spread=0.15, noise_px=0.5, img=384):
    """V cameras ``step`` radians apart on an arc of radius ``depth`` around ``target``, each looking at it, focal
    lengths ``focal`` +- 5 %, P distortion coefficients ~ N(0, 0.05) (view 1 without), world points ``target`` +
    N(0, spread * depth), keypoints = their projections + ``noise_px`` noise.  Returns float64 copies of fp32 values:
    points (B, V, K, 2), K, E, dist, world points (B, K, 3).  ``step`` / (baseline over depth) and ``target``
    (translation scale) set the DLT's conditioning."""
    gen = torch.Generator().manual_seed(seed)
    T = torch.tensor(target, dtype=torch.float64)
    K = torch.zeros(b, v, 3, 3, dtype=torch.float64)
    E = torch.zeros(b, v, 3, 4, dtype=torch.float64)
    for j in range(v):
        a = (j - (v - 1) / 2) * step
        R = rot_y(a)
        C = T - depth * torch.tensor([math.sin(a), 0.0, math.cos(a)], dtype=torch.float64)
        E[:, j, :, :3], E[:, j, :, 3] = R, -R @ C
        f = focal * (1 + 0.05 * torch.randn(b, generator=gen, dtype=torch.float64))
        K[:, j, 0, 0], K[:, j, 1, 1], K[:, j, 2, 2] = f, f, 1.0
        K[:, j, 0, 2] = img / 2 + torch.randn(b, generator=gen, dtype=torch.float64) * 10
        K[:, j, 1, 2] = img / 2 + torch.randn(b, generator=gen, dtype=torch.float64) * 10
    D = torch.randn(b, v, p, generator=gen, dtype=torch.float64) * 0.05
    if v > 1:
        D[:, 1] = 0.0
    X = T + torch.randn(b, k, 3, generator=gen, dtype=torch.float64) * spread * depth
    K, E, D, X = (f32(t) for t in (K, E, D, X))
    pts = project_points_ref(X, K, E, D) + torch.randn(b, v, k, 2, generator=gen, dtype=torch.float64) * noise_px
    return f32(pts), K, E, D, X


def random_bbox(b, v, seed):
    gen = torch.Generator().manual_seed(seed)
    return f32(torch.cat([torch.rand(b, v, 2, generator=gen) * 40, 300 + torch.rand(b, v, 2, generator=gen) * 100], -1).reshape(b, 4 * v))


def f32(t):
    """float64 tensor of the fp32-rounded values"""
    return t.float().double()


def ulp_perturbed(t: torch.Tensor, rng) -> torch.Tensor:
    """every finite non-zero entry of ``t`` (fp32 values) moved one fp32 ulp up or down at random; zeros stay exact"""
    a = t.float().numpy()
    moved = np.where(rng.random(a.shape) < 0.5, np.nextafter(a, np.float32(np.inf)), np.nextafter(a, np.float32(-np.inf)))
    return torch.from_numpy(np.where(np.isfinite(a) & (a != 0), moved, a).astype(np.float64))


def point_deviation(a, b):
    """per point (last axis) max |a - b|; 0 where both are equal (inf included) or both NaN, inf where only one is NaN"""
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    with np.errstate(invalid="ignore"):
        d = np.where(same, 0.0, np.abs(a - b))
    return np.nan_to_num(d, nan=np.inf).max(-1, initial=0.0)


def sensitivity(fn, inputs: dict, seeds=(1, 2, 3)):
    """per output and point, the largest float64 deviation of ``fn(inputs)`` when every fp32 input is moved by +-1 ulp
    (independent signs per entry, one draw per seed): what the inputs' own precision leaves undetermined."""
    base = fn(inputs)
    dev = {k: np.zeros(v.shape[:-1]) for k, v in base.items()}
    for s in seeds:
        rng = np.random.default_rng(s)
        out = fn({k: None if t is None else ulp_perturbed(t, rng) for k, t in inputs.items()})
        for k in base:
            dev[k] = np.maximum(dev[k], point_deviation(out[k], base[k]))
    return dev


class EdgeCase:
    """One rig and the operations to run on it.  Inputs are float64 tensors holding fp32 values (the kernels get the
    same values in fp32).  ops: "tri" triangulate_pairs(points); "proj" project_points(points3d); "pmean"
    project_points(pairs3d, mean_over_pairs); "reproj" project_points(triangulate_pairs(points), mean_over_pairs);
    "f2m" frame_to_model(points).  The projections are fused with frame -> model when ``bbox`` is given.
    sens: the bar adds 4x the measured input sensitivity.  grad_nonfinite: "zero" (NaN data, zero gradient) or "match"
    (degenerate boxes: non-finite exactly where float64 is).  sign_free: triangulated points at infinity, compared up
    to the sign no convention can fix from a rounding-level v3."""

    INPUTS = ("points", "K", "E", "dist", "bbox", "points3d", "pairs3d")

    def __init__(self, name, ops, K, E, dist, points=None, points3d=None, pairs3d=None, bbox=None, model_size=(256, 256),
                 sens=False, grad_nonfinite="zero", sign_free=False, seed=0):
        self.name, self.ops, self.model_size = name, tuple(ops), model_size
        self.sens, self.grad_nonfinite, self.sign_free = sens, grad_nonfinite, sign_free
        self.x = {"points": points, "K": K, "E": E, "dist": dist, "bbox": bbox, "points3d": points3d, "pairs3d": pairs3d}
        self.x = {k: None if t is None else f32(t) for k, t in self.x.items()}
        b, v = K.shape[:2]
        gen = torch.Generator().manual_seed(1000 + seed)
        rn = lambda *shape: torch.randn(*shape, generator=gen, dtype=torch.float64).float().double()
        self.g = {}
        if points is not None:
            n = points.shape[2]
            self.g.update(tri=rn(b, v * (v - 1) // 2, n, 3), reproj=rn(b, v, n, 2), f2m=rn(b, v, n, 2))
        if points3d is not None:
            self.g["proj"] = rn(b, v, points3d.shape[1], 2)
        if pairs3d is not None:
            self.g["pmean"] = rn(b, v, pairs3d.shape[2], 2)

    def __repr__(self):
        return self.name


def case_outputs(c: EdgeCase, x=None, num_iters=5, eps=1e-8, dlt_dtype=None, pairs=None, dist_perm=None,
                 pair_mean_grad_scaled=True, f2m_keep_offset=False):
    """float64 forward ("<op>") and gradient ("<op>_grad", for the case's seeded upstream gradient) of every op of the
    case, as numpy arrays.  ``x`` replaces the inputs (perturbed copies); the other keywords are mutants."""
    x = c.x if x is None else x
    K, E, D, bb, hw = x["K"], x["E"], x["dist"], x["bbox"], c.model_size
    if dist_perm is not None:
        D = F.pad(D, [0, 12 - D.shape[-1]])[..., list(dist_perm)]
    tri_kw = dict(num_iters=num_iters, eps=eps, dlt_dtype=dlt_dtype, pairs=pairs)
    proj_kw = dict(bbox=bb, model_size=hw, eps=eps, pair_mean_grad_scaled=pair_mean_grad_scaled)
    out = {}
    with torch.enable_grad():
        for op in c.ops:
            inp = x["points3d" if op == "proj" else "pairs3d" if op == "pmean" else "points"].clone().requires_grad_(True)
            if op == "tri":
                y = triangulate_pairs_ref(inp, K, E, D, **tri_kw)
            elif op == "proj":
                y = project_points_ref(inp, K, E, D, **proj_kw)
            elif op == "pmean":
                y = project_points_ref(inp, K, E, D, mean_over_pairs=True, **proj_kw)
            elif op == "reproj":  # the triangulated points reach the projection as fp32, as between the two kernels
                p3 = triangulate_pairs_ref(inp, K, E, D, **tri_kw)
                y = project_points_ref(p3 + (f32(p3) - p3).detach(), K, E, D, mean_over_pairs=True, **proj_kw)
            else:
                y = frame_to_model_batch(inp, bb, *hw)
            if op == "f2m" and f2m_keep_offset:
                g = frame_to_model_batch(c.g[op], bb, *hw)
            else:
                (g,) = torch.autograd.grad(y, inp, c.g[op])
            out[op], out[op + "_grad"] = y.detach().numpy(), g.numpy()
    return out


def case_sensitivity(c: EdgeCase):
    return sensitivity(lambda x: case_outputs(c, x), c.x) if c.sens else None


def bar_failures(c: EdgeCase, got: dict, ref: dict, sens=None):
    """The acceptance bars; returns one message per output that misses them (empty: the case passes).
    Forward: NaN / +-inf exactly where float64 has them; elsewhere, per point, |got - ref| <= 5e-7 max|ref point| (a few
    fp32 ulps of its magnitude).  Gradients: |got - ref| <= 1e-5 |ref| + 1e-6 max|ref|; with grad_nonfinite "zero" the
    gradient is finite and 0 where float64 is NaN (NaN data), with "match" non-finite exactly where float64 is.  With
    ``sens``, each point's bar adds 4x its measured input sensitivity."""
    fails = []
    for key, r in ref.items():
        r = np.asarray(r, np.float64)
        gt = np.asarray(got[key], np.float64)
        if gt.shape != r.shape:
            fails.append(f"{c.name}/{key}: shape {gt.shape} != {r.shape}")
            continue
        grad = key.endswith("_grad")
        fin = np.isfinite(r)
        if not grad or c.grad_nonfinite == "match":
            if not grad and not (np.array_equal(np.isnan(gt), np.isnan(r)) and np.array_equal(gt[np.isinf(r)], r[np.isinf(r)])
                                 and not np.isinf(gt[fin]).any()):
                fails.append(f"{c.name}/{key}: NaN/inf at {np.argwhere(~np.isfinite(gt))[:4].tolist()}, float64 at "
                             f"{np.argwhere(~fin)[:4].tolist()}")
                continue
            if grad and not np.array_equal(np.isfinite(gt), fin):
                fails.append(f"{c.name}/{key}: non-finite at {np.argwhere(~np.isfinite(gt))[:4].tolist()}, float64 at "
                             f"{np.argwhere(~fin)[:4].tolist()}")
                continue
        else:
            if not np.isfinite(gt).all() or (gt[np.isnan(r)] != 0).any():
                fails.append(f"{c.name}/{key}: want finite with 0 where float64 is NaN; got non-finite at "
                             f"{np.argwhere(~np.isfinite(gt))[:4].tolist()}, non-zero at {np.argwhere(np.isnan(r) & (gt != 0))[:4].tolist()}")
                continue
        fin_pt = fin.all(-1)
        with np.errstate(invalid="ignore"):
            err = np.where(fin, np.abs(gt - r), 0.0)
            if grad:
                tol = 1e-5 * np.abs(r) + 1e-6 * (np.abs(r[fin]).max() if fin.any() else 0.0)
            else:
                tol = 5e-7 * np.where(fin, np.abs(r), 0.0).max(-1, initial=0.0)[..., None]
        if sens is not None:
            tol = tol + 4 * sens[key][..., None]
        bad = (err > tol) & fin_pt[..., None]
        if bad.any():
            i = tuple(np.argwhere(bad)[0])
            fails.append(f"{c.name}/{key}: {int(bad.sum())} entries past the bar, first {list(i)}: got {gt[i]!r}, "
                         f"float64 {r[i]!r}, bar {np.broadcast_to(tol, r.shape)[i]:.3e}")
    return fails


# distortion coefficient values for one-at-a-time cases, raised where needed so that each moves the normalised points
# of ``distortion_case`` by >= 1.5e-2 (k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4)
DIST_ALONE = (-0.3, 0.5, 0.05, -0.05, 1.0, 0.3, -0.5, 1.0, 0.08, -0.3, -0.08, 0.3)
DIST_NAMES = ("k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6", "s1", "s2", "s3", "s4")


def distortion_case(p, i):
    """coefficient i alone (P = p) in views 0 and 2 of example 0, view 1 all zero; example 1: view 0 with it, view 1 a
    row of -0.0 (no distortion: dist != 0 is false), view 2 with -0.7 times it.  Points reach r^2 ~ 0.25."""
    pts, K, E, _, X = arc_rig(2, 3, 7, p, seed=200 + 12 * p + i, spread=0.18, step=0.6)
    D = torch.zeros(2, 3, p, dtype=torch.float64)
    D[0, 0, i] = D[0, 2, i] = D[1, 0, i] = 1.0
    D[1, 2, i] = -0.7
    moved = (project_points_ref(X, K, E, DIST_ALONE[i] * D) - project_points_ref(X, K, E, 0 * D)).abs() / K[:, :, None, 0:1, 0]
    D = f32(D * DIST_ALONE[i] * max(1.0, 1.5e-2 / float(moved.max())))
    D[1, 1] = -0.0
    pts = f32(project_points_ref(X, K, E, D) + 0.3 * torch.randn(pts.shape, generator=torch.Generator().manual_seed(i), dtype=torch.float64))
    return EdgeCase(f"dist_P{p}_{DIST_NAMES[i]}", ("tri", "proj", "reproj"), K, E, D, points=pts, points3d=X,
                    bbox=random_bbox(2, 3, p + i), seed=i)


def divergence_case():
    """k1 = -0.5: x (1 + k1 r^2) turns over at r^2 = 2/3 (distorted radius 0.544); keypoints at distorted radii 0.55 to
    0.7 have no undistorted preimage and the 5 fixed-point iterations run away (finitely).  Projections with the
    same coefficients of points spread along x."""
    _, K, E, _, X = arc_rig(2, 2, 8, 5, seed=300, step=0.5)
    D = torch.zeros(2, 2, 5, dtype=torch.float64)
    D[..., 0] = -0.5
    D[1, 1, 1] = 0.05
    gen = torch.Generator().manual_seed(301)
    ang = torch.rand(2, 2, 8, generator=gen, dtype=torch.float64) * 2 * math.pi
    rad = torch.linspace(0.3, 0.7, 8, dtype=torch.float64)  # normalised distorted radius, 0.55 .. 0.7 past the turn-over
    fx, cx, cy = K[..., 0, 0, None], K[..., 0, 2, None], K[..., 1, 2, None]
    pts = torch.stack([cx + fx * rad * torch.cos(ang), cy + fx * rad * torch.sin(ang)], -1)
    X = X.clone()
    X[..., 0] = torch.linspace(-0.3, 0.45, 8, dtype=torch.float64) * 2.0
    return EdgeCase("distortion_divergence", ("tri", "proj", "reproj"), K, E, D, points=f32(pts), points3d=f32(X), sens=True, seed=7)


def conditioning_case(ratio, focal, tscale):
    """3 views, neighbouring cameras ``ratio`` (baseline over depth) apart, focal ``focal``, the whole rig ``tscale``
    times larger and moved by ``tscale`` (translations in mm); 3e-4 rad of keypoint noise."""
    pts, K, E, D, X = arc_rig(2, 3, 9, 5, seed=400, step=ratio, depth=2.0 * tscale, focal=focal, target=(0.7 * tscale, -0.4 * tscale, 0.5 * tscale),
                              noise_px=3e-4 * focal)
    return EdgeCase(f"cond_b{ratio:g}_f{focal:g}_t{tscale:g}", ("tri", "proj", "reproj"), K, E, D, points=pts, points3d=X, sens=True, seed=8)


def fly_case(g):
    """the reference fixture's anipose-fly calibration (focal lengths up to 1e5, k1 = -1906), from cameras.npz"""
    t = lambda k: torch.from_numpy(g[f"fly_in_{k}"]).double()
    return EdgeCase("cond_fly", ("tri", "proj", "reproj"), t("K"), t("E"), t("dist"), points=t("points"), points3d=t("points3d"),
                    bbox=t("bbox"), model_size=tuple(int(v) for v in g["fly_in_model_hw"]), sens=True, seed=9)


def _parallel_rig(b, baseline=1.0, focal=800.0):
    """two cameras with identity rotation, principal point at the pixel origin, the second ``baseline`` along x"""
    K = torch.zeros(b, 2, 3, 3, dtype=torch.float64)
    K[..., 0, 0] = K[..., 1, 1] = focal
    K[..., 2, 2] = 1.0
    E = torch.zeros(b, 2, 3, 4, dtype=torch.float64)
    E[..., :3] = torch.eye(3, dtype=torch.float64)
    E[:, 1, 0, 3] = -baseline
    return K, E, torch.zeros(b, 2, 4, dtype=torch.float64)


def far_points_case():
    """Triangulated points at depths 1e2 .. 1e9 near camera 0's optical axis (|v3| ~ 1 / depth through 1e-2 .. 1e-9,
    both sides of the 1e-8 switch of the dehomogenisation).  The principal points sit at the pixel origin, so the fp32
    keypoints keep the tiny disparities: the depth stays determined by the inputs."""
    depths = torch.tensor([1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 5e7, 9e7, 1.1e8, 1e9], dtype=torch.float64)
    K, E, D = _parallel_rig(1)
    gen = torch.Generator().manual_seed(500)
    X = torch.stack([torch.randn(10, generator=gen, dtype=torch.float64) * 0.3, torch.randn(10, generator=gen, dtype=torch.float64) * 0.3, depths], -1)[None]
    X = f32(X)
    pts = project_points_ref(X, K, E, D)
    c = EdgeCase("dehomog_far_points", ("tri",), K, E, D, points=f32(pts), sens=True, seed=10)
    c.v3 = 1 / torch.sqrt(1 + (X**2).sum(-1))  # of the unit homogeneous vector the DLT solves for
    return c


def parallel_rays_case():
    """the same pixel in two cameras with identity rotations: exactly parallel rays, v3 = 0 up to rounding; the result is
    the ray direction (kornia's eps leaves v[:3] undivided), with a sign rounding decides"""
    K, E, D = _parallel_rig(2)
    gen = torch.Generator().manual_seed(501)
    uv = f32(torch.randn(2, 1, 6, 2, generator=gen, dtype=torch.float64) * 200).expand(2, 2, 6, 2).clone()
    return EdgeCase("dehomog_parallel_rays", ("tri",), K, E, D, points=uv, sign_free=True, seed=11)


def principal_plane_case():
    """world points with camera-0 depth c2 exactly 0, within +-1e-8 (scale 1), just past it (scale 1 / (c2 + 1e-8),
    up to 5e7) and negative (behind the camera, mirrored); view 1 is an ordinary distorted ring camera"""
    _, K, E, _, _ = arc_rig(2, 2, 1, 5, seed=502, step=0.8)
    E[:, 0] = 0.0
    E[:, 0, :, :3] = torch.tensor([[0.6, 0.8, 0.0], [-0.8, 0.6, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    D = torch.zeros(2, 2, 5, dtype=torch.float64)
    D[:, 1] = torch.tensor([-0.1, 0.02, 0.001, -0.002, 0.0], dtype=torch.float64)
    z = torch.tensor([0.0, 4e-9, -4e-9, 9e-9, -9e-9, 1.5e-8, 3e-8, -3e-8, 1e-6, -0.5, -2.0], dtype=torch.float64)
    gen = torch.Generator().manual_seed(503)
    X = torch.cat([torch.randn(2, len(z), 2, generator=gen, dtype=torch.float64) * 0.3, z.expand(2, -1)[..., None]], -1)
    return EdgeCase("dehomog_principal_plane", ("proj",), K, E, D, points3d=f32(X), sens=True, seed=12)


def baseline_keypoint_case():
    """cameras 0 (centre (0, 0, -2), looking along +z) and 1 (centre (-2, 0, 0), looking along +x) and a keypoint on
    their baseline, at each one's epipole: normalised (-1, 0) and (1, 0), exact in fp32.  The DLT matrix has rank 2
    exactly, lambda_min is double and the SVD's gradient is infinite; keypoint 1 is an ordinary one."""
    K = torch.zeros(1, 2, 3, 3, dtype=torch.float64)
    K[..., 0, 0] = K[..., 1, 1] = 800.0
    K[..., 0, 2] = K[..., 1, 2] = 192.0
    K[..., 2, 2] = 1.0
    E = torch.tensor([[[1.0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 2]], [[0.0, 0, -1, 0], [0, 1, 0, 0], [1, 0, 0, 2]]], dtype=torch.float64)[None]
    X = torch.tensor([[[-1.0, 0.0, -1.0], [-1.3, 0.2, -0.6]]], dtype=torch.float64)  # keypoint 0 on the baseline
    pts = f32(project_points_ref(X, K, E, torch.zeros(1, 2, 4, dtype=torch.float64)))
    assert pts[0, 0, 0].tolist() == [-608.0, 192.0] and pts[0, 1, 0].tolist() == [992.0, 192.0]
    return EdgeCase("degenerate_baseline_keypoint", ("tri",), K, E, torch.zeros(1, 2, 4, dtype=torch.float64), points=pts, seed=13)


def shape_case(v, k, b=2, p=8):
    """ordinary cameras on an arc (neighbours min(0.6, 0.75 pi / (V - 1)) apart), V views, K keypoints, batch b"""
    pts, K, E, D, X = arc_rig(b, v, k, p, seed=600 + v * 64 + k, step=min(0.6, 0.75 * math.pi / max(v - 1, 1)))
    pairs3d = triangulate_pairs_ref(pts, K, E, D) if v > 1 else None
    return EdgeCase(f"shape_B{b}_V{v}_K{k}", ("tri", "proj", "pmean", "reproj", "f2m"), K, E, D, points=pts, points3d=X,
                    pairs3d=pairs3d, bbox=random_bbox(b, v, v + k), seed=14)


def nan_case():
    """NaN keypoints: x only, y only, one view, every view; NaN world points: x only, every coordinate; a pair mean with
    one NaN pair (the mean, hence every view of that keypoint, is NaN and every pair gets a zero gradient)"""
    pts, K, E, D, X = arc_rig(2, 4, 6, 5, seed=700)
    pairs3d = triangulate_pairs_ref(pts, K, E, D).clone()
    nan = float("nan")
    pts[0, 0, 0, 0] = nan
    pts[0, 1, 1, 1] = nan
    pts[0, 2, 2] = nan
    pts[1, :, 3] = nan
    X[0, 0, 0] = nan
    X[1, 2] = nan
    pairs3d[0, 2, 4] = nan
    pairs3d[1, :, 5, 1] = nan
    return EdgeCase("nan", ("tri", "proj", "pmean", "reproj", "f2m"), K, E, D, points=pts, points3d=X, pairs3d=pairs3d,
                    bbox=random_bbox(2, 4, 7), seed=15)


def bbox_case():
    """box sizes 0, negative and infinite.  Example 0 (finite gradients): view 1 h < 0, view 2 w = inf (model x = 0, zero
    gradient).  Example 1: view 1 w = 0 with one keypoint exactly at its box corner (0 / 0 = NaN), view 2 h = 0, and
    negative w and h in view 0."""
    pts, K, E, D, X = arc_rig(2, 3, 5, 5, seed=800)
    bbox = random_bbox(2, 3, 801).reshape(2, 3, 4)
    bbox[0, 1, 2] = -bbox[0, 1, 2]
    bbox[0, 2, 3] = float("inf")
    bbox[1, 0, 2:] = -bbox[1, 0, 2:]
    bbox[1, 1, 3] = 0.0
    bbox[1, 2, 2] = 0.0
    pts[1, 1, 2] = bbox[1, 1, :2]
    pairs3d = triangulate_pairs_ref(pts, K, E, D)
    return EdgeCase("bbox_degenerate", ("proj", "pmean", "reproj", "f2m"), K, E, D, points=pts, points3d=X, pairs3d=pairs3d,
                    bbox=bbox.reshape(2, 12), grad_nonfinite="match", seed=16)


def edge_cases(golden=None):
    """every case compared with float64 under the bars, by name (not the shape sweep, nor the degenerate DLT, which
    has no float64 answer to compare with)"""
    cases = [distortion_case(p, i) for p in (4, 5, 8, 12) for i in range(p)]
    cases += [divergence_case()]
    cases += [conditioning_case(r, f, t) for r in (1.0, 1e-1, 1e-2, 1e-3) for f in (1e2, 1e5) for t in (1.0, 1e3)]
    if golden is not None:
        cases.append(fly_case(golden))
    cases += [far_points_case(), parallel_rays_case(), principal_plane_case(), nan_case(), bbox_case()]
    return {c.name: c for c in cases}


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
