"""float64 restatement of the Gaussian-target rule and of what is built on it.  TEST INFRASTRUCTURE ONLY.

The rule (lightning_pose/data/heatmaps.py:37-87): a keypoint in image pixels is scaled onto the heatmap grid in fp32, as
the reference's in-place multiply of an fp32 tensor by a Python float does; it is "bad" when its grid x is NaN or either
coordinate lies outside [-1, size + 1] (NaN comparisons are false, so a NaN y alone is not bad); both coordinates are
clamped to that range (NaN stays NaN); the plane is the normalised Gaussian exp(-((c - x)^2 + (r - y)^2) / (2 sigma^2)).
Without a visibility a bad keypoint gives a zero plane; with one, 0 gives zeros, 1 the uniform plane 1 / (h w), 2 zeros
when bad, and every other value (3, -1, ...) keeps the clamped Gaussian, NaN included.

Classification uses the fp32 grid coordinates; everything after it is float64, on the device of the inputs.  Also here:
the fused target + MSE loss and its gradient, the labeled-frame out-of-frame mask (datasets.py:496-508), the windowed
evaluation (heatmaps.py:90-142), the edge batch the tests share, and the acceptance rules of
``test_targets_edges_gpu.py`` (``test_targets_oracle.py`` shows on the CPU that they reject plausible wrong rules).
"""
from __future__ import annotations

import math

import numpy as np
import torch

F64 = torch.float64
ZERO, UNIFORM, GAUSS, NAN = 0, 1, 2, 3  # plane patterns (NAN: a Gaussian plane whose centre is NaN)
VIS_VALUES = (0, 1, 2, 3, -1)  # every visibility the edge batch carries
# (image height, width, heatmap height, width) of the edge tests: a power-of-two ratio square, a power-of-two ratio
# non-square, and ratios that are not powers of two with a grid wider than one 128-thread pass
CONFIGS = [(384, 384, 96, 96), (256, 320, 64, 80), (406, 612, 128, 192)]
SIGMAS = (0.5, 1.25, 3.0)


# ------------------------------------------------------------------------------------------------
# the rule
# ------------------------------------------------------------------------------------------------
def grid_scale(height, width, oh, ow) -> tuple[np.float32, np.float32]:
    """(sx, sy) = fp32(ow / width), fp32(oh / height)."""
    return np.float32(ow / width), np.float32(oh / height)


def grid_coords(kp, height, width, oh, ow, swap_scale=False):
    """fp32 grid coordinates (x, y) of image-pixel keypoints kp (..., 2): one correctly rounded fp32 product each."""
    sx, sy = grid_scale(height, width, oh, ow)
    if swap_scale:
        sx, sy = sy, sx
    kp = kp.detach().float()
    return kp[..., 0] * torch.tensor(sx, device=kp.device), kp[..., 1] * torch.tensor(sy, device=kp.device)


def classify(x, y, vis, oh, ow, clamp_inclusive=False, nan_y=False):
    """Target mode (ZERO / UNIFORM / GAUSS) per plane from the fp32 grid coordinates.  ``clamp_inclusive`` and ``nan_y``
    are wrong rules (a keypoint on the clamp bound counted bad; a NaN y counted bad) for the plausible-bug check."""
    if clamp_inclusive:
        outside = lambda v, hi: (v <= -1) | (v >= hi)  # noqa: E731
    else:
        outside = lambda v, hi: (v < -1) | (v > hi)  # noqa: E731
    bad = torch.isnan(x) | outside(x, ow + 1) | outside(y, oh + 1)
    if nan_y:
        bad = bad | torch.isnan(y)
    if vis is None:
        return torch.where(bad, ZERO, GAUSS)
    vis = vis.to(x.device)
    mode = torch.full_like(x, GAUSS, dtype=torch.int64)
    mode[vis == 0] = ZERO
    mode[vis == 1] = UNIFORM
    mode[(vis == 2) & bad] = ZERO
    return mode


def _gaussians(xc, yc, oh, ow, two_s2):
    """Normalised Gaussian planes (n, oh, ow) centred at the float64 clamped coordinates (n,)."""
    cols = torch.arange(ow, dtype=F64, device=xc.device)
    rows = torch.arange(oh, dtype=F64, device=xc.device)
    ex = torch.exp(-((cols[None, :] - xc[:, None]) ** 2) / two_s2)
    ey = torch.exp(-((rows[None, :] - yc[:, None]) ** 2) / two_s2)
    return ey[:, :, None] * ex[:, None, :] / (ex.sum(1) * ey.sum(1))[:, None, None]


def target_planes(kp, height, width, oh, ow, sigma=1.25, visibility=None, keep_gradients=False, gout=None,
                  clamp_inclusive=False, nan_y=False, sigma_as_two_s2=False, swap_scale=False):
    """generate_heatmaps: (planes (B, K, oh, ow) float64, mode (B, K)); with ``keep_gradients`` also d sum(planes * gout)
    / d kp (B, K, 2) through autograd.  Zero and uniform planes do not depend on the keypoint: their gradient is 0 (the
    reference's autograd would put 0 * NaN there for a NaN keypoint).  The clamp passes the gradient on its bounds, as
    torch.clamp does.  The last four flags are wrong rules for the plausible-bug check."""
    b, k = kp.shape[:2]
    x, y = grid_coords(kp, height, width, oh, ow, swap_scale)
    mode = classify(x, y, visibility, oh, ow, clamp_inclusive, nan_y).reshape(-1)
    two_s2 = float(sigma) if sigma_as_two_s2 else 2.0 * float(sigma) ** 2
    n = oh * ow
    planes = torch.zeros((b * k, oh, ow), dtype=F64, device=kp.device)
    planes[mode == UNIFORM] = 1.0 / n
    gi = torch.nonzero(mode == GAUSS).reshape(-1)
    xl = x.reshape(-1)[gi].double().requires_grad_(keep_gradients)
    yl = y.reshape(-1)[gi].double().requires_grad_(keep_gradients)
    with torch.set_grad_enabled(keep_gradients):
        g = _gaussians(xl.clamp(-1, ow + 1), yl.clamp(-1, oh + 1), oh, ow, two_s2)
    planes[gi] = g.detach()
    planes = planes.reshape(b, k, oh, ow)
    mode = mode.reshape(b, k)
    if not keep_gradients:
        return planes, mode
    gk = torch.zeros((b * k, 2), dtype=F64, device=kp.device)
    if gi.numel():
        (g * gout.reshape(b * k, oh, ow)[gi].double()).sum().backward()
        sx, sy = grid_scale(height, width, oh, ow)
        gk[gi, 0] = xl.grad * float(sx)
        gk[gi, 1] = yl.grad * float(sy)
    return planes, mode, gk.reshape(b, k, 2)


def plane_pattern(planes):
    """(B, K) pattern of planes: ZERO (all 0), NAN (any NaN), UNIFORM (all equal and nonzero), GAUSS otherwise."""
    p = planes.reshape(planes.shape[0], planes.shape[1], -1)
    pat = torch.full(p.shape[:2], GAUSS, dtype=torch.int64, device=p.device)
    pat[(p == p[..., :1]).all(-1)] = UNIFORM
    pat[(p == 0).all(-1)] = ZERO
    pat[torch.isnan(p).any(-1)] = NAN
    return pat


def mse_from_keypoints(kp, preds, height, width, sigma=1.25, visibility=None):
    """Fused target + HeatmapMSELoss: (loss, d loss / d preds) in float64.  A plane is kept when its target is not all
    zero (NaN planes are kept); loss = sum over kept planes of sum (t - p)^2 / n_kept (NaN when nothing is kept),
    gradient 2 (p - t) / n_kept on kept planes and 0 on the others."""
    oh, ow = preds.shape[-2:]
    t, _ = target_planes(kp, height, width, oh, ow, sigma, visibility)
    keep = ~(t == 0).all(-1).all(-1)
    p = preds.double()
    n_kept = int(keep.sum())
    d = torch.where(keep[..., None, None], p - t, torch.zeros((), dtype=F64, device=p.device))
    loss = (d * d).sum() / n_kept if n_kept else torch.tensor(float("nan"), dtype=F64)
    grad = 2.0 * d / n_kept if n_kept else torch.zeros_like(p)
    return loss, grad


def mask_oob(kp, height, width):
    """Labeled keypoints outside [0, width) x [0, height) -> NaN in both coordinates; fp32 comparisons, NaN compares
    false (so NaN in one coordinate alone is kept)."""
    kp = kp.detach().float()
    x, y = kp[..., 0], kp[..., 1]
    oob = (x < 0) | (y < 0) | (x >= np.float32(width)) | (y >= np.float32(height))
    out = kp.clone()
    out[oob] = float("nan")
    return out


def window_radius(sigma=1.25, num_stds=2) -> int:
    return int(math.floor(sigma * num_stds))


def window_sum(heatmaps, locs, radius):
    """Sum of the (2r+1)^2 window of each plane around (trunc(y), trunc(x)) of the fp32 locations (truncation toward
    zero), the plane zero-padded by r, in float64."""
    b, k, h, w = heatmaps.shape
    pad = torch.zeros((b * k, h + 2 * radius, w + 2 * radius), dtype=F64, device=heatmaps.device)
    pad[:, radius:radius + h, radius:radius + w] = heatmaps.reshape(b * k, h, w).double()
    loc = locs.detach().float().reshape(b * k, 2)
    cx = torch.trunc(loc[:, 0]).long() + radius
    cy = torch.trunc(loc[:, 1]).long() + radius
    out = torch.zeros(b * k, dtype=F64, device=heatmaps.device)
    idx = torch.arange(b * k, device=heatmaps.device)
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            out += pad[idx, cy + dy, cx + dx]
    return out.reshape(b, k)


# ------------------------------------------------------------------------------------------------
# the edge batch
# ------------------------------------------------------------------------------------------------
def _image_coords_for(target: float, s: np.float32) -> dict:
    """fp32 image coordinates whose fp32 product with s is exactly ``target`` ("on"), the nearest product above it and
    the nearest below it."""
    x0 = np.float32(target / float(s))
    cands = [x0]
    lo = hi = x0
    for _ in range(64):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        cands += [lo, hi]
    prods = {c: np.float32(c * s) for c in cands}
    on = [c for c in cands if prods[c] == np.float32(target)]
    assert on, f"no fp32 coordinate lands exactly on {target} with scale {s}"
    above = min((c for c in cands if prods[c] > target), key=lambda c: prods[c])
    below = max((c for c in cands if prods[c] < target), key=lambda c: prods[c])
    return {"on": float(on[0]), "above": float(above), "below": float(below)}


def edge_rows(height, width, oh, ow) -> torch.Tensor:
    """(n, 2) fp32 image-pixel keypoints at the rule's edges for this (image, heatmap) pair: each coordinate exactly on
    -1 and size + 1 after scaling and the nearest fp32 product on either side, two corners on the bounds, NaN in x, in y
    and in both, +-inf in each coordinate, -0.0, and three interior points."""
    sx, sy = grid_scale(height, width, oh, ow)
    mid_x, mid_y = 0.43 * width, 0.57 * height
    rows = []
    ex = {t: _image_coords_for(t, sx) for t in (-1.0, ow + 1.0)}
    ey = {t: _image_coords_for(t, sy) for t in (-1.0, oh + 1.0)}
    for t in ex:
        rows += [(v, mid_y) for v in ex[t].values()]
    for t in ey:
        rows += [(mid_x, v) for v in ey[t].values()]
    rows += [(ex[-1.0]["on"], ey[oh + 1.0]["on"]), (ex[ow + 1.0]["on"], ey[-1.0]["on"])]
    nan, inf = float("nan"), float("inf")
    rows += [(nan, mid_y), (mid_x, nan), (nan, nan)]
    rows += [(inf, mid_y), (-inf, mid_y), (mid_x, inf), (mid_x, -inf)]
    rows += [(-0.0, mid_y), (mid_x, -0.0), (-0.0, -0.0)]
    rows += [(0.131 * width, 0.872 * height), (0.5 * width + 0.25, 0.5 * height - 0.25), (0.97 * width, 0.03 * height)]
    return torch.tensor(rows, dtype=torch.float32)


def edge_batch(height, width, oh, ow, min_planes=0):
    """(kp (B, n, 2), vis (B, n) int32): the edge rows once for every visibility in VIS_VALUES, then repeated until the
    batch has at least ``min_planes`` planes (the repeats carry the same values)."""
    rows = edge_rows(height, width, oh, ow)
    n = rows.shape[0]
    per = len(VIS_VALUES)
    reps = max(1, -(-min_planes // (per * n)))
    kp = rows[None].repeat(per * reps, 1, 1)
    vis = torch.tensor(VIS_VALUES, dtype=torch.int32).repeat(reps)[:, None].expand(-1, n).contiguous()
    return kp, vis


# ------------------------------------------------------------------------------------------------
# acceptance rules (error / allowed ratios are returned so the tests can report their headroom)
# ------------------------------------------------------------------------------------------------
def check_planes(got, ref, case=""):
    """Same pattern per plane; Gaussian planes within 1e-6 + 1e-5 max(plane); uniform ones within 1e-6 of 1 / (h w).
    Returns the worst error / allowed ratio."""
    got, ref = got.double(), ref.to(got.device)
    pg, pr = plane_pattern(got), plane_pattern(ref)
    bad = torch.nonzero(pg != pr)
    assert bad.numel() == 0, f"{case}: plane patterns differ at {bad[:8].tolist()} (got {pg[pg != pr][:8].tolist()}, " \
                             f"want {pr[pg != pr][:8].tolist()})"
    fin = (pr == GAUSS) | (pr == UNIFORM)
    if not bool(fin.any()):
        return 0.0
    g, r = got[fin].flatten(1), ref[fin].flatten(1)
    allowed = 1e-6 + 1e-5 * r.abs().amax(1, keepdim=True)
    ratio = float(((g - r).abs() / allowed).max())
    assert ratio <= 1.0, f"{case}: plane error {ratio:.3g} x allowed"
    return ratio


def keep_gradients_scale(kp, height, width, oh, ow, sigma, visibility, gout):
    """(B, K) error scale of the keep_gradients gradient: per keypoint, the larger over x and y of the sum of the
    magnitudes of its per-pixel terms |gout g (c - xbar)| / sigma^2 * sx (0 on a clamped coordinate and on zero / uniform
    planes, NaN on NaN planes).  The gradient is a sum of signed terms that cancel, so fp32 can only be held to a
    fraction of this sum, not of the sum's value."""
    planes, mode = target_planes(kp, height, width, oh, ow, sigma, visibility)
    x, y = grid_coords(kp, height, width, oh, ow)
    sx, sy = grid_scale(height, width, oh, ow)
    cols = torch.arange(ow, dtype=F64, device=planes.device)
    rows = torch.arange(oh, dtype=F64, device=planes.device)[:, None]
    pg = (planes * gout.double()).abs()
    lx = (pg * (cols - (planes * cols).sum((-1, -2))[..., None, None]).abs()).sum((-1, -2)) / sigma**2 * float(sx)
    ly = (pg * (rows - (planes * rows).sum((-1, -2))[..., None, None]).abs()).sum((-1, -2)) / sigma**2 * float(sy)
    gauss = mode == GAUSS
    lx = torch.where(gauss & (x >= -1) & (x <= ow + 1), lx, 0.0)
    ly = torch.where(gauss & (y >= -1) & (y <= oh + 1), ly, 0.0)
    return torch.maximum(lx, ly)


def check_relative_per_plane(got, ref, rel=1e-5, case="", scale=None):
    """NaN where the reference is NaN and nowhere else; elsewhere |got - ref| <= rel * scale, with scale the largest
    |ref| over the plane (the last two dims) unless given (one value per plane), and exactly 0 where the scale is 0.
    Returns the worst ratio."""
    got, ref = got.double(), ref.to(got.device).double()
    nan_g, nan_r = torch.isnan(got), torch.isnan(ref)
    assert torch.equal(nan_g, nan_r), f"{case}: NaN pattern differs at {torch.nonzero(nan_g != nan_r)[:8].tolist()}"
    g = torch.where(nan_r, 0.0, got).flatten(-2)
    r = torch.where(nan_r, 0.0, ref).flatten(-2)
    if scale is None:
        scale = r.abs().amax(-1, keepdim=True)
    else:
        scale = torch.nan_to_num(scale.to(got.device).double(), nan=0.0)[..., None]
    err = (g - r).abs()
    zero = (scale == 0).expand_as(err)
    assert not bool((err[zero] != 0).any()), f"{case}: nonzero where the reference is exactly 0"
    ratio = err / (rel * torch.where(scale == 0, 1.0, scale))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    assert worst <= 1.0, f"{case}: error {worst:.3g} x allowed"
    return worst
