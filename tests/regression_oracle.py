"""float64 restatement of the reference's regression model pieces (lightning_pose/models/heads/regression.py,
losses/losses.py:857-996, data/utils.py:142-188), checked against the reference's own outputs in
tests/golden/regression.npz (scripts/gen_regression_golden.py) and used by the GPU tests as their reference."""
from __future__ import annotations

import numpy as np


def head_forward(features, weight, bias):
    """(B, C, h, w) -> mean over the pixels -> linear: the reference's avgpool + LinearRegressionHead."""
    f = np.asarray(features, dtype=np.float64)
    pooled = f.reshape(f.shape[0], f.shape[1], -1).mean(-1)
    return pooled @ np.asarray(weight, np.float64).T + np.asarray(bias, np.float64), pooled


def head_backward(grad_out, pooled, weight, feat_shape):
    """(d features broadcast over the pixels, d weight, d bias)."""
    g = np.asarray(grad_out, np.float64)
    b, c, h, w = feat_shape
    dpool = g @ np.asarray(weight, np.float64) / (h * w)
    return np.broadcast_to(dpool[:, :, None, None], feat_shape), g.T @ pooled, g.sum(0)


def regression_mse(targets, preds):
    """RegressionMSELoss: mean of (t - p)^2 over the non-NaN targets; NaN when there is none (torch.mean of empty)."""
    t, p = np.asarray(targets, np.float64).ravel(), np.asarray(preds, np.float64).ravel()
    keep = ~np.isnan(t)
    return float(np.mean((t[keep] - p[keep]) ** 2)) if keep.any() else float("nan"), int(keep.sum())


def regression_rmse(targets, preds):
    """RegressionRMSELoss: the kept entries compacted in order, then paired as (x, y) by reshape(-1, 2), mean over the
    pairs of sqrt(pair mean).  NaN when nothing is kept; an odd count (where the reference's reshape raises) is NaN."""
    t, p = np.asarray(targets, np.float64).ravel(), np.asarray(preds, np.float64).ravel()
    keep = ~np.isnan(t)
    d2 = (t[keep] - p[keep]) ** 2
    if d2.size == 0 or d2.size % 2:
        return float("nan")
    return float(np.mean(np.sqrt(d2.reshape(-1, 2).mean(1))))


def undo_affine(keypoints, transform):
    """(T, K, 2) keypoints, (2, 3) or (T, 2, 3) matrices [A | t] -> A^-1 (p - t)."""
    kp = np.asarray(keypoints, np.float64)
    m = np.asarray(transform, np.float64)
    m = np.broadcast_to(m, (kp.shape[0], 2, 3)) if m.ndim == 2 else m
    a_inv = np.linalg.inv(m[:, :, :2])
    return np.einsum("tij,tkj->tki", a_inv, kp - m[:, None, :, 2])
