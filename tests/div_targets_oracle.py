"""float64 restatement of the fused Gaussian-target + KL / JS heatmap losses.  TEST INFRASTRUCTURE ONLY.

Extends ``targets_oracle.py`` (the target rule, whose planes it reuses) with HeatmapKLLoss and HeatmapJSLoss
(lightning_pose/losses/losses.py:338-423): both operands get 1e-10 (:375-376, :420-421); a plane is kept when its target
is not all zero (NaN planes are kept, so the loss is NaN); loss = sum over kept planes of the plane's sum of terms /
n_kept (NaN when nothing is kept); the gradient is the per-pixel derivative / n_kept on kept planes, 0 elsewhere.

Also the error scales the tests accept against.  A term is a difference of logarithms times an operand, so fp32 can
be held to a fraction of the operands' magnitudes (|t| (|log t| + |log p| + 1) for KL), not of the term's value, which
cancels where t is close to p.
"""
from __future__ import annotations

import torch

import targets_oracle as TO

F64 = torch.float64
EPS = 1e-10


def _terms(kind, t, p):
    """(per-pixel terms, d term / d p, magnitude of the term's rounding, magnitude of the gradient's rounding)."""
    tt, pp = t + EPS, p + EPS
    lt, lp = torch.log(tt), torch.log(pp)
    if kind == "kl":
        term = tt * (lt - lp)
        grad = -tt / pp
        mag = tt * (lt.abs() + lp.abs() + 1.0)
        gmag = grad.abs()
    else:
        m = 0.5 * (tt + pp)
        lm = torch.log(m)
        term = 0.5 * (tt * (lt - lm) + pp * (lp - lm))
        grad = 0.5 * (lp - lm)
        mag = 0.5 * (tt * (lt.abs() + lm.abs() + 1.0) + pp * (lp.abs() + lm.abs() + 1.0))
        gmag = 0.5 * (lp.abs() + lm.abs())
    return term, grad, mag, gmag


def div_from_keypoints(kind, kp, preds, height, width, sigma=1.25, visibility=None, targets=None):
    """Fused target + HeatmapKLLoss / HeatmapJSLoss in float64: (loss, d loss / d preds, loss error scale, (B, K)
    gradient error scale per plane).  ``targets`` overrides the planes (dense targets given as they are)."""
    oh, ow = preds.shape[-2:]
    t = TO.target_planes(kp, height, width, oh, ow, sigma, visibility)[0] if targets is None else targets.to(F64)
    keep = ~(t == 0).all(-1).all(-1)
    p = preds.to(F64)
    term, grad, mag, gmag = _terms(kind, t, p)
    n_kept = int(keep.sum())
    zero = torch.zeros((), dtype=F64, device=p.device)
    kept = keep[..., None, None]
    if n_kept == 0:
        nan = torch.tensor(float("nan"), dtype=F64)
        return nan, torch.zeros_like(p), torch.tensor(0.0, dtype=F64), torch.zeros(keep.shape, dtype=F64)
    loss = torch.where(kept, term, zero).sum() / n_kept
    scale = torch.where(kept, mag, zero).nan_to_num(0.0).sum() / n_kept
    g = torch.where(kept, grad, zero) / n_kept
    gscale = torch.where(kept, gmag, zero).nan_to_num(0.0).flatten(-2).amax(-1) / n_kept
    return loss, g, scale, gscale


def check_loss(got, ref, scale, rel=1e-5, case=""):
    """NaN exactly when the reference is NaN; otherwise |got - ref| <= rel * scale.  Returns the ratio."""
    got, ref = float(got), float(ref)
    if ref != ref:
        assert got != got, f"{case}: loss {got}, want NaN"
        return 0.0
    r = abs(got - ref) / (rel * float(scale))
    assert r <= 1.0, f"{case}: loss {got} vs {ref}: {r:.3g} x allowed"
    return r
