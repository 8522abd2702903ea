"""The unsupervised loss stack at its edges against float64: the temporal loss and the single- and multi-view PCA losses
(``unsup_losses_fwd_kernel`` / ``unsup_losses_bwd_kernel``) and the temporal heatmap loss (``temporal_heatmap_*_kernel``),
all in csrc/losses.cu.

Every case compares the per-clip values ``out[:, :3]`` of ``ops.unsup_losses`` (or the scalar of
``ops.temporal_heatmap_loss``) and the gradient of a randomly weighted sum of them with float64 autograd through the
references of tests/scale_oracle.py and oracle/lp_oracle.py.  The references run on the CPU: ``torch.quantile``'s
backward sends a tied median's gradient to the positions a stable sort gives, which is what the CPU sort does and what
``median_interp``'s tie-break by position reproduces.

Tolerances (the rule of tests/test_scale_gpu.py): values 1e-5 abs + 1e-4 rel, the fp32 accumulation of at most a few
thousand terms of the kernels; gradients 1e-6 * max|g| abs + 1e-3 rel, where the fp32 1 / norm and the mixing by the
PCA components are the largest error.  The temporal KL gradient takes the max per plane, because -p / q at a zero
pixel is 1e8 times its neighbours'.

NaN follows float64 autograd, checked on the CPU with the references:
- Forward: a NaN term makes its loss NaN (``F.relu(NaN)`` is NaN); ``torch.quantile`` is NaN for a frame with a NaN,
  so median centring spreads it over the frame.  A confidence-masked pair is 0 in the forward even when its distance is
  NaN (``masked_fill``), and a NaN confidence does not mask (``NaN < thr`` is false).
- Temporal backward: a pair whose distance is NaN gives NaN in both coordinates of both of its keypoints, whether the
  pair is masked, rectified away or not: the norm's backward is ``diff * (g / norm)``, and ``0 * NaN`` is NaN.
- PCA backward: ``relu`` passes the gradient of a NaN residual norm, so both coordinates of that pair are NaN; the
  projection mixes the row (and centring the frame), spreading it there.
- Temporal heatmap backward: a pair's ``d`` is a per-pixel sum, so a pair with a NaN pixel gives NaN at the pixels where
  either plane is NaN and its exact gradient elsewhere when it is unmasked, and 0 elsewhere when it is masked.
NaN positions of values and gradients must match exactly; the finite entries must be close.

Every case with finite results also runs twice and must give the same bits, forward and backward."""
import numpy as np
import pytest
import torch

import scale_oracle as S
from oracle import lp_oracle as O

pytestmark = pytest.mark.gpu

F64 = torch.float64
NAN = float("nan")
UNSUPPORTED = -3  # LPB_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


def gen(seed):
    return torch.Generator().manual_seed(seed)


def f32(x):
    """x rounded to fp32 as the kernels see it, back in float64 for the references."""
    return torch.as_tensor(x, dtype=torch.float32).to(F64)


def close(a, b, atol, rtol, what):
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), f"{what}: NaN at {na.nonzero().tolist()[:8]}, reference NaN at {nb.nonzero().tolist()[:8]}"
    err = (a - b).abs()
    bad = ~(err <= atol + rtol * b.abs()) & ~nb
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {b.numel()} differ; worst {float(err[bad].max())} "
                                 f"(atol {atol}, rtol {rtol}) at {bad.nonzero().tolist()[:4]}")


def finite_max(g):
    g = g.detach().abs()
    g = g[~torch.isnan(g)]
    return float(g.max()) if g.numel() else 0.0


def close_values(a, b, what="values"):
    close(a, b, 1e-5, 1e-4, what)


def close_grads(a, b, what="gradient"):
    close(a, b, 1e-6 * finite_max(b), 1e-3, what)


def same_bits(a, b, what):
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{what} differs between two identical calls"


# ------------------------------------------------------------------------------------------------
# ops.unsup_losses against float64
# ------------------------------------------------------------------------------------------------
class Pca:
    """One PCA loss: the kernel's PcaParams and its float64 reference.  ``sel`` is the single-view column list, or the
    multi-view mirrored_column_matches (views x n_sel)."""

    def __init__(self, sel, mean, kept, eps, centering=None, multiview=False):
        self.sel, self.centering, self.multiview = sel, centering, multiview
        self.mean = torch.as_tensor(mean, dtype=torch.float32)
        self.kept = torch.as_tensor(kept, dtype=torch.float32).reshape(-1, self.mean.numel())
        self.eps = float(np.float32(eps))

    def params(self, lpb, dev):
        if self.multiview:
            mcm = np.asarray(self.sel, np.int32)
            return lpb.PcaParams(mcm.reshape(-1), mcm.shape[1], mcm.shape[0], None, self.mean.numpy(), self.kept.numpy(), self.eps, dev)
        idx = np.asarray(self.sel, np.int32)
        return lpb.PcaParams(idx, len(idx), 0, self.centering, self.mean.numpy(), self.kept.numpy(), self.eps, dev)

    def ref(self, x):
        if self.multiview:
            return S.pca_multiview_ref(x, [list(v) for v in self.sel], self.mean, self.kept, self.eps)
        return S.pca_singleview_ref(x, list(self.sel), self.centering, self.mean, self.kept, self.eps)

    def residuals(self, kp):
        """float64 reprojection errors of every (row, pair) over all clips: where to put an epsilon."""
        out = []
        for x in kp.cpu().to(F64):
            if self.multiview:
                data = O.pca_format_multiview(x, [list(v) for v in self.sel])
            else:
                data = O.pca_format_singleview(x, list(self.sel), self.centering)
            out.append(O.pca_reprojection_error(data, self.mean.to(F64), self.kept.to(F64)).reshape(-1))
        return torch.cat(out)


def eps_between(resid):
    """An fp32 epsilon halfway across the widest relative gap between neighbouring values in their middle half: some
    pairs pass the rectification and some do not, and none lies within fp32 rounding of the threshold."""
    s = torch.unique(resid[~torch.isnan(resid)])
    if s.numel() < 2:
        return float(np.float32(s[0] + 1))
    lo, hi = s.numel() // 4, max(s.numel() // 4 + 1, 3 * s.numel() // 4)
    gaps = (s[lo + 1 : hi + 1] - s[lo:hi]) / s[lo + 1 : hi + 1]
    i = lo + int(gaps.argmax())
    return float(np.float32((s[i] + s[i + 1]) / 2))


def basis(d, n_comp, g):
    """n_comp orthonormal rows of length d."""
    if n_comp == 0:
        return torch.zeros(0, d)
    return torch.linalg.qr(torch.randn(d, n_comp, generator=g, dtype=F64))[0].T.float().contiguous()


def sv_loss(kp, cols, centering, n_comp, seed, eps=None):
    g = gen(seed)
    d = 2 * len(cols)
    p = Pca(cols, torch.randn(d, generator=g) * 5, basis(d, n_comp, g), 0.0, centering)
    p.eps = eps_between(p.residuals(kp)) if eps is None else float(np.float32(eps))
    return p


def mv_loss(kp, mcm, n_comp, seed, eps=None):
    g = gen(seed)
    d = 2 * len(mcm)
    p = Pca(mcm, torch.randn(d, generator=g) * 5 + 100, basis(d, n_comp, g), 0.0, multiview=True)
    p.eps = eps_between(p.residuals(kp)) if eps is None else float(np.float32(eps))
    return p


def keypoints(n_clips, t, k, seed, scale=30.0):
    """Smooth-ish tracks: a random walk around 100 px, so temporal distances spread around a few pixels."""
    g = gen(seed)
    start = 100 + scale * torch.randn(n_clips, 1, 2 * k, generator=g)
    steps = 3.0 * torch.randn(n_clips, t, 2 * k, generator=g) * torch.rand(n_clips, 1, 2 * k, generator=g) * 2
    return (start + steps.cumsum(1)).float()


def run_unsup(lpb, dev, kp, conf, eps, thr, sv, mv, wts):
    x = kp.to(dev).clone().requires_grad_(True)
    out = lpb.unsup_losses(x, None if conf is None else conf.to(dev), temporal_eps=eps, prob_threshold=thr,
                           pca_singleview=None if sv is None else sv.params(lpb, dev),
                           pca_multiview=None if mv is None else mv.params(lpb, dev))
    (out[:, :3] * wts.to(dev)).sum().backward()
    return out[:, :3].detach(), x.grad


def ref_unsup(kp, conf, eps, thr, sv, mv, wts):
    """float64 values (n_clips, 3) and the gradient of sum(values * wts); T = 1 gives a NaN temporal value with no
    gradient (the mean of an empty tensor)."""
    xr = kp.cpu().to(F64).requires_grad_(True)
    zero = torch.zeros((), dtype=F64)
    rows = []
    for i in range(kp.shape[0]):
        if eps is None:
            lt = zero
        elif kp.shape[1] == 1:
            lt = torch.tensor(NAN, dtype=F64)
        else:
            lt = S.temporal_loss_ref(xr[i], None if conf is None else conf[i].cpu().to(F64), f32(eps), thr)
        rows.append(torch.stack([lt, sv.ref(xr[i]) if sv is not None else zero, mv.ref(xr[i]) if mv is not None else zero]))
    ref = torch.stack(rows)
    xr.grad = torch.zeros_like(xr)
    ref_w = ref * wts.to(F64)
    if ref_w.requires_grad:
        ref_w.sum().backward()
    return ref.detach(), xr.grad


def check_unsup(lpb, dev, kp, conf=None, eps=None, thr=0.0, sv=None, mv=None, seed=0):
    wts = torch.rand(kp.shape[0], 3, generator=gen(seed + 1000)) + 0.5
    out, grad = run_unsup(lpb, dev, kp, conf, eps, thr, sv, mv, wts)
    ref, gref = ref_unsup(kp, conf, eps, thr, sv, mv, wts)
    close_values(out, ref)
    close_grads(grad, gref)
    if bool(torch.isfinite(out).all()) and bool(torch.isfinite(grad).all()):
        out2, grad2 = run_unsup(lpb, dev, kp, conf, eps, thr, sv, mv, wts)
        same_bits(out, out2, "unsup_losses forward")
        same_bits(grad, grad2, "unsup_losses backward")
    return out, grad, ref, gref


# ---- temporal --------------------------------------------------------------------------------------------------------
TK = 6
TEMPORAL_CASES = {
    "T1": dict(t=1, eps=2.0),
    "T2": dict(t=2, eps=2.0),
    "T2_conf": dict(t=2, eps=1.0, conf="rand", thr=0.3),
    "scalar_eps": dict(t=9, eps=3.0, conf="rand", thr=0.25),
    "per_keypoint_eps_with_0": dict(t=9, eps=[0.0, 1.5, 3.0, 0.0, 5.0, 2.25], conf="rand", thr=0.25),
    "zero_distances_eps0": dict(t=9, eps=0.0, zero_dist=True),
    "zero_distances_per_keypoint_eps": dict(t=9, eps=[0.0, 1.5, 3.0, 0.0, 5.0, 2.25], zero_dist=True, conf="rand", thr=0.25),
    "conf_at_threshold": dict(t=9, eps=2.0, conf="at_thr", thr=0.5),
    "nan_confidence": dict(t=9, eps=2.0, conf="nan", thr=0.5),
    "no_confidences": dict(t=9, eps=2.0),
    "threshold_0": dict(t=9, eps=2.0, conf="rand", thr=0.0),
}


def temporal_inputs(t, eps, conf=None, thr=0.0, zero_dist=False, n_clips=3, k=TK, seed=1):
    kp = keypoints(n_clips, t, k, seed)
    if zero_dist and t > 2:
        kp[:, 3] = kp[:, 2]  # every keypoint still between frames 2 and 3
        kp[0, 5, 2:4] = kp[0, 4, 2:4]
    c = None
    if conf is not None:
        c = torch.rand(n_clips, t, k, generator=gen(seed + 1))
        if conf == "at_thr":
            c[:, ::2, ::2] = thr     # exactly at the threshold: kept (the mask is conf < thr)
            c[:, 1::3, 1] = 0.4999   # just below: masked
        elif conf == "nan":
            c[:, :, 1] = NAN         # never masked
            c[0, 2, 3] = NAN
    return kp, c


@pytest.mark.parametrize("case", list(TEMPORAL_CASES))
def test_temporal_edges(lpb, dev, case):
    kw = dict(TEMPORAL_CASES[case])
    kp, conf = temporal_inputs(kw.pop("t"), kw["eps"], kw.get("conf"), kw.get("thr", 0.0), kw.get("zero_dist", False))
    out, grad, ref, _ = check_unsup(lpb, dev, kp, conf, kw["eps"], kw.get("thr", 0.0))
    if kp.shape[1] == 1:
        assert bool(torch.isnan(out[:, 0]).all()) and bool((grad == 0).all())
    else:
        assert bool(torch.isfinite(ref).all())


# ---- single-view PCA --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("centering", [None, "mean", "median"])
@pytest.mark.parametrize("n_sel", [1, 2, 3, 16, 17, 256])
def test_singleview_selection_sizes(lpb, dev, centering, n_sel):
    """n_sel up to UL_MAX_SEL * 4 = 256, the most make_pca_dev accepts; columns a random permutation of a larger K."""
    k = n_sel + 3
    kp = keypoints(2, 6, k, seed=10 + n_sel)
    cols = torch.randperm(k, generator=gen(n_sel))[:n_sel].tolist()
    sv = sv_loss(kp, cols, centering, min(3, 2 * n_sel - 1), seed=20 + n_sel)
    check_unsup(lpb, dev, kp, sv=sv, seed=n_sel)


def plant(kp, cols, t, c, values):
    for q, v in zip(range(len(cols)), values):
        kp[:, t, 2 * cols[q] + c] = v


@pytest.mark.parametrize("n_sel", [5, 6])
def test_singleview_median_ties(lpb, dev, n_sel):
    """Exact ties in a frame: the gradient of each centre goes to the ranks' stable-sort positions.
    Odd n_sel = 5: [4, 4, 1, 4, 9] has the median at rank 2, the second 4.  Even n_sel = 6: [7, 1, 7, 9, 3, 7] has both
    middle ranks 2 and 3 on the tied 7s at positions 0 and 2 (not 5), and [2, 8, 5, 5, 0, 9] the middle ranks on the
    two 5s.  A frame whose values are all equal ties every rank."""
    k = 9
    kp = keypoints(2, 5, k, seed=30)
    cols = [6, 1, 4, 0, 8, 3][:n_sel]
    if n_sel == 5:
        plant(kp, cols, 0, 0, [104.0, 104.0, 101.0, 104.0, 109.0])
        plant(kp, cols, 1, 1, [96.0, 93.0, 96.0, 93.0, 99.0])
    else:
        plant(kp, cols, 0, 0, [107.0, 101.0, 107.0, 109.0, 103.0, 107.0])
        plant(kp, cols, 1, 1, [102.0, 108.0, 105.0, 105.0, 100.0, 109.0])
    plant(kp, cols, 2, 0, [111.0] * n_sel)
    plant(kp, cols, 3, 1, [88.0] * n_sel)
    sv = sv_loss(kp, cols, "median", 2, seed=31)
    check_unsup(lpb, dev, kp, sv=sv, seed=32)


@pytest.mark.parametrize("centering", [None, "mean", "median"])
def test_singleview_columns_out_of_order_and_repeated(lpb, dev, centering):
    k = 9
    kp = keypoints(3, 7, k, seed=40)
    cols = [5, 2, 2, 7, 0, 3]
    sv = sv_loss(kp, cols, centering, 4, seed=41)
    _, grad, _, _ = check_unsup(lpb, dev, kp, sv=sv, seed=42)
    unused = [q for q in range(k) if q not in cols]
    assert bool((grad.reshape(3, 7, k, 2)[:, :, unused] == 0).all())


@pytest.mark.parametrize("centering", [None, "mean", "median"])
def test_singleview_no_components(lpb, dev, centering):
    """n_comp = 0: the reprojection is the mean; ``kept`` is an empty tensor (null pointer), which is never read."""
    kp = keypoints(2, 6, 7, seed=50)
    sv = sv_loss(kp, [0, 3, 1, 6, 5], centering, 0, seed=51)
    assert sv.params(lpb, dev).kept.numel() == 0
    check_unsup(lpb, dev, kp, sv=sv, seed=52)


@pytest.mark.parametrize("centering", [None, "median"])
def test_singleview_all_components_zero_residual(lpb, dev, centering):
    """n_comp = D: every point is its own reprojection.  With a signed permutation as the basis and quarter-pixel
    keypoints the residual is exactly 0 in fp32 and float64 (odd n_sel: the median is one of the values), so the loss
    is 0 and the gradient is 0, as torch's norm gives at a zero norm, for epsilon 0 and above."""
    k, cols = 8, [7, 2, 4, 0, 5]
    d = 2 * len(cols)
    kp = torch.round(keypoints(2, 6, k, seed=60) * 4) / 4
    perm = torch.randperm(d, generator=gen(61))
    kept = torch.zeros(d, d)
    kept[torch.arange(d), perm] = torch.where(torch.arange(d) % 3 == 0, -1.0, 1.0)
    for eps in (0.0, 2.0):
        sv = Pca(cols, torch.arange(d) * 3.0 - 7.0, kept, eps, centering)
        out, grad, _, _ = check_unsup(lpb, dev, kp, sv=sv, seed=62)
        assert bool((out[:, 1] == 0).all()) and bool((grad == 0).all())


def test_singleview_epsilon_edges(lpb, dev):
    """Epsilon 0 (every residual passes) and one larger than every residual (loss 0, gradient 0)."""
    kp = keypoints(3, 6, 9, seed=70)
    cols = [1, 4, 2, 8, 6, 0, 3]
    sv = sv_loss(kp, cols, "mean", 3, seed=71, eps=0.0)
    check_unsup(lpb, dev, kp, sv=sv, seed=72)
    sv = sv_loss(kp, cols, "median", 3, seed=71, eps=0.0)
    sv.eps = float(np.float32(sv.residuals(kp).max() * 2 + 1))
    out, grad, _, _ = check_unsup(lpb, dev, kp, sv=sv, seed=73)
    assert bool((out[:, 1] == 0).all()) and bool((grad == 0).all())


# ---- multi-view PCA ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("views", [2, 3, 4, 8])
@pytest.mark.parametrize("n_sel", [1, 5])
def test_multiview_views(lpb, dev, views, n_sel):
    k = views * n_sel + 2
    kp = keypoints(2, 7, k, seed=80 + views)
    mcm = torch.randperm(k, generator=gen(81 + views))[: views * n_sel].reshape(views, n_sel).tolist()
    mv = mv_loss(kp, mcm, min(3, 2 * views - 1), seed=82 + views)
    check_unsup(lpb, dev, kp, mv=mv, seed=83)


def test_multiview_table_not_monotone_with_keypoints_outside(lpb, dev):
    """Keypoints 3 and 9 are in no view: their gradient is exactly 0."""
    k = 10
    mcm = [[7, 0, 5, 2], [8, 4, 6, 1]]
    kp = keypoints(3, 8, k, seed=90)
    mv = mv_loss(kp, mcm, 2, seed=91)
    _, grad, _, _ = check_unsup(lpb, dev, kp, mv=mv, seed=92)
    g = grad.reshape(3, 8, k, 2)
    assert bool((g[:, :, [3, 9]] == 0).all()) and bool((g[:, :, [0, 1, 2, 4, 5, 6, 7, 8]] != 0).any())


def test_all_three_losses_with_a_keypoint_reached_twice(lpb, dev):
    """Temporal + single-view (median) + multi-view in one call.  Keypoint 3 is in two views of the table (at two
    positions) and twice in the single-view columns, so several shared-memory atomicAdds meet on it in the backward:
    the two runs must still give the same bits."""
    k = 9
    mcm = [[3, 0, 5], [2, 3, 8], [6, 1, 7]]
    cols = [4, 3, 0, 3, 8, 1, 6]
    kp = keypoints(4, 10, k, seed=100)
    conf = torch.rand(4, 10, k, generator=gen(101))
    sv = sv_loss(kp, cols, "median", 3, seed=102)
    mv = mv_loss(kp, mcm, 3, seed=103)
    check_unsup(lpb, dev, kp, conf, [1.0, 2.0, 0.0, 3.0, 1.5, 2.5, 0.5, 4.0, 2.0], 0.2, sv, mv, seed=104)


# ---- scale ------------------------------------------------------------------------------------------------------------
def test_more_clips_than_one_wave(lpb, dev):
    """One CTA per clip in both directions: 2 x SMs + 5 clips, with all three losses on."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    n_clips, k = 2 * sms + 5, 17
    kp = keypoints(n_clips, 8, k, seed=110)
    conf = torch.rand(n_clips, 8, k, generator=gen(111))
    cols = list(range(0, k, 2))
    mcm = [list(range(0, 8)), list(range(8, 16))]
    sv = sv_loss(kp, cols, "median", 3, seed=112)
    mv = mv_loss(kp, mcm, 3, seed=113)
    check_unsup(lpb, dev, kp, conf, 3.0, 0.2, sv, mv, seed=114)


def unsup_bwd_bytes(t, k, pcas):
    """lpb_unsup_losses_bwd's dynamic shared memory (losses.cu): the largest pca_scratch_floats(bwd) of its PCA losses,
    the clip's gradient (T * K * 2) and 4 floats."""
    def scratch(n_sel, views, n_comp):
        d = 2 * views if views else 2 * n_sel
        rows = t * n_sel if views else t
        return 2 * (rows * d + rows * n_comp) + 2 * t

    return (max(scratch(*p) for p in pcas) + t * k * 2 + 4) * 4


def test_largest_clip_the_backward_fits_and_one_more_is_refused(lpb, dev):
    """Four views of 17 keypoints, 3 components, temporal on: the largest T whose backward fits the device's opt-in
    shared memory (the backward kernel has no static shared memory) runs against float64; T + 1 is refused by
    ``set_dynamic_smem`` with LPB_ERR_UNSUPPORTED before anything is queued, and the next call runs."""
    from lightning_pose_b200._lib import LpbError

    limit = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    views, n_sel, n_comp = 4, 17, 3
    k = views * n_sel
    t = max(t for t in range(2, 4096) if unsup_bwd_bytes(t, k, [(n_sel, views, n_comp)]) <= limit)
    mcm = torch.arange(k).reshape(views, n_sel).tolist()
    kp = keypoints(2, t, k, seed=120)
    conf = torch.rand(2, t, k, generator=gen(121))
    mv = mv_loss(kp, mcm, n_comp, seed=122)
    check_unsup(lpb, dev, kp, conf, 3.0, 0.1, None, mv, seed=123)

    kp = keypoints(1, t + 1, k, seed=124).to(dev).requires_grad_(True)
    out = lpb.unsup_losses(kp, temporal_eps=3.0, pca_multiview=mv.params(lpb, dev))  # the forward needs less and runs
    need = unsup_bwd_bytes(t + 1, k, [(n_sel, views, n_comp)])
    with pytest.raises(LpbError, match=f"error {UNSUPPORTED}: unsup_losses_bwd: needs {need} B"):
        out[:, :3].sum().backward()
    assert kp.grad is None
    check_unsup(lpb, dev, keypoints(2, 6, k, seed=125), None, 3.0, 0.0, None, mv_loss(keypoints(2, 6, k, seed=125), mcm, 2, 126))
    torch.cuda.synchronize()


# ---- NaN --------------------------------------------------------------------------------------------------------------
NAN_CASES = {
    # (centering of the single-view loss, components of both PCA losses, mask the NaN keypoint's frame, NaN coordinate)
    "x_median": ("median", 3, False, 0),
    "y_mean": ("mean", 3, False, 1),
    "x_none_no_components": (None, 0, False, 0),
    "y_median_no_components": ("median", 0, False, 1),
    "x_median_masked": ("median", 3, True, 0),
    "x_none_no_components_masked": (None, 0, True, 0),
}


@pytest.mark.parametrize("case", list(NAN_CASES))
def test_nan_keypoint(lpb, dev, case):
    """One NaN coordinate of keypoint 2 at frame 3 of clip 0, read by all three losses; clip 1 stays finite.  With
    ``masked`` the keypoint's confidence at frame 3 is below the threshold, so both of its temporal pairs are masked:
    the temporal value stays finite and its gradient still has the NaN (0 * NaN)."""
    centering, n_comp, masked, coord = NAN_CASES[case]
    k, t = 8, 7
    kp = keypoints(2, t, k, seed=130)
    conf = torch.rand(2, t, k, generator=gen(131)) * 0.7 + 0.3
    if masked:
        conf[0, 3, 2] = 0.1
    sv = sv_loss(kp, [2, 5, 0, 7, 3], centering, n_comp, seed=132)
    mv = mv_loss(kp, [[2, 6], [1, 4]], min(n_comp, 3), seed=133)
    kp[0, 3, 2 * 2 + coord] = NAN
    out, grad, ref, gref = check_unsup(lpb, dev, kp, conf, [1.0, 0.5, 2.0, 0.0, 1.0, 3.0, 2.0, 1.0], 0.2, sv, mv, seed=134)
    assert bool(torch.isnan(ref[0, 1:]).all()) and bool(torch.isfinite(ref[1]).all())
    assert bool(torch.isnan(ref[0, 0])) != masked
    assert bool(torch.isnan(gref[0]).any()) and not bool(torch.isnan(gref[1]).any())


def test_nan_keypoint_outside_the_pca_selections(lpb, dev):
    """A NaN keypoint that neither PCA loss selects makes only the temporal loss NaN."""
    k, t = 8, 6
    kp = keypoints(2, t, k, seed=140)
    sv = sv_loss(kp, [0, 1, 3], "median", 2, seed=141)
    mv = mv_loss(kp, [[4, 5], [6, 3]], 2, seed=142)
    kp[1, 0, 2 * 2 + 1] = NAN
    out, _, ref, _ = check_unsup(lpb, dev, kp, None, 2.0, 0.0, sv, mv, seed=143)
    assert bool(torch.isnan(ref[1, 0])) and bool(torch.isfinite(ref[1, 1:]).all()) and bool(torch.isfinite(ref[0]).all())


# ------------------------------------------------------------------------------------------------
# ops.temporal_heatmap_loss against float64
# ------------------------------------------------------------------------------------------------
def planes(t, k, h, w, seed, zeros=False):
    """Non-negative planes at per-plane scales from 0 to 2, so the pair terms d spread over a decade; ``zeros`` puts
    exact zeros in a fifth of the pixels (KL's 1e-10 guard)."""
    g = gen(seed)
    hm = torch.rand(t, k, h, w, generator=g) * torch.rand(t, k, 1, 1, generator=g) * 2
    if zeros:
        hm[torch.rand(t, k, h, w, generator=g) < 0.2] = 0.0
    return hm


def thm_eps(hm, kind, per_keypoint, with_zero=True):
    """Epsilons between the pair terms (mse: means of squares, kl: sums over pixels), so some pairs pass and some do
    not; the per-keypoint list starts with 0 unless ``with_zero`` is False."""
    a, b = hm[:-1].to(F64), hm[1:].to(F64)
    terms = ((a - b) ** 2).flatten(2).mean(-1) if kind == "mse" else O.kl_div_2d(a + 1e-10, b + 1e-10)
    terms = terms[~torch.isnan(terms)]
    if not per_keypoint:
        return eps_between(terms)
    k = hm.shape[1]
    qs = torch.quantile(terms, torch.linspace(0.1, 0.9, k - 1 if with_zero else k, dtype=F64))
    return ([0.0] if with_zero else []) + [float(np.float32(q)) for q in qs]


def run_thm(lpb, dev, hm, conf, kind, eps, thr, w, unaligned=False):
    if unaligned:
        buf = torch.zeros(hm.numel() + 1, device=dev)
        view = buf[1:].view(hm.shape)
        view.copy_(hm.to(dev))
        h = view.detach().requires_grad_(True)  # same storage, 4 bytes past a 16-byte boundary
        assert h.data_ptr() % 16 != 0
    else:
        h = hm.to(dev).clone().requires_grad_(True)
    v = lpb.temporal_heatmap_loss(h, conf.to(dev), kind, torch.tensor(eps, dtype=torch.float32), thr)
    (w * v).backward()
    return v.detach().reshape(()), h.grad


def check_thm(lpb, dev, hm, conf, kind, eps, thr, seed=0, unaligned=False):
    w = float(torch.rand((), generator=gen(seed + 2000))) + 0.5
    v, grad = run_thm(lpb, dev, hm, conf, kind, eps, thr, w, unaligned)
    hr = hm.to(F64).requires_grad_(True)
    ref = O.temporal_heatmap_loss(hr, conf.to(F64), kind, eps, thr)
    (w * ref).backward()
    close_values(v, ref.detach(), "temporal heatmap loss")
    if kind == "kl":  # -p / q at a zero pixel is 1e8 times its neighbours': take the scale per plane
        b = hr.grad.abs().masked_fill(torch.isnan(hr.grad), 0).flatten(2).amax(-1)[..., None, None]
        g, r = grad.detach().cpu().to(F64), hr.grad
        na, nb = torch.isnan(g), torch.isnan(r)
        assert torch.equal(na, nb), f"gradient NaN at {na.nonzero().tolist()[:8]}, reference at {nb.nonzero().tolist()[:8]}"
        bad = ~((g - r).abs() <= 1e-6 * b + 1e-3 * r.abs()) & ~nb
        assert not bool(bad.any()), f"{int(bad.sum())} gradient entries differ, worst {float((g - r).abs()[bad].max())}"
    else:
        close_grads(grad, hr.grad)
    if bool(torch.isfinite(v)) and bool(torch.isfinite(grad).all()):
        v2, grad2 = run_thm(lpb, dev, hm, conf, kind, eps, thr, w, unaligned)
        same_bits(v, v2, "temporal heatmap forward")
        same_bits(grad, grad2, "temporal heatmap backward")
    return v, grad, ref.detach(), hr.grad


KINDS = ["mse", "kl"]


@pytest.mark.parametrize("kind", KINDS)
def test_temporal_heatmap_two_frames(lpb, dev, kind):
    hm = planes(2, 5, 12, 16, seed=200)
    conf = torch.rand(2, 5, generator=gen(201))
    check_thm(lpb, dev, hm, conf, kind, thm_eps(hm, kind, False), 0.2, seed=202)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("unaligned", [False, True], ids=["aligned", "unaligned"])
def test_temporal_heatmap_odd_plane(lpb, dev, kind, unaligned):
    """17 x 23 planes (391 pixels, odd), also read through a view 4 bytes past a 16-byte boundary."""
    hm = planes(6, 4, 17, 23, seed=210)
    conf = torch.rand(6, 4, generator=gen(211))
    check_thm(lpb, dev, hm, conf, kind, thm_eps(hm, kind, True), 0.25, seed=212, unaligned=unaligned)


@pytest.mark.parametrize("kind", KINDS)
def test_temporal_heatmap_identical_planes_and_zeros(lpb, dev, kind):
    """Planes 2 and 3 are identical, and so are planes (4, 1) and (5, 1): d = 0, which is no gradient at eps 0 or above;
    a fifth of all pixels are exact zeros.  MSE runs at eps 0 too.  KL does not: the float64 reference evaluates the KL
    of identical planes as xlogy(p, p) - p * log(p), whose two logs differ in the last bit, so its d is about +-1e-17
    and F.relu's gradient at eps 0 turns on or off with that sign; the kernel's p * (log p - log q) is exactly 0."""
    hm = planes(6, 4, 16, 16, seed=220, zeros=True)
    hm[3] = hm[2]
    hm[5, 1] = hm[4, 1]
    conf = torch.rand(6, 4, generator=gen(221))
    cases = (0.0, thm_eps(hm, kind, True)) if kind == "mse" else (thm_eps(hm, kind, True, with_zero=False),)
    for eps in cases:
        check_thm(lpb, dev, hm, conf, kind, eps, 0.1, seed=222)


@pytest.mark.parametrize("kind", KINDS)
def test_temporal_heatmap_confidence_at_threshold(lpb, dev, kind):
    """Confidences exactly at the threshold are kept (conf < thr masks); just below are masked; NaN is kept."""
    hm = planes(7, 5, 10, 12, seed=230)
    conf = torch.rand(7, 5, generator=gen(231))
    conf[::2, ::2] = 0.5
    conf[1::3, 1] = 0.4999
    conf[4, 3] = NAN
    check_thm(lpb, dev, hm, conf, kind, thm_eps(hm, kind, True), 0.5, seed=232)


@pytest.mark.parametrize("kind", KINDS)
def test_temporal_heatmap_pairs_past_one_wave(lpb, dev, kind):
    """(T - 1) * K pair CTAs: more than two waves at the pair kernel's full residency (8 CTAs of 256 threads per SM);
    the final kernel's single CTA loops over all of them."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    k = 64
    t = -(-2 * 8 * sms // k) + 2
    assert (t - 1) * k > 2 * 8 * sms
    hm = planes(t, k, 8, 8, seed=240)
    conf = torch.rand(t, k, generator=gen(241))
    check_thm(lpb, dev, hm, conf, kind, thm_eps(hm, kind, True), 0.15, seed=242)


THM_NAN_CASES = {
    # (what is NaN, mask the NaN plane's frame)
    "pixel": ("pixel", False),
    "plane": ("plane", False),
    "pixel_masked": ("pixel", True),
    "plane_masked": ("plane", True),
}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", list(THM_NAN_CASES))
def test_temporal_heatmap_nan(lpb, dev, kind, case):
    """One NaN pixel or one all-NaN plane at (t = 2, k = 1).  Unmasked, the loss is NaN; masked (confidence of
    keypoint 1 at frame 2 below the threshold, so both of its pairs), the loss stays finite and the NaN reaches only the
    gradient, at the NaN pixels of planes 1, 2 and 3."""
    what, masked = THM_NAN_CASES[case]
    hm = planes(5, 3, 9, 11, seed=250)
    conf = torch.rand(5, 3, generator=gen(251)) * 0.5 + 0.5
    eps = thm_eps(hm, kind, True)
    if what == "pixel":
        hm[2, 1, 4, 7] = NAN
    else:
        hm[2, 1] = NAN
    if masked:
        conf[2, 1] = 0.1
    v, grad, ref, gref = check_thm(lpb, dev, hm, conf, kind, eps, 0.3, seed=252)
    assert bool(torch.isnan(ref)) != masked
    assert bool(torch.isnan(gref[1:4, 1]).any()) and not bool(torch.isnan(gref[:, [0, 2]]).any())
