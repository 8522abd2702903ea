"""Training from keypoint targets made on the device (no target plane written): the fused Gaussian-target + KL / JS
kernels (lpb_heatmap_loss_from_keypoints_*) against float64, and every tracker fed a keypoint-only labeled batch
against the same seeded tracker fed dense targets.

Kernels: the edge batch of ``targets_oracle.py`` (keypoints on, just inside and just outside every edge, NaN and +-inf
coordinates, visibility 0, 1, 2, 3, -1 and none) at heatmaps 64^2, 96^2, 128^2 and 64 x 96, sigma 1.25 and 2.0, and 51
keypoints, past one wave of CTAs; the loss within 1e-5 of its operands' magnitudes and the gradient within 1e-5 per
plane (``div_targets_oracle.py``); MSE through the new entry bit-identical to lpb_heatmap_mse_from_keypoints_*; the
fused KL / JS against materialize() + the dense loss; and a profile showing no target plane rendered.

Trackers (stand-in backbones defined here): loss, every parameter gradient and ``last_rmse`` of a keypoint-only batch
against ``O.gaussian_targets`` dense heatmaps, for heatmap_mse, heatmap_kl and heatmap_js."""
import math

import pytest
import torch

import div_targets_oracle as DO
import targets_oracle as TO
from oracle import lp_oracle as O

pytestmark = pytest.mark.gpu

KINDS = ("kl", "js")
LOSSES = ("heatmap_mse", "heatmap_kl", "heatmap_js")
# (image height, width, heatmap height, width)
MAPS = [(256, 256, 64, 64), (384, 384, 96, 96), (512, 512, 128, 128), (256, 384, 64, 96)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


@pytest.fixture(scope="module")
def min_planes(dev):
    """Planes that make the one-CTA-per-plane launches run past one wave: 2 x SMs x 8."""
    return 2 * torch.cuda.get_device_properties(dev).multi_processor_count * 8


def report(name, ratio):
    print(f"\nworst error/allowed {name}: {ratio:.3g}")


def _preds(b, k, oh, ow, dev, seed):
    """Positive planes of the scale of a softmax output, with some exact zeros (p + 1e-10 then matters)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    p = torch.rand(b, k, oh, ow, device=dev, generator=g) * (2.0 / (oh * ow))
    p[..., ::7, ::5] = 0.0
    return p


def _fused(ops, kind, kp, preds, h, w, sigma, vis, gout=1.0):
    p = preds.clone().requires_grad_(True)
    loss, count = ops.heatmap_loss_from_keypoints(kind, kp, p, h, w, sigma, visibility=vis, return_count=True)
    (g,) = torch.autograd.grad(loss, p, torch.tensor(gout, device=p.device))
    return loss.detach(), count, g


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", MAPS)
@pytest.mark.parametrize("sigma", [1.25, 2.0])
@pytest.mark.parametrize("kind", KINDS)
def test_div_from_keypoints_edges(ops, dev, min_planes, cfg, sigma, kind):
    """The edge batch with every visibility form: NaN planes kept (NaN loss, NaN on the same gradient planes), finite
    when those planes get visibility 0, and every plane dropped (NaN loss, zero gradient)."""
    h, w, oh, ow = cfg
    kp, vis = (t.to(dev) for t in TO.edge_batch(h, w, oh, ow, min_planes=min_planes))
    preds = _preds(kp.shape[0], kp.shape[1], oh, ow, dev, seed=8)
    nan = TO.plane_pattern(TO.target_planes(kp, h, w, oh, ow, sigma, vis)[0]) == TO.NAN
    finite = torch.where(nan, 0, vis).to(torch.int32)
    worst = 0.0
    for v in (None, vis, finite, torch.zeros_like(vis)):
        loss, count, g = _fused(ops, kind, kp, preds, h, w, sigma, v, gout=0.75)
        ref_loss, ref_g, scale, gscale = DO.div_from_keypoints(kind, kp, preds, h, w, sigma, v)
        case = f"{kind} {cfg} sigma {sigma} vis {'none' if v is None else 'given'}"
        worst = max(worst, DO.check_loss(loss, ref_loss, scale, case=case))
        worst = max(worst, TO.check_relative_per_plane(g, 0.75 * ref_g, 1e-5, case, scale=0.75 * gscale))
        t, _ = TO.target_planes(kp, h, w, oh, ow, sigma, v)
        assert int(count) == int((~(t == 0).all(-1).all(-1)).sum()), case
    assert torch.isnan(DO.div_from_keypoints(kind, kp, preds, h, w, sigma, vis)[0])
    assert not torch.isnan(DO.div_from_keypoints(kind, kp, preds, h, w, sigma, finite)[0])
    loss, count, g = _fused(ops, kind, torch.full_like(kp, float("nan")), preds, h, w, sigma, None)
    assert torch.isnan(loss) and int(count) == 0 and bool((g == 0).all())
    report(f"{kind} from keypoints {cfg} sigma {sigma}", worst)


@pytest.mark.parametrize("kind", KINDS)
def test_div_from_keypoints_51_keypoints_past_one_wave(ops, dev, kind):
    """768 x 17 planes (past one wave) and 51 keypoints per frame, random labels with every visibility value."""
    worst = 0.0
    for b, k, cfg in ((768, 17, (384, 384, 96, 96)), (64, 51, (256, 384, 64, 96))):
        h, w, oh, ow = cfg
        g = torch.Generator(device=dev).manual_seed(b + k)
        kp = torch.rand(b, k, 2, device=dev, generator=g) * torch.tensor([w * 1.1, h * 1.1], device=dev) - 0.05 * torch.tensor([w, h], device=dev)
        vis = torch.tensor(TO.VIS_VALUES, dtype=torch.int32, device=dev)[torch.randint(0, 5, (b, k), device=dev, generator=g)]
        preds = _preds(b, k, oh, ow, dev, seed=k)
        for v in (None, vis):
            loss, _, grad = _fused(ops, kind, kp, preds, h, w, 1.25, v)
            ref_loss, ref_g, scale, gscale = DO.div_from_keypoints(kind, kp, preds, h, w, 1.25, v)
            worst = max(worst, DO.check_loss(loss, ref_loss, scale, case=f"{kind} {b}x{k}"))
            worst = max(worst, TO.check_relative_per_plane(grad, ref_g, 1e-5, f"{kind} {b}x{k}", scale=gscale))
    report(f"{kind} from keypoints past one wave", worst)


def _bits(x):
    return x.reshape(1).view(torch.int32).item()


@pytest.mark.parametrize("cfg", MAPS)
def test_mse_through_the_new_entry_is_the_mse_entry(ops, dev, min_planes, cfg):
    """kind "mse" with the kept count runs lpb_heatmap_mse_from_keypoints_*: the same bits of loss (NaN included: the
    NaN planes of the batch without a visibility are kept) and dense gradient."""
    h, w, oh, ow = cfg
    kp, vis = (t.to(dev) for t in TO.edge_batch(h, w, oh, ow, min_planes=min_planes))
    preds = _preds(kp.shape[0], kp.shape[1], oh, ow, dev, seed=9)
    finite = torch.where(TO.plane_pattern(TO.target_planes(kp, h, w, oh, ow, 1.25, vis)[0]) == TO.NAN, 0, vis).to(torch.int32)
    for v in (None, finite):
        loss, _, g = _fused(ops, "mse", kp, preds, h, w, 1.25, v)
        p = preds.clone().requires_grad_(True)
        old = ops.heatmap_mse_from_keypoints(kp, p, h, w, 1.25, visibility=v)
        (g_old,) = torch.autograd.grad(old, p)
        g_old = g_old.materialize() if isinstance(g_old, ops.MseKeypointGrad) else g_old
        assert _bits(loss) == _bits(old.detach()) and torch.equal(g.view(torch.int32), g_old.view(torch.int32))
        # without the count the new op is the old one, gradient held implicitly
        p2 = preds.clone().requires_grad_(True)
        (g_imp,) = torch.autograd.grad(ops.heatmap_loss_from_keypoints("mse", kp, p2, h, w, 1.25, visibility=v), p2)
        assert isinstance(g_imp, ops.MseKeypointGrad) and torch.equal(g_imp.materialize().view(torch.int32), g_old.view(torch.int32))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cfg", MAPS[:2])
def test_div_from_keypoints_matches_materialized_targets(ops, dev, min_planes, kind, cfg):
    """The fused loss and gradient against GaussianTargets.materialize() + ops.heatmap_loss, within fp32 summation
    tolerance (the same per-pixel arithmetic, summed in another order)."""
    from lightning_pose_b200.data.heatmaps import GaussianTargets

    h, w, oh, ow = cfg
    kp, vis = (t.to(dev) for t in TO.edge_batch(h, w, oh, ow, min_planes=min_planes))
    finite = torch.where(TO.plane_pattern(TO.target_planes(kp, h, w, oh, ow, 1.25, vis)[0]) == TO.NAN, 0, vis).to(torch.int32)
    preds = _preds(kp.shape[0], kp.shape[1], oh, ow, dev, seed=10)
    targ = GaussianTargets(kp, h, w, (oh, ow), visibility=finite, ignore_nans=True)
    loss, _, g = _fused(ops, kind, kp, preds, h, w, 1.25, finite)
    p = preds.clone().requires_grad_(True)
    dense = ops.heatmap_loss(targ.materialize(), p, kind)
    (g_dense,) = torch.autograd.grad(dense, p)
    _, _, scale, gscale = DO.div_from_keypoints(kind, kp, preds, h, w, 1.25, finite)
    DO.check_loss(loss, dense.detach(), scale, case=f"{kind} fused vs dense")
    ratio = TO.check_relative_per_plane(g, g_dense, 1e-5, f"{kind} fused vs dense", scale=gscale)
    report(f"{kind} fused vs materialized {cfg}", ratio)


def test_losses_given_gaussian_targets_render_no_target_plane(ops, dev):
    """HeatmapKLLoss, HeatmapJSLoss and ReprojectionHeatmapLoss given GaussianTargets, forward and backward: no
    generate_heatmaps_kernel for the targets (the reprojection loss renders its predicted planes once, and their
    backward), no dense loss kernel; and the same losses within fp32 tolerance of dense targets."""
    from torch.profiler import ProfilerActivity, profile

    from lightning_pose_b200.data.heatmaps import GaussianTargets
    from lightning_pose_b200.losses.losses import HeatmapJSLoss, HeatmapKLLoss, ReprojectionHeatmapLoss

    b, k, h, w, oh, ow = 8, 17, 256, 256, 64, 64
    g = torch.Generator(device=dev).manual_seed(3)
    kp = torch.rand(b, k, 2, device=dev, generator=g) * 256
    kp[0, 1] = -5.0
    vis = torch.randint(0, 3, (b, k), device=dev, generator=g).to(torch.int32)
    targ = GaussianTargets(kp, h, w, (oh, ow), visibility=vis)
    preds = torch.softmax(torch.randn(b, k, oh * ow, device=dev, generator=g), -1).reshape(b, k, oh, ow).requires_grad_(True)
    kp_rep = (kp + torch.randn(b, k, 2, device=dev, generator=g) * 3).requires_grad_(True)
    rep = ReprojectionHeatmapLoss(h, w, oh, ow)

    def run():
        out = []
        for loss in (HeatmapKLLoss(), HeatmapJSLoss()):
            v, _ = loss(targ, preds)
            out.append((v, torch.autograd.grad(v, preds)[0]))
        v, _ = rep(targ, kp_rep)
        out.append((v, torch.autograd.grad(v, kp_rep)[0]))
        return out

    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # the session can lose the record of its first kernel (it is launched before the first activity buffer is
        # handed out), so a throwaway kernel goes first and the counted ones all come after it
        torch.zeros(1, device=dev).add_(1.0)
        torch.cuda.synchronize()
        fused = run()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert sum("generate_heatmaps_kernel" in n for n in names) == 1, [n for n in names if "generate" in n]
    assert not any("heatmap_loss_plane_kernel" in n or "heatmap_loss_bwd_kernel" in n for n in names)
    assert sum("heatmap_div_from_kp_kernel" in n for n in names) == 2
    assert sum("heatmap_div_from_kp_bwd_kernel" in n for n in names) == 2
    assert any("heatmap_mse_from_kp_kernel" in n for n in names) and any("heatmap_mse_from_kp_bwd_kernel" in n for n in names)

    dense_t = targ.materialize()
    want = []
    for loss in (HeatmapKLLoss(), HeatmapJSLoss()):
        v, _ = loss(dense_t, preds)
        want.append((v, torch.autograd.grad(v, preds)[0]))
    v, _ = rep(dense_t, kp_rep)
    want.append((v, torch.autograd.grad(v, kp_rep)[0]))
    for i, ((a, ga), (b_, gb)) in enumerate(zip(fused, want)):
        assert torch.isfinite(a) and float(a.detach()) != 0.0, i
        torch.testing.assert_close(a, b_, rtol=2e-5, atol=0, msg=f"loss {i}")
        assert float((ga - gb).abs().max()) <= 1e-4 * float(gb.abs().max()), i


def test_reprojection_loss_with_every_plane_dropped_is_zero(ops, dev):
    """The reference's zero-loss result when no plane is kept (losses.py:483-486), with a zero gradient."""
    from lightning_pose_b200.data.heatmaps import GaussianTargets
    from lightning_pose_b200.losses.losses import ReprojectionHeatmapLoss

    kp = torch.rand(2, 5, 2, device=dev) * 128
    targ = GaussianTargets(kp, 128, 128, (32, 32), visibility=torch.zeros(2, 5, dtype=torch.int32, device=dev))
    kp_rep = (kp + 1.0).requires_grad_(True)
    v, _ = ReprojectionHeatmapLoss(128, 128, 32, 32)(targ, kp_rep)
    (g,) = torch.autograd.grad(v, kp_rep)
    assert float(v) == 0.0 and bool((g == 0).all())


# ------------------------------------------------------------------------------------------------
# trackers: keypoint-only batches against dense targets
# ------------------------------------------------------------------------------------------------
def _mask(kp, h, w):
    """The out-of-frame -> NaN rule of compute_heatmap (datasets.py:496-508), on the host."""
    out = kp.clone()
    oob = (kp[..., 0] < 0) | (kp[..., 1] < 0) | (kp[..., 0] >= w) | (kp[..., 1] >= h)
    out[oob] = float("nan")
    return out


def _labels(b, planes, h, w, seed):
    """(keypoints (b, planes, 2) image pixels with out-of-frame ones and a NaN, visibility (b, planes) in 0..2)."""
    g = torch.Generator().manual_seed(seed)
    kp = torch.rand(b, planes, 2, generator=g) * torch.tensor([w, h], dtype=torch.float32)
    kp[0, 1] = torch.tensor([-3.0, 10.0])
    kp[1 % b, 2] = torch.tensor([20.0, float(h)])
    kp[b - 1, 0] = float("nan")
    vis = torch.randint(0, 3, (b, planes), generator=g)
    vis[0, :3] = 2  # the out-of-frame and NaN planes are Gaussian-or-dropped, not uniform
    vis[1 % b, 2] = 2
    vis[b - 1, 0] = 2
    return kp, vis


def _grads_close(new, ref, rel=1e-2, floor=1e-5, case=""):
    """Every parameter gradient within ``rel`` of its own largest value plus ``floor`` of the largest gradient entry of
    the model.  The dense and the fused target gradients differ in the last bits, which a bf16 operand can carry one
    bf16 step, and the head's bias gradients are float-atomic sums of terms that cancel (the last layer's exactly,
    through the softmax), so a bias gradient near zero is held to the rounding of the model's gradients, not its own: a
    gradient whose largest entry is below 1e-3 of the model's largest (the last layer's bias) is rounding noise, and
    need only stay below that bound."""
    pairs = [(name, a.grad, b.grad) for (name, a), b in zip(new.named_parameters(), ref.parameters())]
    top = max(float(b.abs().max()) for _, _, b in pairs if b is not None)
    assert top > 0, case
    for name, a, b in pairs:
        if b is None:
            assert a is None, (case, name)
            continue
        if float(b.abs().max()) <= 1e-3 * top:
            assert float(a.abs().max()) <= 1e-3 * top, f"{case} {name}: {float(a.abs().max()):.3g} (top {top:.3g})"
            continue
        err = float((a - b).abs().max())
        assert err <= rel * float(b.abs().max()) + floor * top, f"{case} {name}: {err:.3g} vs {float(b.abs().max()):.3g} (top {top:.3g})"


def _compare(new, ref, loss_new, loss_ref, case=""):
    """Loss to 1e-5 relative, the gradients by ``_grads_close``, last_rmse to 1e-5."""
    torch.testing.assert_close(loss_new, loss_ref, rtol=1e-5, atol=0, msg=case)
    _grads_close(new, ref, case=case)
    torch.testing.assert_close(new.last_rmse, ref.last_rmse, rtol=1e-5, atol=1e-5, msg=case)


class _Conv(torch.nn.Module):
    """A strided convolution standing in for a backbone; ``bf16`` outputs the 16-bit features the tensor-core head reads."""

    def __init__(self, c, stride, bf16):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, c, stride, stride=stride)
        self.bf16 = bf16

    def forward(self, x):
        y = self.conv(x)
        return y.bfloat16() if self.bf16 else y


@pytest.mark.parametrize("loss", LOSSES)
def test_heatmap_tracker_with_folded_views(ops, dev, loss):
    """HeatmapTracker on (B, V, 3, H, W): the views fold into the batch and the targets are (B, V K, h, w)."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    b, v, k, img = 3, 2, 6, 128

    def make():
        torch.manual_seed(77)
        t = HeatmapTracker(k, loss_factory=LossFactory({loss: {"log_weight": 0.0}}, None), backbone=_Conv(64, 32, False), num_fc_input_features=64).to(dev)
        for layer in list(t.head.upsampling_layers)[1:]:
            torch.nn.init.xavier_uniform_(layer.weight, gain=2.0)
        return t

    kp, vis = _labels(b, v * k, img, img, seed=1)
    images = torch.randn(b, v, 3, img, img)
    bbox = torch.tensor([[0.0, 0.0, float(img), float(img)] * v]).repeat(b, 1)
    dense = O.gaussian_targets(_mask(kp, img, img), img, img, (img // 4, img // 4), visibility=vis).float()
    common = {"images": images.to(dev), "bbox": bbox.to(dev), "is_multiview": True}
    ref = make()
    l_ref = ref.evaluate_labeled({**common, "keypoints": _mask(kp, img, img).reshape(b, -1).to(dev), "heatmaps": dense.to(dev)}, "train", 1.0)
    l_ref.backward()
    new = make()
    l_new = new.evaluate_labeled({**common, "keypoints": kp.reshape(b, -1).to(dev), "visibility": vis.to(dev)}, "train", 1.0)
    l_new.backward()
    _compare(new, ref, l_new, l_ref, case=f"folded views {loss}")


CONTEXT = {"stride32_uf2": ("resnet50", 2048, 32), "stride16_uf1": ("vits_dino", 384, 16)}


def _context_tracker(dev, arch, c, stride, loss, semi=False):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import HeatmapTrackerMHCRNN, SemiSupervisedHeatmapTrackerMHCRNN

    torch.manual_seed(31)
    kw = {"loss_factory": LossFactory({loss: {"log_weight": 0.0}}, None), "backbone": _Conv(c, stride, True), "backbone_arch": arch,
          "num_fc_input_features": c}
    if semi:
        kw["loss_factory_unsupervised"] = LossFactory({"temporal": {"log_weight": 0.5, "epsilon": 1.0, "prob_threshold": 0.0}}, None)
        tr = SemiSupervisedHeatmapTrackerMHCRNN(5, **kw).to(dev)
    else:
        tr = HeatmapTrackerMHCRNN(5, **kw).to(dev)
    torch.manual_seed(32)
    head = tr.head
    for layer in [*list(head.head_sf.upsampling_layers)[1:], head.head_mf.W_f, head.head_mf.W_b]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return tr


@pytest.mark.parametrize("case", list(CONTEXT))
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("views", [1, 2])
def test_context_tracker(ops, dev, case, loss, views):
    """HeatmapTrackerMHCRNN on (B, 5, 3, H, W) and (B, V, 5, 3, H, W): the centre frame's keypoints; targets standing
    for cat([heatmaps, heatmaps]), one copy per head; the out-of-frame rule reaching the RMSE targets."""
    arch, c, stride = CONTEXT[case]
    b, k, img = 2, 5, 256
    kp, vis = _labels(b, views * k, img, img, seed=2)
    shape = (b, 5, 3, img, img) if views == 1 else (b, views, 5, 3, img, img)
    images = torch.randn(shape)
    bbox = torch.tensor([[2.0, 3.0, img * 1.5, img * 1.2] * views]).repeat(b, 1)
    dense = O.gaussian_targets(_mask(kp, img, img), img, img, (img // 4, img // 4), visibility=vis).float()
    common = {"images": images.to(dev), "bbox": bbox.to(dev)}
    if views > 1:
        common["num_views"] = torch.full((b,), views, device=dev)
    ref = _context_tracker(dev, arch, c, stride, loss)
    l_ref = ref.evaluate_labeled({**common, "keypoints": _mask(kp, img, img).reshape(b, -1).to(dev), "heatmaps": dense.to(dev)}, "train", 1.0)
    l_ref.backward()
    new = _context_tracker(dev, arch, c, stride, loss)
    batch = {**common, "keypoints": kp.reshape(b, -1).to(dev), "visibility": vis.to(dev)}
    kp_before = batch["keypoints"].clone()
    l_new = new.evaluate_labeled(batch, "train", 1.0)
    l_new.backward()
    assert torch.equal(batch["keypoints"].isnan(), kp_before.isnan())  # the batch's keypoints are left as they were
    _compare(new, ref, l_new, l_ref, case=f"context {case} {loss} views {views}")


# ---- multi-view transformer -----------------------------------------------------------------------------------------------
D = 128
MV_V, MV_K, MV_B, MV_IMG = 4, 5, 2, 128


class _Patch(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = torch.nn.Conv2d(3, D, 16, stride=16)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class _Mix(torch.nn.Module):
    """Stands in for the attention blocks: mixes the tokens of all views of an example."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(D, D)

    def forward(self, t):
        return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()


MV_LOSSES = {
    "uncalibrated": None,
    "calibrated": {
        "supervised_pairwise_projections": {"log_weight": 0.0},
        "supervised_reprojection_heatmap_mse": {"log_weight": 0.0, "original_image_height": MV_IMG, "original_image_width": MV_IMG,
                                                "downsampled_image_height": MV_IMG // 4, "downsampled_image_width": MV_IMG // 4},
    },
}


def _mv_tracker(dev, losses, semi=False):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import (HeatmapTrackerMultiviewTransformer,
                                                                      SemiSupervisedHeatmapTrackerMultiviewTransformer)

    torch.manual_seed(41)
    fac = LossFactory(losses, None)
    if semi:
        unsup = LossFactory({"temporal": {"log_weight": 0.5, "epsilon": 1.0, "prob_threshold": 0.0}}, None)
        tr = SemiSupervisedHeatmapTrackerMultiviewTransformer(MV_K, MV_V, _Patch(), _Mix(), D, loss_factory=fac, loss_factory_unsupervised=unsup)
    else:
        tr = HeatmapTrackerMultiviewTransformer(MV_K, MV_V, _Patch(), _Mix(), D, loss_factory=fac)
    tr = tr.to(dev)
    for layer in list(tr.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return tr


def _cameras(b, v, seed):
    """Cameras on a half circle, 2 units from the origin, looking at it (no two facing each other)."""
    g = torch.Generator().manual_seed(seed)
    K = torch.zeros(b, v, 3, 3)
    E = torch.zeros(b, v, 3, 4)
    for j in range(v):
        K[:, j, 0, 0] = K[:, j, 1, 1] = 300.0 + torch.randn(b, generator=g) * 20
        K[:, j, 0, 2], K[:, j, 1, 2], K[:, j, 2, 2] = MV_IMG / 2, MV_IMG / 2, 1.0
        a = j / v * math.pi
        E[:, j] = torch.tensor([[math.cos(a), 0.0, -math.sin(a), 0.0], [0.0, 1.0, 0.0, 0.0], [math.sin(a), 0.0, math.cos(a), 2.0]])
    return K, E, torch.randn(b, v, 5, generator=g) * 0.02


def _mv_batches(dev, calibrated, ignore_nans, seed=5):
    """(dense-target batch, keypoint-only batch) of the same labels, keypoints (B, V K 2) view-major."""
    b, v, k, img = MV_B, MV_V, MV_K, MV_IMG
    kp, vis = _labels(b, v * k, img, img, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    common = {"images": torch.randn(b, v, 3, img, img, generator=g).to(dev), "is_multiview": True,
              "bbox": torch.tensor([[img / 2 - 2, img / 2 - 2, 4.0, 4.0] * v], device=dev).repeat(b, 1)}
    if calibrated:
        K, E, Dist = _cameras(b, v, seed + 2)
        kp3 = torch.randn(b, k, 3, generator=g) * 0.3
        kp3[0, 3] = float("nan")
        common.update({"keypoints_3d": kp3.to(dev), "intrinsic_matrix": K.to(dev), "extrinsic_matrix": E.to(dev), "distortions": Dist.to(dev)})
    kp_t = kp if ignore_nans else _mask(kp, img, img)
    dense = O.gaussian_targets(kp_t, img, img, (img // 4, img // 4), visibility=vis).float()
    ref = {**common, "keypoints": kp_t.reshape(b, -1).to(dev), "heatmaps": dense.to(dev)}
    new = {**common, "keypoints": kp.reshape(b, -1).to(dev), "visibility": vis.to(dev)}
    if ignore_nans is not None:
        new["ignore_nans"] = ignore_nans
    return ref, new


@pytest.mark.parametrize("form", ["uncalibrated", "calibrated", "calibrated_ignore_nans_false", "calibrated_ignore_nans_true"])
@pytest.mark.parametrize("loss", LOSSES)
def test_multiview_transformer(ops, dev, form, loss):
    """Planes view-major (v K + k); the out-of-frame rule unless ``ignore_nans`` is True.  Calibrated batches also
    carry the pairwise-projection and reprojection losses (the latter evaluating its targets from the keypoints)."""
    calibrated = form != "uncalibrated"
    ignore = {"calibrated_ignore_nans_false": False, "calibrated_ignore_nans_true": True}.get(form)
    losses = {loss: {"log_weight": 0.0}, **(MV_LOSSES["calibrated"] if calibrated else {})}
    ref_b, new_b = _mv_batches(dev, calibrated, bool(ignore))
    if ignore is None:
        new_b.pop("ignore_nans", None)
    ref = _mv_tracker(dev, losses)
    l_ref = ref.evaluate_labeled(ref_b, "train", 1.0)
    l_ref.backward()
    new = _mv_tracker(dev, losses)
    l_new = new.evaluate_labeled(new_b, "train", 1.0)
    l_new.backward()
    assert torch.isfinite(l_new)
    if calibrated:
        names = {d["name"] for d in new.last_logs}
        assert "train_supervised_reprojection_heatmap_mse_loss" in names
        rep = [d["value"] for d in new.last_logs if d["name"] == "train_supervised_reprojection_heatmap_mse_loss"][0]
        rep_ref = [d["value"] for d in ref.last_logs if d["name"] == "train_supervised_reprojection_heatmap_mse_loss"][0]
        torch.testing.assert_close(rep, rep_ref, rtol=1e-5, atol=0)
    _compare(new, ref, l_new, l_ref, case=f"multiview {form} {loss}")


def test_multiview_ignore_nans_changes_the_targets(ops, dev):
    """The two forms differ on a batch with an out-of-frame keypoint: the rule drops its plane, ignore_nans keeps a
    clamped Gaussian."""
    _, with_rule = _mv_batches(dev, True, False)
    _, without = _mv_batches(dev, True, True)
    tr = _mv_tracker(dev, {"heatmap_mse": {"log_weight": 0.0}})
    a = tr._keypoint_targets(with_rule).keypoints
    b = tr._keypoint_targets(without).keypoints
    assert bool(torch.isnan(a[0, 1]).all()) and not bool(torch.isnan(b[0, 1]).any())


# ---- semi-supervised training steps -----------------------------------------------------------------------------------------
def _semi_compare(tr_ref, tr_new, batch_ref, batch_new, unlabeled, case):
    l_ref = tr_ref.training_step({"labeled": batch_ref, "unlabeled": unlabeled}, 0)["loss"]
    l_ref.backward()
    l_new = tr_new.training_step({"labeled": batch_new, "unlabeled": unlabeled}, 0)["loss"]
    l_new.backward()
    assert torch.isfinite(l_new)
    torch.testing.assert_close(l_new, l_ref, rtol=1e-5, atol=0, msg=case)
    _grads_close(tr_new, tr_ref, case=case)


def test_semisupervised_heatmap_tracker_step(ops, dev):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import SemiSupervisedHeatmapTracker

    b, k, img, t = 3, 6, 128, 6

    def make():
        torch.manual_seed(5)
        return SemiSupervisedHeatmapTracker(
            k, loss_factory=LossFactory({"heatmap_kl": {"log_weight": 0.0}}, None), backbone=_Conv(64, 32, False), num_fc_input_features=64,
            loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": 0.5, "epsilon": 1.0, "prob_threshold": 0.0}}, None)).to(dev)

    kp, vis = _labels(b, k, img, img, seed=7)
    common = {"images": torch.randn(b, 3, img, img).to(dev), "bbox": torch.tensor([[0.0, 0.0, 100.0, 90.0]]).repeat(b, 1).to(dev)}
    dense = O.gaussian_targets(_mask(kp, img, img), img, img, (img // 4, img // 4), visibility=vis).float().to(dev)
    unlabeled = {"frames": torch.randn(t, 3, img, img).to(dev), "transforms": torch.tensor([-1.0], device=dev),
                 "bbox": torch.tensor([[0.0, 0.0, 100.0, 90.0]]).repeat(t, 1).to(dev)}
    _semi_compare(make(), make(), {**common, "keypoints": _mask(kp, img, img).reshape(b, -1).to(dev), "heatmaps": dense},
                  {**common, "keypoints": kp.reshape(b, -1).to(dev), "visibility": vis.to(dev)}, unlabeled, "semi HeatmapTracker")


def test_semisupervised_context_tracker_step(ops, dev):
    b, k, img, t = 2, 5, 256, 7
    kp, vis = _labels(b, k, img, img, seed=8)
    common = {"images": torch.randn(b, 5, 3, img, img).to(dev), "bbox": torch.tensor([[0.0, 0.0, 300.0, 280.0]]).repeat(b, 1).to(dev)}
    dense = O.gaussian_targets(_mask(kp, img, img), img, img, (img // 4, img // 4), visibility=vis).float().to(dev)
    unlabeled = {"frames": torch.randn(t, 3, img, img).to(dev), "transforms": torch.tensor([-1.0], device=dev),
                 "bbox": torch.tensor([[0.0, 0.0, 300.0, 280.0]]).repeat(t, 1).to(dev), "is_multiview": False}
    arch, c, stride = CONTEXT["stride16_uf1"]
    _semi_compare(_context_tracker(dev, arch, c, stride, "heatmap_js", semi=True), _context_tracker(dev, arch, c, stride, "heatmap_js", semi=True),
                  {**common, "keypoints": _mask(kp, img, img).reshape(b, -1).to(dev), "heatmaps": dense},
                  {**common, "keypoints": kp.reshape(b, -1).to(dev), "visibility": vis.to(dev)}, unlabeled, "semi context")


def test_semisupervised_multiview_step(ops, dev):
    t = 5
    ref_b, new_b = _mv_batches(dev, True, False)
    g = torch.Generator().manual_seed(9)
    unlabeled = {"frames": torch.randn(t, MV_V, 3, MV_IMG, MV_IMG, generator=g).to(dev), "transforms": -torch.ones(MV_V, 1, device=dev),
                 "bbox": torch.tensor([[0.0, 0.0, 150.0, 140.0] * MV_V]).repeat(t, 1).to(dev), "is_multiview": True}
    losses = {"heatmap_mse": {"log_weight": 0.0}, **MV_LOSSES["calibrated"]}
    _semi_compare(_mv_tracker(dev, losses, semi=True), _mv_tracker(dev, losses, semi=True), ref_b, new_b, unlabeled, "semi multiview")


# ---- one CUDA graph -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss", ["heatmap_mse", "heatmap_kl"])
def test_multiview_keypoint_only_step_replays_in_cuda_graph(ops, dev, loss):
    """A calibrated keypoint-only labeled training_step (targets built by a kernel, reprojection loss on them) captured
    once: two replays equal two eager steps."""
    losses = {loss: {"log_weight": 0.0}, **MV_LOSSES["calibrated"]}
    tr = _mv_tracker(dev, losses)
    _, batch = _mv_batches(dev, True, False)
    kp0 = batch["keypoints"].clone()
    params = list(tr.head.parameters()) + [tr.view_embeddings]

    def step():
        batch["keypoints"].copy_(kp0)
        out = tr.training_step(batch, 0)["loss"]
        return [out.detach(), *torch.autograd.grad(out, params)]

    eager = [[x.clone() for x in step()] for _ in range(2)]
    assert torch.isfinite(eager[0][0])
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for i in range(2):
        graph.replay()
        got = [x.clone() for x in out]
        torch.testing.assert_close(got[0], eager[i][0], rtol=1e-6, atol=0, msg=f"replay {i}")
        for a, b in zip(eager[i][1:], got[1:]):  # the head's bias gradient is summed with float atomics
            assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()), i
    torch.cuda.synchronize(dev)
