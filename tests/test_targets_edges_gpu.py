"""Every kernel built on the Gaussian-target rule (csrc/targets.cuh) against the float64 restatement of
``targets_oracle.py``, on one edge batch: keypoints that scale to exactly -1 and size + 1 on the heatmap grid and to the
nearest fp32 products on either side (at a power-of-two image-to-grid ratio and at ratios that are not), NaN in x, in y
and in both, +-inf, -0.0, and visibility 0, 1, 2, 3 and -1 (any value other than 0, 1, 2 keeps the clamped Gaussian, as
the reference's masks do).  Sigma 0.5, 1.25 and 3.0; heatmaps 96x96, 64x80 from a 256x320 image, and 128x192 (wider
than one 128-thread pass of the target kernels).

Consumers: generate_heatmaps (forward and keep_gradients backward), heatmap_mse_from_keypoints (loss and the dense
gradient), the bf16 head's backward fed that gradient implicitly (lpb_head_bwd_bf16_targets: plane_dot_targets_kernel
and the target forms of the layer-2 gradient kernels, with and without decode windows), keypoints_mask_oob and
evaluate_heatmaps_at_location.  The one-CTA-per-plane kernels get at least 2 x SMs x 8 planes (SM count read from the
device).  The acceptance rules live in ``targets_oracle.py``; ``test_targets_oracle.py`` shows on the CPU that they
reject plausible wrong rules.  Each test prints its worst error / allowed ratio."""
import numpy as np
import pytest
import torch

import targets_oracle as TO
from head_support import features, head_params, make_head

pytestmark = pytest.mark.gpu

F64 = torch.float64
HEAD_IMG = (406, 384)  # image (height, width) of the head tests: sy = 96 / 406 is not a power of two


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


def edge_batch(cfg, n, dev):
    h, w, oh, ow = cfg
    kp, vis = TO.edge_batch(h, w, oh, ow, min_planes=n)
    assert kp.shape[0] * kp.shape[1] >= n
    return kp.to(dev), vis.to(dev)


def nan_planes(kp, cfg, sigma, vis):
    h, w, oh, ow = cfg
    return TO.plane_pattern(TO.target_planes(kp, h, w, oh, ow, sigma, vis)[0]) == TO.NAN


def dense(g, ops):
    return g.materialize() if isinstance(g, ops.MseKeypointGrad) else g


# ------------------------------------------------------------------------------------------------
# generate_heatmaps
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", TO.CONFIGS)
@pytest.mark.parametrize("sigma", TO.SIGMAS)
def test_generate_heatmaps_edges(ops, dev, min_planes, cfg, sigma):
    h, w, oh, ow = cfg
    kp, vis = edge_batch(cfg, min_planes, dev)
    worst = 0.0
    for v in (None, vis):
        got = ops.generate_heatmaps(kp, h, w, (oh, ow), sigma, visibility=v)
        ref, _ = TO.target_planes(kp, h, w, oh, ow, sigma, v)
        worst = max(worst, TO.check_planes(got, ref, f"{cfg} sigma {sigma} vis {v is not None}"))
    report(f"generate_heatmaps {cfg} sigma {sigma}", worst)


@pytest.mark.parametrize("cfg", TO.CONFIGS)
@pytest.mark.parametrize("sigma", TO.SIGMAS)
def test_generate_heatmaps_keep_gradients_edges(ops, dev, min_planes, cfg, sigma):
    """d sum(planes * gout) / d keypoints per keypoint within 1e-5 of the sum of the magnitudes of its per-pixel terms
    (``TO.keep_gradients_scale``: with a random gout the terms cancel, and a keypoint's gradient can be far smaller than
    the rounding of its terms); keypoints exactly on the clamp bounds pass the gradient, as torch.clamp does; NaN exactly
    where float64 has it, and exact zeros where no term reaches the keypoint."""
    h, w, oh, ow = cfg
    kp, vis = edge_batch(cfg, min_planes, dev)
    gout = torch.randn(kp.shape[0], kp.shape[1], oh, ow, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    x, y = TO.grid_coords(kp, h, w, oh, ow)
    worst = 0.0
    for v in (None, vis):
        leaf = kp.clone().requires_grad_(True)
        (ops.generate_heatmaps(leaf, h, w, (oh, ow), sigma, keep_gradients=True, visibility=v) * gout).sum().backward()
        _, mode, ref = TO.target_planes(kp, h, w, oh, ow, sigma, v, keep_gradients=True, gout=gout)
        on = (mode == TO.GAUSS) & ((x == -1) | (x == ow + 1))
        assert bool(on.any()) and bool((ref[..., 0][on] != 0).all()), "no gradient through a keypoint on the clamp bound"
        scale = TO.keep_gradients_scale(kp, h, w, oh, ow, sigma, v, gout).reshape(-1)
        worst = max(worst, TO.check_relative_per_plane(leaf.grad.reshape(-1, 1, 2), ref.reshape(-1, 1, 2), 1e-5,
                                                       f"{cfg} sigma {sigma} vis {v is not None}", scale=scale))
    report(f"generate_heatmaps backward {cfg} sigma {sigma}", worst)


# ------------------------------------------------------------------------------------------------
# heatmap_mse_from_keypoints
# ------------------------------------------------------------------------------------------------
def _mse(ops, kp, preds, cfg, sigma, v):
    h, w = cfg[:2]
    p = preds.clone().requires_grad_(True)
    loss = ops.heatmap_mse_from_keypoints(kp, p, h, w, sigma, visibility=v)
    (g,) = torch.autograd.grad(loss, p)
    return loss.detach(), dense(g, ops)


@pytest.mark.parametrize("cfg", TO.CONFIGS)
@pytest.mark.parametrize("sigma", TO.SIGMAS)
def test_heatmap_mse_from_keypoints_edges(ops, dev, min_planes, cfg, sigma):
    """Loss within 1e-5 relative and d loss / d preds within 1e-5 of each plane's largest reference value.  On the full
    edge batch NaN planes are kept, so the loss is NaN on both sides and NaN lands on the same gradient planes; with the
    NaN planes given visibility 0 the loss is finite; with every plane dropped the loss is NaN and the gradient zero."""
    h, w, oh, ow = cfg
    kp, vis = edge_batch(cfg, min_planes, dev)
    preds = torch.rand(kp.shape[0], kp.shape[1], oh, ow, device=dev, generator=torch.Generator(device=dev).manual_seed(8)) * (2.0 / (oh * ow))
    finite = torch.where(nan_planes(kp, cfg, sigma, vis), 0, vis).to(torch.int32)
    worst = 0.0
    for v in (None, vis, finite, torch.zeros_like(vis)):
        loss, g = _mse(ops, kp, preds, cfg, sigma, v)
        ref_loss, ref_g = TO.mse_from_keypoints(kp, preds, h, w, sigma, v)
        if torch.isnan(ref_loss):
            assert torch.isnan(loss), float(loss)
        else:
            r = abs(float(loss) - float(ref_loss)) / (1e-5 * abs(float(ref_loss)))
            assert r <= 1.0, (float(loss), float(ref_loss))
            worst = max(worst, r)
        worst = max(worst, TO.check_relative_per_plane(g, ref_g, 1e-5, f"{cfg} sigma {sigma}"))
    assert torch.isnan(TO.mse_from_keypoints(kp, preds, h, w, sigma, vis)[0])
    assert not torch.isnan(TO.mse_from_keypoints(kp, preds, h, w, sigma, finite)[0])
    # keypoints all NaN without a visibility: every plane dropped
    loss, g = _mse(ops, torch.full_like(kp, float("nan")), preds, cfg, sigma, None)
    assert torch.isnan(loss) and bool((g == 0).all())
    report(f"heatmap_mse_from_keypoints {cfg} sigma {sigma}", worst)


# ------------------------------------------------------------------------------------------------
# the bf16 head's backward with the MSE gradient implicit (target form)
# ------------------------------------------------------------------------------------------------
HEAD_CASES = [  # (C, H, W, channels, frames, sigma)
    (2048, 12, 12, (17, 17), 256, 3.0),  # config 2
    (2048, 12, 12, (51, 51), 64, 0.5),   # keypoint groups
    (384, 16, 16, (17,), 64, 2.0),       # one deconv (config 3)
]


def _head_labels(b, k, oh, ow, sigma, dev):
    """The edge rows dealt over the head's (b, k) planes with visibility 0, 1, 2, 3, -1 in turn; planes whose target is
    NaN get visibility 0 (one NaN plane would make every weight gradient NaN)."""
    rows = TO.edge_rows(*HEAD_IMG, oh, ow)
    i = torch.arange(b * k)
    kp = rows[i % rows.shape[0]].reshape(b, k, 2).to(dev)
    vis = torch.tensor(TO.VIS_VALUES, dtype=torch.int32)[(i // rows.shape[0]) % len(TO.VIS_VALUES)].reshape(b, k).to(dev)
    vis = torch.where(nan_planes(kp, (*HEAD_IMG, oh, ow), sigma, vis), 0, vis).to(torch.int32)
    return kp, vis


def _assert_bitwise(a, b, case):
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape and x.stride() == y.stride(), (case, i)
        view = torch.int16 if x.element_size() == 2 else torch.int32
        assert torch.equal(x.view(view), y.view(view)), (case, i)


@pytest.mark.parametrize("c,h,w,channels,b,sigma", HEAD_CASES)
def test_head_backward_target_form_edges(ops, dev, c, h, w, channels, b, sigma):
    """(a) Through autograd, the head's gradients with the MSE gradient implicit are bit-identical to those with it dense
    (plane_dot_targets_kernel and g2_build_kernel's target form).  (b) The dense gradient is within 1e-5 of each plane's
    largest float64 value."""
    head = make_head(c, channels, seed=23)
    f = features(b, c, h, w, seed=24, dtype=torch.bfloat16).requires_grad_(True)
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    hm = head(f)
    oh, ow = hm.shape[-2:]
    kp, vis = _head_labels(b, channels[-1], oh, ow, sigma, dev)
    assert bool((vis == 3).any()) and bool((vis == -1).any())
    loss = ops.heatmap_mse_from_keypoints(kp, hm, *HEAD_IMG, sigma, visibility=vis)
    g = torch.autograd.grad(loss, hm, retain_graph=True)[0]
    assert isinstance(g, ops.MseKeypointGrad)
    implicit = [t.clone() for t in torch.autograd.grad(hm, [f] + params, g, retain_graph=True)]
    assert g.dense is None, "the head backward materialised the gradient"
    d_hm = g.materialize().clone()
    want = [t.clone() for t in torch.autograd.grad(hm, [f] + params, d_hm, retain_graph=True)]
    _assert_bitwise(implicit, want, (c, channels))
    _, ref = TO.mse_from_keypoints(kp, hm.detach(), *HEAD_IMG, sigma, vis)
    ratio = TO.check_relative_per_plane(d_hm, ref, 1e-5, f"head {c} {channels}")
    report(f"head backward target form d hm {c} {channels}", ratio)


def _peaked_planes(b, k, oh, ow, seed, n_diffuse):
    """Softmax planes with one sharp peak each (the decode's support fits its 32 x 32 window: flag 1), the first
    ``n_diffuse`` flat (the support overflows: flag 2, the dense fallback)."""
    g = torch.Generator().manual_seed(seed)
    cy = torch.rand(b, k, 1, 1, generator=g) * (oh - 1)
    cx = torch.rand(b, k, 1, 1, generator=g) * (ow - 1)
    yy = torch.arange(oh).view(1, 1, oh, 1).float()
    xx = torch.arange(ow).view(1, 1, 1, ow).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * 1.6**2) + 0.05 * torch.randn(b, k, oh, ow, generator=g)
    logits.view(b * k, oh, ow)[:n_diffuse] *= 1e-3
    return torch.softmax(logits.reshape(b, k, -1), -1).reshape(b, k, oh, ow)


@pytest.mark.parametrize("c,h,w,channels,b,sigma", HEAD_CASES)
def test_head_backward_target_form_with_decode_windows(ops, dev, c, h, w, channels, b, sigma):
    """A keypoint-loss gradient as well: one set of decode windows (valid windows, flag 1, and dense fallback planes,
    flag 2) goes to the head backward twice, once with the MSE gradient implicit and once dense.  The window planes then
    take g2_patch_kernel's target form and the fallback planes g2_build_kernel's, and all gradients are bit-identical;
    the implicit backward run again gives the same bits."""
    (ws, bs) = head_params(make_head(c, channels, seed=33))
    f = features(b, c, h, w, seed=34, dtype=torch.bfloat16)
    probs, saved = ops._head_forward_bf16(f, ws, bs, True, train=True)
    bb, k, oh, ow = probs.shape
    kp, vis = _head_labels(bb, k, oh, ow, sigma, dev)
    p = probs.detach().requires_grad_(True)
    (g,) = torch.autograd.grad(ops.heatmap_mse_from_keypoints(kp, p, *HEAD_IMG, sigma, visibility=vis), p)
    assert isinstance(g, ops.MseKeypointGrad) and g.implicit_for(probs)
    ds, temp = 2, 1000.0
    peaked = _peaked_planes(bb, k, oh, ow, seed=35, n_diffuse=3 * k + 2).to(dev)
    _, _, stats = ops.decode_forward(peaked, ds, temp)
    g_kp = torch.randn(bb, k, 2, device=dev, generator=torch.Generator(device=dev).manual_seed(36))
    windows = ops.decode_backward_windows(peaked, stats, g_kp, ds, temp)
    flags = windows[1][:, 2]
    assert int((flags == 1).sum()) >= bb * k // 2 and int((flags == 2).sum()) >= 1, flags.bincount().tolist()
    w2 = ws[1] if len(ws) > 1 else None

    def backward(g_out, mse):
        return [t.clone() for t in ops.head_backward_bf16(g_out, saved, f.shape, ws[0], w2, probs=probs, windows=windows, mse=mse)
                if t is not None]

    implicit = backward(None, g)
    assert g.dense is None, "the head backward materialised the gradient"
    again = backward(None, g)
    dense = backward(g.materialize().clone(), None)
    _assert_bitwise(implicit, dense, (c, channels, "implicit vs dense"))
    _assert_bitwise(implicit, again, (c, channels, "implicit twice"))


@pytest.mark.parametrize("c,h,w,channels,b,sigma", HEAD_CASES)
def test_head_backward_keypoint_loss_through_autograd(ops, dev, c, h, w, channels, b, sigma):
    """MSE loss + keypoint loss on a freshly initialised head through autograd, implicit against dense.  Every decode
    backward recomputes the decode windows, and a fresh head's flat planes all take the dense fallback (flag 2), whose
    row segments meet through float atomics (decode_bwd_kernel): its gradient differs in the last bits from call to
    call, and the bf16 rounding of the head's gradient operand carries that into every gradient.  So the flags and the
    valid windows are required to be the same bits, the fallback gradient to agree to 1e-6 of its largest value, and the head's
    gradients to agree to 1e-3 of the largest value of each weight gradient."""
    head = make_head(c, channels, seed=23)
    f = features(b, c, h, w, seed=24, dtype=torch.bfloat16).requires_grad_(True)
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    hm, kpp, _ = head.forward_with_keypoints(f)
    g_kp = torch.randn(kpp.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(25))
    oh, ow = hm.shape[-2:]
    kp, vis = _head_labels(b, channels[-1], oh, ow, sigma, dev)
    g = torch.autograd.grad(ops.heatmap_mse_from_keypoints(kp, hm, *HEAD_IMG, sigma, visibility=vis), hm, retain_graph=True)[0]
    implicit = [t.clone() for t in torch.autograd.grad([hm, kpp], [f] + params, [g, g_kp], retain_graph=True)]
    assert g.dense is None, "the head backward materialised the gradient"
    want = [t.clone() for t in torch.autograd.grad([hm, kpp], [f] + params, [g.materialize().clone(), g_kp], retain_graph=True)]
    # the decode windows of two calls: the same bits except the atomically summed fallback planes
    ds, temp = int(head.downsample_factor), float(head.temperature)
    _, _, stats = ops.decode_forward(hm.detach(), ds, temp)
    w1, w2 = (ops.decode_backward_windows(hm.detach(), stats, g_kp.reshape(kpp.shape[0], -1, 2), ds, temp) for _ in range(2))
    assert torch.equal(w1[1][:, 2], w2[1][:, 2])
    ok = w1[1][:, 2] == 1  # a valid window is written whole, with its dot; the fallback planes' windows are not written
    assert torch.equal(w1[1][ok], w2[1][ok]) and torch.equal(w1[0][ok], w2[0][ok])
    fb = w1[1][:, 2] == 2
    assert bool(fb.any())
    o1, o2 = w1[2].reshape(fb.shape[0], -1)[fb], w2[2].reshape(fb.shape[0], -1)[fb]
    assert float((o1 - o2).abs().max()) <= 1e-6 * float(o1.abs().max())
    worst = 0.0
    names = ["dfeat"] + [f"{n}{i}" for i in range(1, len(params) // 2 + 1) for n in ("dw", "db")]
    for i, (name, x, y) in enumerate(zip(names, implicit, want)):
        scale = float(want[i if name.startswith("d") and not name.startswith("db") else i - 1].float().abs().max())
        r = float((x.float() - y.float()).abs().max()) / (1e-3 * scale)
        assert r <= 1.0, (name, r)
        worst = max(worst, r)
    report(f"head backward keypoint loss implicit vs dense {c} {channels}", worst)


# ------------------------------------------------------------------------------------------------
# keypoints_mask_oob and evaluate_heatmaps_at_location
# ------------------------------------------------------------------------------------------------
def test_keypoints_mask_oob_edges(ops, dev, min_planes):
    """Bit for bit the restatement: x == width and y == height are out, one ulp below is in, -0.0 is in (and keeps its
    sign), NaN in one coordinate alone is kept, +-inf is out."""
    height, width = 406.0, 384.0
    ulp_below = lambda v: float(np.nextafter(np.float32(v), np.float32(0)))  # noqa: E731
    nan, inf = float("nan"), float("inf")
    vals = [0.0, -0.0, float(-np.float32(1e-45)), ulp_below(width), width, 12.5, nan, inf, -inf]
    yvals = [0.0, -0.0, float(-np.float32(1e-45)), ulp_below(height), height, 17.25, nan, inf, -inf]
    rows = torch.tensor([(x, y) for x in vals for y in yvals], dtype=torch.float32)
    reps = -(-min_planes // rows.shape[0])
    kp = rows.repeat(reps, 1).reshape(reps, rows.shape[0], 2).to(dev)
    got = ops.keypoints_mask_oob(kp, height, width)
    ref = TO.mask_oob(kp, height, width)
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    fin = ~torch.isnan(ref)
    assert torch.equal(got[fin].view(torch.int32), ref[fin].view(torch.int32))
    x, y = kp[..., 0], kp[..., 1]
    assert bool(torch.isnan(got[(x == width) & (y == 12.5)]).all()) and bool(torch.isnan(got[(y == height) & (x == 12.5)]).all())
    assert bool((~torch.isnan(got[(x == ulp_below(width)) & (y == 17.25)])).all())
    assert bool(torch.isnan(got[..., 0][torch.isnan(x) & (y == 17.25)]).all()) and bool((got[..., 1][torch.isnan(x) & (y == 17.25)] == 17.25).all())
    report("keypoints_mask_oob", 0.0)


@pytest.mark.parametrize("shape", [(96, 96), (64, 80), (128, 192)])
@pytest.mark.parametrize("radius", [1, 2, 3])
def test_evaluate_heatmaps_at_location_edges(ops, dev, min_planes, shape, radius):
    """Windows at 0, -0.5 (truncates to 0), w - 1 + 0.999, -0.0, on all four borders and the corners, and inside; within
    2e-6 of the float64 window sum on normalised planes."""
    hh, ww = shape
    xs = [0.0, -0.5, -0.0, ww - 1 + 0.999, ww - 1.0, 0.999, ww / 2 + 0.3]
    ys = [0.0, -0.5, -0.0, hh - 1 + 0.999, hh - 1.0, 0.999, hh / 2 + 0.7]
    rows = torch.tensor([(x, y) for x in xs for y in ys], dtype=torch.float32)
    reps = -(-min_planes // rows.shape[0])
    locs = rows.repeat(reps, 1).reshape(reps, rows.shape[0], 2).to(dev)
    heat = torch.rand(reps, rows.shape[0], hh, ww, device=dev, generator=torch.Generator(device=dev).manual_seed(radius)) ** 4
    heat = heat / heat.sum((-1, -2), keepdim=True) * 4.0  # peaky planes whose windows sum to O(0.01 .. 1)
    got = ops.evaluate_heatmaps_at_location(heat, locs, radius)
    ref = TO.window_sum(heat, locs, radius)
    err = float((got.double() - ref).abs().max())
    assert err <= 2e-6, err
    report(f"evaluate_heatmaps_at_location {shape} radius {radius}", err / 2e-6)
