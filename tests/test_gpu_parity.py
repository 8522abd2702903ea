"""GPU parity: the CUDA path (through the C-ABI) vs the golden vectors produced by the reference's own
code and vs the CPU oracle on seeded inputs.  Tolerances follow BASELINE.json's north star:
1e-4 relative in fp32 for heatmaps, decoded (x, y, confidence) and every loss scalar."""
import numpy as np
import pytest
import torch

from head_support import features, gen, grads, make_head, softmax_split
from oracle import lp_oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-4  # north_star: "within 1e-4 rel fp32"
T = torch.from_numpy


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


def close(a, b, atol=1e-6, rtol=RTOL):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    np.testing.assert_allclose(a, b, atol=atol, rtol=rtol, equal_nan=True)


# ------------------------------------------------------------------------------------------------
# decode (a3/a4/a5)
# ------------------------------------------------------------------------------------------------
def test_decode_reference_known_answers(lpb, dev, golden):
    g = golden("decode")
    for ds in (1, 2, 3):
        p, c = lpb.decode_softargmax(T(g[f"kat_ds{ds}_in"]).to(dev), ds, 1000.0)
        close(p, g[f"kat_ds{ds}_out_preds"], atol=2e-5)
        close(c, g[f"kat_ds{ds}_out_conf"], atol=1e-6)
    # tests/models/heads/test_heatmap.py:126-156: peaks at (2,2),(4,4) -> (8,8),(16,16), confidence 1
    p, c = lpb.decode_softargmax(T(g["kat_ds2_in"]).to(dev), 2, 1000.0)
    close(p[0, :4], [8.0, 8.0, 16.0, 16.0], atol=1e-5)
    close(c[0, :2], [1.0, 1.0], atol=1e-6)
    for temp in (1000, 100, 10):
        p, c = lpb.decode_softargmax(T(g["temp_in"]).to(dev), 2, float(temp))
        close(p, g[f"temp{temp}_out_preds"], atol=2e-5)
        close(c, g[f"temp{temp}_out_conf"], atol=1e-6)


@pytest.mark.parametrize("name", ["peaked", "flat", "edge", "multi", "raw"])
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_golden_regimes(lpb, dev, golden, name, ds):
    g = golden("decode")
    p, c = lpb.decode_softargmax(T(g[f"{name}_in"]).to(dev), ds, 1000.0)
    # flat planes: the expectation is a mean over ~1e4..1e5 almost-equal weights -> absolute tolerance
    close(p, g[f"{name}_ds{ds}_out_preds"], atol=5e-4 if name == "flat" else 5e-5)
    close(c, g[f"{name}_ds{ds}_out_conf"], atol=1e-6)


def test_decode_a3_table(lpb, dev, golden):
    g = golden("decode")
    t = lpb.generate_heatmaps(T(g["a3_in_keypoints"]).to(dev), 384, 384, (96, 96))
    close(t.sum((2, 3)), g["a3_out_targets_sum"], atol=2e-6)
    close(t.amax((2, 3)), g["a3_out_targets_peak"], atol=1e-7)
    p, c = lpb.decode_softargmax(t, 2, 1000.0)
    close(p, g["a3_out_preds"], atol=1e-4)
    close(c, g["a3_out_conf"], atol=2e-6)


@pytest.mark.parametrize("shape", [(2, 3, 96, 96), (1, 2, 30, 41), (2, 2, 8, 8), (1, 1, 5, 7), (1, 2, 128, 128)])
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_vs_oracle_shapes(lpb, dev, shape, ds):
    """Odd sizes exercise the non-TMA staging path (w % 4 != 0) and all-border planes."""
    b, k, h, w = shape
    gen = torch.Generator().manual_seed(100 + h + ds)
    kp = torch.rand(b, k, 2, generator=gen) * torch.tensor([w * 4.0, h * 4.0])
    hm = O.gaussian_targets(kp, 4 * h, 4 * w, (h, w)) + 1e-6
    hm = hm / hm.sum((2, 3), keepdim=True)
    po, co = O.decode_softargmax(hm, ds, 1000.0)
    p, c = lpb.decode_softargmax(hm.to(dev), ds, 1000.0)
    close(p, po, atol=1e-4)
    close(c, co, atol=2e-6)


def test_decode_fullsize_roundtrip_property(lpb, dev):
    """BASELINE config size (17 kpts, 96x96 -> 384x384), many frames: decode(generate(kp)) ~= kp.
    Size-independent property (SURVEY A.2: mean error 0.004 px, max 0.09 px away from borders)."""
    gen = torch.Generator().manual_seed(7)
    kp = (torch.rand(256, 17, 2, generator=gen) * 368 + 8).to(dev)
    hm = lpb.generate_heatmaps(kp, 384, 384, (96, 96)) + 1e-6
    hm = hm / hm.sum((2, 3), keepdim=True)
    p, c = lpb.decode_softargmax(hm, 2, 1000.0)
    err = (p.reshape(256, 17, 2) - kp).abs()
    assert float(err.max()) < 0.12 and float(err.mean()) < 0.01
    assert float(c.min()) > 0.99
    # plane-permutation equivariance: a checksum over shuffled planes is unchanged
    perm = torch.randperm(256 * 17, generator=gen).to(dev)
    hp = hm.reshape(-1, 1, 96, 96)[perm].reshape(256, 17, 96, 96)
    p2, c2 = lpb.decode_softargmax(hp, 2, 1000.0)
    assert torch.equal(p2.reshape(-1, 2), p.reshape(-1, 2)[perm]) and torch.equal(c2.reshape(-1), c.reshape(-1)[perm])


def test_decode_backward_vs_autograd(lpb, dev):
    gen = torch.Generator().manual_seed(11)
    logits = torch.randn(2, 3, 24 * 32, generator=gen) * 2.5
    hm = torch.softmax(logits, -1).reshape(2, 3, 24, 32)
    gxy = torch.randn(2, 6, generator=gen)
    ref = hm.clone().double().requires_grad_(True)
    field = ref
    for _ in range(2):  # float64 oracle of the same algorithm for a clean gradient reference
        up = torch.nn.functional.interpolate(field, scale_factor=2, mode="bicubic", align_corners=False)
        k = torch.outer(torch.tensor([1.0, 4, 6, 4, 1]), torch.tensor([1.0, 4, 6, 4, 1])).double() / 256
        field = torch.nn.functional.conv2d(torch.nn.functional.pad(up, (2, 2, 2, 2)), k.reshape(1, 1, 5, 5).repeat(3, 1, 1, 1), groups=3)
    p = torch.softmax(field.reshape(2, 3, -1) * 1000.0, -1).reshape(field.shape)
    ex = (p.sum(2) * torch.arange(p.shape[3], dtype=torch.double)).sum(-1)
    ey = (p.sum(3) * torch.arange(p.shape[2], dtype=torch.double)).sum(-1)
    (torch.stack([ex, ey], -1).reshape(2, 6) * gxy.double()).sum().backward()
    x = hm.to(dev).requires_grad_(True)
    preds, _ = lpb.decode_softargmax(x, 2, 1000.0)
    (preds * gxy.to(dev)).sum().backward()
    g_ref = ref.grad.float()
    scale = float(g_ref.abs().max())
    close(x.grad, g_ref, atol=2e-3 * scale, rtol=2e-3)


# ------------------------------------------------------------------------------------------------
# targets (a6) and windowed evaluation (a5)
# ------------------------------------------------------------------------------------------------
def test_generate_heatmaps_golden(lpb, dev, golden):
    g = golden("targets")
    kp, vis = T(g["in_keypoints"]).to(dev), T(g["in_visibility"]).to(dev)
    close(lpb.generate_heatmaps(kp, 48, 64, (12, 16)), g["out_vis_none"], atol=1e-7)
    close(lpb.generate_heatmaps(kp, 48, 64, (12, 16), visibility=vis), g["out_vis"], atol=1e-7)
    close(lpb.generate_heatmaps(kp, 48, 64, (24, 32), sigma=2.0), g["out_sigma2_ds1"], atol=1e-7)
    close(lpb.evaluate_heatmaps_at_location(T(g["eval_in_heatmaps"]).to(dev), T(g["eval_in_locs"]).to(dev)), g["eval_out"], atol=2e-6)


def test_generate_heatmaps_backward(lpb, dev):
    gen = torch.Generator().manual_seed(5)
    kp = torch.rand(3, 4, 2, generator=gen) * torch.tensor([64.0, 48.0])
    kp[0, 1] = torch.tensor([-9.0, 3.0])  # clamped + bad -> zero plane -> zero grad
    gout = torch.randn(3, 4, 12, 16, generator=gen)
    ref = kp.clone().double().requires_grad_(True)
    x = ref[..., 0] * (16 / 64)
    y = ref[..., 1] * (12 / 48)
    bad = (x < -1) | (x > 17) | (y < -1) | (y > 13)
    xc, yc = x.clamp(-1, 17)[..., None, None], y.clamp(-1, 13)[..., None, None]
    cols = torch.arange(16, dtype=torch.double)[None, None, None, :]
    rows = torch.arange(12, dtype=torch.double)[None, None, :, None]
    gmap = torch.exp(-((cols - xc) ** 2 + (rows - yc) ** 2) / (2 * 1.25**2))
    gmap = gmap / gmap.sum((2, 3), keepdim=True)
    gmap = torch.where(bad[..., None, None], torch.zeros_like(gmap), gmap)
    (gmap * gout.double()).sum().backward()
    k = kp.to(dev).requires_grad_(True)
    out = lpb.generate_heatmaps(k, 48, 64, (12, 16), keep_gradients=True)
    (out * gout.to(dev)).sum().backward()
    close(k.grad, ref.grad.float(), atol=1e-6, rtol=1e-3)


# ------------------------------------------------------------------------------------------------
# head (a1/a2)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,nl", [("resnet", 2), ("vit", 1)])
def test_head_golden(lpb, dev, golden, tag, nl):
    g = golden("head")
    ws = [T(g[f"{tag}_w{i}"]).to(dev) for i in range(nl)]
    bs = [T(g[f"{tag}_b{i}"]).to(dev) for i in range(nl)]
    f = T(g[f"{tag}_in_features"]).to(dev)
    close(lpb.head_forward(f, ws, bs, True), g[f"{tag}_out_heatmaps"], atol=1e-8)
    close(lpb.head_forward(f, ws, bs, False), g[f"{tag}_out_logits"], atol=2e-5)


@pytest.mark.parametrize("cfg", [(2048, (17, 17), 12, 12, 2), (384, (17,), 16, 16, 2), (512, (17, 17), 4, 6, 3)])
def test_head_module_vs_oracle(lpb, dev, cfg):
    """Real channel counts of BASELINE configs 2 and 3 (random weights with a peaked-logit gain)."""
    cin, ch, fh, fw, b = cfg
    k = ch[-1]
    head = make_head(cin, ch, seed=3, gain=2.0)
    feats = torch.randn(b, cin, fh, fw) * 0.5
    deconvs = list(head.upsampling_layers)[1:]
    ref = O.head_forward(feats, [d.weight.detach().cpu() for d in deconvs], [d.bias.detach().cpu() for d in deconvs])
    out = head(feats.to(dev))
    assert out.shape == ref.shape
    close(out, ref, atol=1e-9)
    close(out.sum((2, 3)), torch.ones(b, k), atol=1e-5)  # tests/models/heads/test_heatmap.py:260-273
    # reference state-dict keys / layouts load unchanged
    assert set(head.state_dict()) == {f"upsampling_layers.{i}.{n}" for i in range(1, len(deconvs) + 1) for n in ("weight", "bias")}


def test_head_backward_matches_oracle_autograd(lpb, dev):
    head = make_head(64, (5, 5), seed=4, gain=2.0)
    feats = torch.randn(2, 64, 3, 4)
    gout = torch.randn(2, 5, 24, 32)
    deconvs = list(head.upsampling_layers)[1:]
    f_ref = feats.clone().requires_grad_(True)
    ws = [d.weight.detach().cpu().requires_grad_(True) for d in deconvs]
    bs = [d.bias.detach().cpu().requires_grad_(True) for d in deconvs]
    (O.head_forward(f_ref, ws, bs) * gout).sum().backward()
    f = feats.to(dev).requires_grad_(True)
    (head(f) * gout.to(dev)).sum().backward()
    close(f.grad, f_ref.grad, atol=1e-7, rtol=1e-3)
    for d, w_ref in zip(list(head.upsampling_layers)[1:], ws):
        close(d.weight.grad, w_ref.grad, atol=1e-7, rtol=1e-3)


# ------------------------------------------------------------------------------------------------
# remap (a8/a9)
# ------------------------------------------------------------------------------------------------
def test_remap_golden(lpb, dev, golden):
    from lightning_pose_b200.data.bboxes import model_to_frame_batch
    from lightning_pose_b200.data.utils import undo_affine_transform_batch

    g = golden("remap")
    kp = T(g["in_keypoints"]).to(dev)
    close(undo_affine_transform_batch(kp.clone(), T(g["in_transform_shared"]).to(dev)), g["out_affine_shared"], atol=2e-5)
    close(undo_affine_transform_batch(kp.clone(), T(g["in_transform_perframe"]).to(dev)), g["out_affine_perframe"], atol=2e-5)
    close(undo_affine_transform_batch(kp.clone(), T(g["in_transform_multiview"]).to(dev), True), g["out_affine_multiview"], atol=2e-5)
    same = undo_affine_transform_batch(kp, torch.ones(1, device=dev))
    assert same is kp
    frames = torch.zeros(6, 3, 128, 256, device=dev)
    inp = kp.clone()
    out = model_to_frame_batch({"frames": frames, "bbox": T(g["in_bbox"]).to(dev), "is_multiview": False}, inp)
    close(out, g["out_frame_single"], atol=2e-5)
    close(inp, g["out_frame_single"], atol=2e-5)  # in-place through the caller's tensor, like the reference
    out = model_to_frame_batch({"frames": frames, "bbox": T(g["in_bbox_ctx"]).to(dev), "is_multiview": False}, kp.clone())
    close(out, g["out_frame_ctx"], atol=2e-5)
    out = model_to_frame_batch({"frames": frames, "bbox": T(g["in_bbox_mv"]).to(dev), "is_multiview": True}, kp.clone())
    close(out, g["out_frame_mv"], atol=2e-5)
    fused = lpb.remap_keypoints(kp, T(g["in_transform_shared"]).to(dev), T(g["in_bbox"]).to(dev), 128, 256)
    ref = O.model_to_frame(O.undo_affine(T(g["in_keypoints"]), T(g["in_transform_shared"])), T(g["in_bbox"]), 128, 256)
    close(fused, ref, atol=2e-5)


# ------------------------------------------------------------------------------------------------
# losses (a10-a16)
# ------------------------------------------------------------------------------------------------
def test_heatmap_losses_golden(lpb, dev, golden):
    from lightning_pose_b200.losses.losses import HeatmapJSLoss, HeatmapKLLoss, HeatmapMSELoss

    g = golden("losses")
    a = O.gaussian_targets(T(g["hm_in_a_kp"]), 384, 384, (96, 96)).to(dev)
    b = O.gaussian_targets(T(g["hm_in_b_kp"]), 384, 384, (96, 96)).to(dev)
    targ = O.gaussian_targets(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"])).to(dev)
    pred = T(g["hmb_in_pred"]).to(dev)
    for nm, cls in (("mse", HeatmapMSELoss), ("kl", HeatmapKLLoss), ("js", HeatmapJSLoss)):
        v, logs = cls()(heatmaps_targ=b, heatmaps_pred=a, stage="train")
        close(v, g[f"hm_{nm}_out_targb_preda"], atol=1e-7)
        assert logs[0]["name"] == f"train_heatmap_{nm}_loss" and logs[1]["name"] == f"heatmap_{nm}_weight"
        v, _ = cls()(heatmaps_targ=a, heatmaps_pred=b)
        close(v, g[f"hm_{nm}_out_targa_predb"], atol=1e-7)
        v, _ = cls()(heatmaps_targ=targ, heatmaps_pred=pred)
        close(v, g[f"hmb_{nm}_out"], atol=1e-7)
    fused = lpb.heatmap_mse_from_keypoints(T(g["hmb_in_kp"]).to(dev), pred, 128, 128, visibility=T(g["hmb_in_vis"]).to(dev))
    close(fused, g["hmb_mse_out"], atol=1e-7)


@pytest.mark.parametrize("kind", ["mse", "kl", "js"])
def test_heatmap_loss_backward(lpb, dev, golden, kind):
    g = golden("losses")
    targ = O.gaussian_targets(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"]))
    pred = T(g["hmb_in_pred"])
    fn = {"mse": O.heatmap_mse_loss, "kl": O.heatmap_kl_loss, "js": O.heatmap_js_loss}[kind]
    pr = pred.clone().requires_grad_(True)
    (fn(targ, pr) * 1.7).backward()
    p = pred.to(dev).requires_grad_(True)
    (lpb.heatmap_loss(targ.to(dev), p, kind) * 1.7).backward()
    close(p.grad, pr.grad, atol=1e-7, rtol=1e-3)


def test_unsup_losses_golden(lpb, dev, golden):
    from lightning_pose_b200.losses.losses import TemporalLoss

    g = golden("losses")
    kp, conf = T(g["temporal_in_kp"]).to(dev), T(g["temporal_in_conf"]).to(dev)
    tl = TemporalLoss(epsilon=[2.0, 20.0], prob_threshold=0.05)
    v, _ = tl(kp, conf)
    close(v, 3.8, atol=1e-6)  # SURVEY A.3 / tests/losses/test_losses.py:343-392
    v, _ = tl(kp)
    close(v, 5.8, atol=1e-6)
    v, _ = TemporalLoss(epsilon=20.0, prob_threshold=0.05)(T(g["temporal2_in_kp"]).to(dev), T(g["temporal2_in_conf"]).to(dev))
    close(v, g["temporal2_out"], atol=1e-6)
    kseq = T(g["pca_in_kp"]).to(dev)
    cols = g["pca_sv_cols"].tolist()
    for centering in (None, "mean", "median"):
        p = lpb.PcaParams(np.asarray(cols, np.int32), len(cols), 0, centering, g["pca_sv_mean"], g["pca_sv_kept"], 2.5, dev)
        close(lpb.unsup_losses(kseq, pca_singleview=p)[1], g[f"pca_sv_out_{centering}"], atol=1e-5)
    mcm = g["pca_mv_mcm"]
    p = lpb.PcaParams(mcm.reshape(-1).astype(np.int32), mcm.shape[1], mcm.shape[0], None, g["pca_mv_mean"], g["pca_mv_kept"], 0.7, dev)
    close(lpb.unsup_losses(kseq, pca_multiview=p)[2], g["pca_mv_out"], atol=1e-5)
    # batched clips: every clip equals the single-clip result
    out = lpb.unsup_losses(torch.stack([kseq, kseq.flip(0)]), temporal_eps=1.0, pca_multiview=p)
    close(out[0, 2], g["pca_mv_out"], atol=1e-5)
    close(out[1, 0], out[0, 0], atol=1e-5)


def test_unsup_losses_backward(lpb, dev, golden):
    g = golden("losses")
    kseq, conf = T(g["pca_in_kp"]), torch.rand(32, 17, generator=torch.Generator().manual_seed(2))
    cols = g["pca_sv_cols"].tolist()
    mcm = g["pca_mv_mcm"]
    for centering in (None, "mean", "median"):
        ref = kseq.clone().requires_grad_(True)
        tot = (
            1.3 * O.temporal_loss(ref, conf, 3.0, 0.2)
            + 0.7 * O.pca_loss(O.pca_format_singleview(ref, cols, centering), T(g["pca_sv_mean"]), T(g["pca_sv_kept"]), 2.5)
            + 2.1 * O.pca_loss(O.pca_format_multiview(ref, mcm.tolist()), T(g["pca_mv_mean"]), T(g["pca_mv_kept"]), 0.7)
        )
        tot.backward()
        x = kseq.to(dev).requires_grad_(True)
        sv = lpb.PcaParams(np.asarray(cols, np.int32), len(cols), 0, centering, g["pca_sv_mean"], g["pca_sv_kept"], 2.5, dev)
        mv = lpb.PcaParams(mcm.reshape(-1).astype(np.int32), mcm.shape[1], mcm.shape[0], None, g["pca_mv_mean"], g["pca_mv_kept"], 0.7, dev)
        out = lpb.unsup_losses(x, conf.to(dev), temporal_eps=3.0, prob_threshold=0.2, pca_singleview=sv, pca_multiview=mv)
        close(1.3 * out[0] + 0.7 * out[1] + 2.1 * out[2], tot, atol=1e-5)
        (1.3 * out[0] + 0.7 * out[1] + 2.1 * out[2]).backward()
        close(x.grad, ref.grad, atol=1e-6, rtol=1e-3)


def test_temporal_heatmap_and_reprojection_golden(lpb, dev, golden):
    from lightning_pose_b200.losses.losses import ReprojectionHeatmapLoss, TemporalHeatmapLoss

    g = golden("losses")
    hseq, cseq = T(g["thm_in_heatmaps"]).to(dev), T(g["thm_in_conf"]).to(dev)
    v, _ = TemporalHeatmapLoss("temporal_heatmap_mse", epsilon=1e-5, prob_threshold=0.2)(hseq, cseq)
    close(v, g["thm_mse_out"], atol=1e-8)
    v, _ = TemporalHeatmapLoss("temporal_heatmap_kl", epsilon=[0.5, 1.0, 2.0], prob_threshold=0.2)(hseq, cseq)
    close(v, g["thm_kl_out"], atol=1e-6)
    targ = O.gaussian_targets(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"])).to(dev)
    v, _ = ReprojectionHeatmapLoss(128, 128, 32, 32, log_weight=1.0)(heatmaps_targ=targ, keypoints_pred_2d_reprojected=T(g["reproj_in_kp"]).to(dev))
    close(v, g["reproj_out"], atol=1e-7)


def test_loss_factory_golden(lpb, dev, golden):
    from lightning_pose_b200.losses.factory import LossFactory

    g = golden("losses")
    targ = O.gaussian_targets(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"])).to(dev)
    fac = LossFactory({"heatmap_mse": {"log_weight": 0.0}, "temporal": {"log_weight": 5.0, "epsilon": 20.0, "prob_threshold": 0.05}}, None)
    tot, logs = fac(stage="train", anneal_weight=0.3, heatmaps_targ=targ, heatmaps_pred=T(g["hmb_in_pred"]).to(dev),
                    keypoints_pred=T(g["temporal2_in_kp"]).to(dev), confidences=T(g["temporal2_in_conf"]).to(dev))
    close(tot, g["factory_out_total"], atol=1e-7)
    assert [d["name"] for d in logs] == g["factory_log_names"].tolist()
    close(torch.stack([torch.as_tensor(d["value"]).float().cpu() for d in logs]), g["factory_log_values"], atol=1e-7)


def test_tracker_semisupervised_step_vs_oracle(lpb, dev):
    """End to end through the mirrored boundary (HeatmapHead -> decode -> remap -> LossFactory)."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(9)
    head = HeatmapHead("resnet50", 256, 17)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=2.5)
    feats = torch.randn(8, 256, 4, 4) * 0.5
    bbox = torch.tensor([[3.0, 5.0, 200.0, 260.0]]).repeat(8, 1)
    ang = 0.1
    tf = torch.tensor([[1.05 * np.cos(ang), -1.05 * np.sin(ang), 2.0], [1.05 * np.sin(ang), 1.05 * np.cos(ang), -1.0]], dtype=torch.float32)
    deconvs = list(head.upsampling_layers)[1:]
    hm_ref = O.head_forward(feats, [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs])
    kp_ref, cf_ref = O.decode_softargmax(hm_ref, 2, 1000.0)
    kp_ref = O.model_to_frame(O.undo_affine(kp_ref, tf), bbox, 128, 128)
    loss_ref = O.temporal_loss(kp_ref, cf_ref, 2.0, 0.05)

    head = head.to(dev)
    hm = head(feats.to(dev))
    kp, cf = head.run_subpixelmaxima(hm)
    kp = lpb.remap_keypoints(kp, tf.to(dev), bbox.to(dev), 128, 128)
    fac = LossFactory({"temporal": {"log_weight": 0.0, "epsilon": 2.0, "prob_threshold": 0.05}}, None)
    tot, _ = fac(stage=None, keypoints_pred=kp, confidences=cf)
    close(hm, hm_ref, atol=1e-9)
    close(kp, kp_ref, atol=2e-3, rtol=RTOL)
    close(cf, cf_ref, atol=1e-5)
    close(tot, 0.5 * loss_ref, atol=1e-4)


@pytest.mark.gpu
def test_head_bf16_backward_is_bitwise_reproducible(lpb, dev):
    """lpb_head_bwd_bf16 sums its gradients over CTAs in a fixed order: two identical backward calls (dense gradient of the
    softmax output, enough frames for many weight-gradient and b2d CTAs) give bit-identical gradients."""
    b, k = 64, 17
    head = make_head(2048, (k, k), seed=31)
    feats = features(b, 2048, 12, 12, 32, torch.bfloat16)
    gout = torch.randn(b, k, 96, 96, device=dev, generator=gen(33))
    runs = [grads(head, feats, gout) for _ in range(2)]
    assert list(runs[0]) == ["dfeat", "dw1", "db1", "dw2", "db2"]
    for name in runs[0]:
        assert torch.equal(runs[0][name], runs[1][name]), name


def _peaked_heatmaps(b, k, h, w, seed, sigma=1.6):
    g = torch.Generator().manual_seed(seed)
    cy = torch.rand(b, k, 1, 1, generator=g) * (h - 1)
    cx = torch.rand(b, k, 1, 1, generator=g) * (w - 1)
    yy = torch.arange(h).view(1, 1, h, 1).float()
    xx = torch.arange(w).view(1, 1, 1, w).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sigma**2) * 1.0 + 0.05 * torch.randn(b, k, h, w, generator=g)
    return torch.softmax(logits.reshape(b, k, -1), -1).reshape(b, k, h, w)


@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_backward_windows_match_dense(lpb, dev, ds):
    """lpb_decode_bwd_windows: the 32x32 windows (+ overflow planes) re-assembled equal lpb_decode_bwd, and
    meta's dot equals sum(g * heatmap); includes peaks at the border, zero-gradient planes and diffuse planes
    that must take the dense fallback."""
    from lightning_pose_b200 import ops

    b, k, h, w = 3, 6, 48, 40
    hm = _peaked_heatmaps(b, k, h, w, seed=5 + ds)
    hm[0, 0] = torch.softmax(torch.randn(h * w, generator=torch.Generator().manual_seed(1)) * 0.01, 0).reshape(h, w)  # diffuse
    hm[1, 1] = 0.0
    hm[1, 1, 0, 0] = 1.0  # corner peak
    hm = hm.to(dev).contiguous()
    xy, conf, stats = ops._decode_fwd(hm, ds, 1000.0)
    gxy = torch.randn(b, k, 2, generator=torch.Generator().manual_seed(2)).to(dev)
    gxy[2, 3] = 0.0  # zero-gradient plane
    dense = ops._decode_bwd(hm, stats, gxy, ds, 1000.0)
    win, meta, ov = ops.decode_backward_windows(hm, stats, gxy, ds, 1000.0)
    meta_c, win_c = meta.cpu(), win.cpu()
    rebuilt = torch.zeros(b * k, h, w)
    flags = meta_c[:, 2].tolist()
    assert flags[0] == 2 and flags[2 * k + 3] == 0 and flags.count(1) >= b * k - 3
    for pl in range(b * k):
        r0, c0, flag, dbits = meta_c[pl].tolist()
        if flag == 2:
            rebuilt[pl] = ov.reshape(b * k, h, w)[pl].cpu()
        elif flag == 1:
            ys = [(r0 + i, i) for i in range(32) if 0 <= r0 + i < h]
            xs = [(c0 + j, j) for j in range(32) if 0 <= c0 + j < w]
            sub = win_c[pl][[i for _, i in ys]][:, [j for _, j in xs]]
            rebuilt[pl][ys[0][0] : ys[-1][0] + 1, xs[0][0] : xs[-1][0] + 1] = sub
            # nothing may fall outside the plane
            mask = torch.ones(32, 32, dtype=torch.bool)
            mask[[i for _, i in ys][0] : [i for _, i in ys][-1] + 1, [j for _, j in xs][0] : [j for _, j in xs][-1] + 1] = False
            assert float(win_c[pl][mask].abs().max() if mask.any() else 0.0) == 0.0
            dot = torch.tensor([dbits], dtype=torch.int32).view(torch.float32).item()
            ref_dot = float((dense.reshape(b * k, h, w)[pl].cpu() * hm.reshape(b * k, h, w)[pl].cpu()).sum())
            assert abs(dot - ref_dot) <= 1e-4 * max(1.0, abs(ref_dot)) + 1e-6
    d = dense.reshape(b * k, h, w).cpu()
    close(rebuilt, d, atol=2e-5 * float(d.abs().max()), rtol=1e-4)


@pytest.mark.parametrize("use_dense", [True, False])
def test_head_with_keypoints_fused_backward_vs_oracle(lpb, dev, use_dense):
    """forward_with_keypoints: heatmaps + soft-argmax keypoints from one node; its single fused backward (decode
    windows [+ dense heatmap-loss gradient] + softmax backward folded into the deconv-gradient operand) against
    oracle autograd.  The soft-argmax gradient (T = 1000: exponentially sensitive to the heatmap values) is taken
    by oracle autograd AT the kernel's heatmaps; everything else is the oracle's own fp32 chain."""
    import torch.nn.functional as F

    b, c, fh, fw, k = 6, 2048, 12, 12, 17
    head = make_head(c, (k, k), seed=31, gain=4.0)
    feats = (torch.randn(b, c, fh, fw) * 0.5).bfloat16()
    g_hm = torch.randn(b, k, 8 * fh, 8 * fw) if use_dense else None
    g_kp = torch.randn(b, 2 * k)
    f_dev = feats.to(dev).requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f_dev)
    loss = (kp * g_kp.to(dev)).sum()
    if use_dense:
        loss = loss + (hm * g_hm.to(dev)).sum()
    loss.backward()
    # oracle
    hm_k = hm.detach().cpu().requires_grad_(True)
    kp_o, cf_o = O.decode_softargmax(hm_k, 2, 1000.0)
    close(kp, kp_o.detach(), atol=2e-3, rtol=RTOL)
    close(cf, cf_o.detach(), atol=1e-4, rtol=1e-3)
    (kp_o * g_kp).sum().backward()
    g_total = hm_k.grad + (g_hm if use_dense else 0.0)
    r = lambda t: (t.bfloat16().float() - t).detach() + t
    d1, d2 = [m.cpu() for m in list(head.upsampling_layers)[1:]]
    f_ref = feats.float().requires_grad_(True)
    p_ref = [t.detach().clone().requires_grad_(True) for t in (d1.weight, d1.bias, d2.weight, d2.bias)]
    mid = F.conv_transpose2d(F.pixel_shuffle(f_ref, 2), r(p_ref[0]), p_ref[1], stride=2, padding=1, output_padding=1)
    mid.retain_grad()
    y = O.spatial_softmax2d(F.conv_transpose2d(r(mid), r(p_ref[2]), p_ref[3], stride=2, padding=1, output_padding=1), 1.0)
    y.backward(g_total)
    # Bias gradients of a softmax head are sums that cancel (db2 is exactly 0, db1 only sees the image border):
    # what is left of them in bf16 is the random-walk rounding noise of the gradient operand,
    # 2^-8 * ||d mid||_2 per channel -- that, not max|ref|, is the meaningful error scale for them.
    noise1 = 2.0**-8 * mid.grad.pow(2).sum((0, 2, 3)).sqrt()
    for name, got, ref in [("dfeat", f_dev.grad.float(), f_ref.grad), ("dw1", d1.weight.grad, p_ref[0].grad), ("db1", d1.bias.grad, p_ref[1].grad),
                           ("dw2", d2.weight.grad, p_ref[2].grad), ("db2", d2.bias.grad, p_ref[3].grad)]:
        err = (got.cpu() - ref).abs()
        if name == "db1":
            assert bool((err <= 2e-2 * ref.abs().max() + 4.0 * noise1).all()), (name, err, noise1)
            continue
        scale = float(ref.abs().max()) if name != "db2" else float(p_ref[2].grad.abs().max())
        assert float(err.max()) <= 2e-2 * scale + 1e-9, (name, float(err.max()), scale)


def test_decode_multimodal_random_fields(lpb, dev):
    """Random spiky planes (several comparable peaks scattered over the plane) exercise the per-strip
    candidate row ranges; widths beyond the 1024-column field limit are rejected loudly."""
    gen = torch.Generator().manual_seed(21)
    hm = torch.softmax(torch.randn(3, 4, 96 * 96, generator=gen) * 4.0, -1).reshape(3, 4, 96, 96)
    po, co = O.decode_softargmax(hm, 2, 1000.0)
    p, c = lpb.decode_softargmax(hm.to(dev), 2, 1000.0)
    close(p, po, atol=2e-4)
    close(c, co, atol=2e-6)
    with pytest.raises(RuntimeError, match="field limit"):
        lpb.decode_softargmax(torch.rand(1, 1, 4, 300, device=dev), 2, 1000.0)


def test_semisupervised_tracker_training_step(lpb, dev):
    """Boundary row a7: the mirrored SemiSupervisedHeatmapTracker (backbone -> head -> decode -> remap -> loss
    factories) against the oracle evaluated on the same backbone features; gradients reach the backbone."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import SemiSupervisedHeatmapTracker

    k = 5
    sup = LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)
    unsup = LossFactory({"temporal": {"log_weight": 1.0, "epsilon": 1.0, "prob_threshold": 0.0}}, None)
    model = SemiSupervisedHeatmapTracker(k, loss_factory=sup, loss_factory_unsupervised=unsup, backbone="resnet18").to(dev)
    for layer in list(model.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    model.train(False)  # BN in eval mode: deterministic features
    gen = torch.Generator().manual_seed(3)
    imgs = torch.randn(4, 3, 64, 96, generator=gen)
    frames = torch.randn(6, 3, 64, 96, generator=gen)
    kps = torch.rand(4, k, 2, generator=gen) * torch.tensor([96.0, 64.0])
    bbox_l = torch.tensor([[1.0, 2.0, 128.0, 192.0]]).repeat(4, 1)
    bbox_u = torch.tensor([[0.0, 0.0, 64.0, 96.0]]).repeat(6, 1)
    targ = O.gaussian_targets(kps, 64, 96, (16, 24))
    batch = {
        "labeled": {"images": imgs.to(dev), "keypoints": kps.reshape(4, -1).to(dev), "heatmaps": targ.to(dev), "bbox": bbox_l.to(dev)},
        "unlabeled": {"frames": frames.to(dev), "transforms": torch.ones(1, device=dev), "bbox": bbox_u.to(dev), "is_multiview": False},
    }
    out = model.training_step(batch, 0)
    out["loss"].backward()
    assert model.backbone[0].weight.grad is not None and torch.isfinite(model.backbone[0].weight.grad).all()
    with torch.no_grad():
        fl = model.backbone(imgs.to(dev)).cpu()
        fu = model.backbone(frames.to(dev)).cpu()
    d = list(model.head.upsampling_layers)[1:]
    ws, bs = [x.weight.detach().cpu() for x in d], [x.bias.detach().cpu() for x in d]
    hl, hu = O.head_forward(fl, ws, bs), O.head_forward(fu, ws, bs)
    ku, cu = O.decode_softargmax(hu, 2, 1000.0)
    ku = O.model_to_frame(ku, bbox_u, 64, 96)
    ref = 0.5 * O.heatmap_mse_loss(targ, hl) + O.loss_weight(1.0) * O.temporal_loss(ku, cu, 1.0, 0.0)
    close(out["loss"], ref, atol=1e-5, rtol=2e-4)
    pk, pc = model.predict_step(batch["unlabeled"], 0)
    close(pk, ku, atol=2e-3, rtol=RTOL)
    kl, _ = O.decode_softargmax(hl, 2, 1000.0)
    close(model.last_rmse, O.model_to_frame(kl, bbox_l, 64, 96).sub(O.model_to_frame(kps.reshape(4, -1), bbox_l, 64, 96)).reshape(-1, 2).pow(2).mean(1).sqrt().mean(), atol=1e-3, rtol=1e-3)


def test_remap_and_fused_mse_backward(lpb, dev, golden):
    g = golden("remap")
    kp0 = T(g["in_keypoints"])
    tf, bbox = T(g["in_transform_perframe"]), T(g["in_bbox"])
    wgt = torch.randn(kp0.shape, generator=torch.Generator().manual_seed(1))
    ref = kp0.clone().requires_grad_(True)
    (O.model_to_frame(O.undo_affine(ref, tf), bbox, 128, 256) * wgt).sum().backward()
    x = kp0.to(dev).requires_grad_(True)
    (lpb.remap_keypoints(x, tf.to(dev), bbox.to(dev), 128, 256) * wgt.to(dev)).sum().backward()
    close(x.grad, ref.grad, atol=1e-6, rtol=1e-4)
    gl = golden("losses")
    kp, vis, pred = T(gl["hmb_in_kp"]), T(gl["hmb_in_vis"]), T(gl["hmb_in_pred"])
    pr = pred.clone().requires_grad_(True)
    (O.heatmap_mse_loss(O.gaussian_targets(kp, 128, 128, (32, 32), visibility=vis), pr) * 1.3).backward()
    p = pred.to(dev).requires_grad_(True)
    (lpb.heatmap_mse_from_keypoints(kp.to(dev), p, 128, 128, visibility=vis.to(dev)) * 1.3).backward()
    close(p.grad, pr.grad, atol=1e-8, rtol=1e-3)


# ------------------------------------------------------------------------------------------------
# round 2: upsample (a3), TemporalHeatmapLoss backward (a14), every BASELINE config on native kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,n,stages", [("U_n16_ds1", 16, 1), ("U_n16_ds2", 16, 2), ("U_n12_ds3", 12, 3), ("U_n96_ds2", 96, 2)])
def test_upsample2x_matches_reference_operator(lpb, dev, golden, key, n, stages):
    """a3: `upsample` (heads/heatmap.py:86-100) is the separable operator U h U^T; the golden U matrices are the
    reference's own impulse responses (oracle/gen_golden.py)."""
    U = torch.from_numpy(golden("decode")[key]).double()
    torch.manual_seed(5)
    h = torch.rand(2, 3, n, n)
    x = h.to(dev)
    for _ in range(stages):
        x = lpb.upsample2x(x)
    ref = torch.einsum("ia,bkac,jc->bkij", U, h.double(), U).float()
    assert x.shape == ref.shape
    close(x, ref, atol=2e-6)
    # and against the oracle's restatement of the same function on a non-square plane
    h2 = torch.rand(1, 2, 10, 14)
    close(lpb.upsample2x(h2.to(dev)), O.upsample(h2), atol=2e-6)


@pytest.mark.parametrize("kind,eps", [("mse", 1e-5), ("kl", [0.5, 1.0, 2.0])])
def test_temporal_heatmap_loss_backward(lpb, dev, golden, kind, eps):
    """a14: the reference trains through TemporalHeatmapLoss (losses.py:793-854); gradient vs oracle autograd."""
    from lightning_pose_b200.losses.losses import TemporalHeatmapLoss

    g = golden("losses")
    hseq, cseq = T(g["thm_in_heatmaps"]), T(g["thm_in_conf"])
    h_ref = hseq.clone().requires_grad_(True)
    O.temporal_heatmap_loss(h_ref, cseq, kind, eps, 0.2).backward()
    h = hseq.to(dev).requires_grad_(True)
    v, _ = TemporalHeatmapLoss(f"temporal_heatmap_{kind}", epsilon=eps, prob_threshold=0.2)(h, cseq.to(dev))
    close(v, g[f"thm_{kind}_out"])
    (3.0 * v).backward()
    assert h.grad is not None and float(h.grad.abs().max()) > 0
    close(h.grad, 3.0 * h_ref.grad, atol=1e-7, rtol=1e-4)


def test_head_fused_keypoints_backward_one_deconv(lpb, dev):
    """config-3 head (ViT, one deconv): forward_with_keypoints + sparse decode windows through the banded kernels."""
    b, c, fh, fw = 4, 384, 16, 16
    head = make_head(c, (17,), seed=37, gain=6.0)
    feats = (torch.randn(b, c, fh, fw) * 0.7).bfloat16()
    f1 = feats.to(dev).requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f1)
    gk = torch.randn_like(kp)
    (kp * gk).sum().backward()
    g_fused = f1.grad.float().clone()
    w_fused = list(head.upsampling_layers)[1].weight.grad.clone()
    # the same through the dense decode backward on the head's own (already verified) dense path
    head.zero_grad()
    f2 = feats.to(dev).requires_grad_(True)
    hm2 = head(f2)
    kp2, _ = lpb.decode_softargmax(hm2, 2, 1000.0)
    close(kp2, kp, atol=1e-4)
    (kp2 * gk).sum().backward()
    sc = float(f2.grad.float().abs().max())
    assert float((g_fused - f2.grad.float()).abs().max()) <= 2e-2 * sc + 1e-9
    wg = list(head.upsampling_layers)[1].weight.grad
    assert float((w_fused - wg).abs().max()) <= 2e-2 * float(wg.abs().max()) + 1e-9


@pytest.mark.parametrize("cfg", [(512, (17, 17), 4, 6, 2), (64, (5,), 5, 7, 2), (256, (7, 7, 7), 3, 3, 2)])
def test_head_fp32_native_backward_any_depth(lpb, dev, cfg):
    """fp32 precision path: 1-, 2- and 3-deconv heads (downsample_factor 1 on a stride-32 backbone -> 3 layers,
    heads/heatmap.py:192-193) train through the native CUDA-core backward; no library convolution anywhere."""
    cin, ch, fh, fw, b = cfg
    head = make_head(cin, ch, seed=8, gain=2.0)
    deconvs = list(head.upsampling_layers)[1:]
    feats = torch.randn(b, cin, fh, fw)
    f_ref = feats.clone().requires_grad_(True)
    ws = [d.weight.detach().cpu().requires_grad_(True) for d in deconvs]
    bs = [d.bias.detach().cpu().requires_grad_(True) for d in deconvs]
    ref = O.head_forward(f_ref, ws, bs)
    gout = torch.randn_like(ref)
    (ref * gout).sum().backward()
    f = feats.to(dev).requires_grad_(True)
    out = head(f)
    close(out, ref, atol=1e-9)
    (out * gout.to(dev)).sum().backward()
    close(f.grad, f_ref.grad, atol=1e-7, rtol=1e-3)
    for d, w_ref, b_ref in zip(deconvs, ws, bs):  # atomically accumulated fp32 sums: absolute floor ~ a few ulps of the largest entries
        close(d.weight.grad, w_ref.grad, atol=1e-6 * max(1.0, float(w_ref.grad.abs().max())), rtol=1e-3)
        close(d.bias.grad, b_ref.grad, atol=2e-6, rtol=1e-3)


@pytest.mark.parametrize("size", [None, (64, 96), (50, 70)])
@pytest.mark.parametrize("dtype,channels_last", [(torch.float32, False), (torch.bfloat16, False), (torch.bfloat16, True)])
def test_video_ingest_boundary(lpb, dev, size, dtype, channels_last):
    """f4: uint8 frames -> normalised FCHW (reference dali.py:157-197: resize, /255, crop_mirror_normalize)."""
    import torch.nn.functional as F
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    torch.manual_seed(2)
    u8 = torch.randint(0, 256, (5, 100, 140, 3), dtype=torch.uint8)
    x = u8.permute(0, 3, 1, 2).float()
    if size is not None:
        x = F.interpolate(x, size=size, mode="bilinear", align_corners=False, antialias=False)
    mean, std = torch.tensor(lpb.IMAGENET_MEAN).view(1, 3, 1, 1), torch.tensor(lpb.IMAGENET_STD).view(1, 3, 1, 1)
    ref = (x / 255.0 - mean) / std
    bd = frames_to_unlabeled_batch(u8.to(dev), resize_dims=size, dtype=dtype, channels_last=channels_last)
    got = bd["frames"].float().cpu()
    if channels_last:
        got = got.permute(0, 3, 1, 2)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    close(got, ref, atol=tol, rtol=1e-4 if dtype == torch.float32 else 1e-2)
    assert bd["is_multiview"] is False and bd["transforms"].tolist() == [-1.0]
    close(bd["bbox"], torch.tensor([[0.0, 0.0, 100.0, 140.0]]).repeat(5, 1))
    mv = frames_to_unlabeled_batch([u8.to(dev), u8.flip(0).to(dev)], resize_dims=size, dtype=dtype)
    assert mv["is_multiview"] and mv["frames"].shape[:3] == (5, 2, 3) and mv["bbox"].shape == (5, 8) and mv["transforms"].shape == (2, 1)


def test_tracker_on_gpu_target_pipeline(lpb, dev):
    """f2: a labeled batch that ships (keypoints, visibility) only - targets rendered inside the supervised loss - gives
    the loss / gradients of the reference flow (worker-rendered ``heatmaps``), out-of-frame rule included."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    torch.manual_seed(12)
    k, b, img = 6, 3, 64

    class Backbone(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 64, 3, stride=32, padding=1)

        def forward(self, x):
            return self.conv(x)

    def make():
        torch.manual_seed(77)
        t = HeatmapTracker(k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None), backbone=Backbone(), num_fc_input_features=64).to(dev)
        for layer in list(t.head.upsampling_layers)[1:]:
            torch.nn.init.xavier_uniform_(layer.weight, gain=2.0)
        return t

    images = torch.randn(b, 3, img, img)
    kp = torch.rand(b, k, 2) * img
    kp[0, 1] = torch.tensor([-3.0, 10.0])   # moved out of the frame by an augmentation -> NaN -> zero plane
    kp[1, 2] = torch.tensor([20.0, 64.0])   # y == height is out
    kp[2, 0] = float("nan")
    vis = torch.randint(0, 3, (b, k))
    bbox = torch.tensor([[0.0, 0.0, float(img), float(img)]]).repeat(b, 1)
    kp_masked = kp.clone()
    oob = (kp[..., 0] < 0) | (kp[..., 1] < 0) | (kp[..., 0] >= img) | (kp[..., 1] >= img)
    kp_masked[oob] = float("nan")
    targets = O.gaussian_targets(kp_masked, img, img, (16, 16), visibility=vis)
    t_ref = make()
    l_ref = t_ref.evaluate_labeled({"images": images.to(dev), "keypoints": kp_masked.reshape(b, -1).to(dev).clone(), "heatmaps": targets.to(dev), "bbox": bbox.to(dev)}, "train", 1.0)
    l_ref.backward()
    t_new = make()
    l_new = t_new.evaluate_labeled({"images": images.to(dev), "keypoints": kp.reshape(b, -1).to(dev).clone(), "visibility": vis.to(dev), "bbox": bbox.to(dev)}, "train", 1.0)
    l_new.backward()
    close(l_new, l_ref, atol=1e-7)
    for p_new, p_ref in zip(t_new.parameters(), t_ref.parameters()):
        close(p_new.grad, p_ref.grad, atol=1e-7, rtol=1e-3)
    close(t_new.last_rmse, t_ref.last_rmse, atol=1e-5)


# ------------------------------------------------------------------------------------------------
# MHCRNN context head (a17 / a18 / f3)
# ------------------------------------------------------------------------------------------------
def _load_mhcrnn(g, tag, arch, cin, uf, dev):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    head = HeatmapMHCRNNHead(arch, cin, 5, upsampling_factor=uf)
    sd = {k[len(f"{tag}_param_"):]: T(g[k]) for k in g.files if k.startswith(f"{tag}_param_")}
    for k in list(sd):  # the ModuleList aliases share storage with the named modules
        pass
    missing, unexpected = head.load_state_dict(sd, strict=False)
    assert not unexpected and all(".layers." in m for m in missing), (missing, unexpected)
    return head.to(dev)


def _mhcrnn_oracle_params(head):
    m = head.head_mf
    c = lambda t: t.detach().cpu().clone()
    p = {"W_f": (c(m.W_f.weight), c(m.W_f.bias)), "W_b": (c(m.W_b.weight), c(m.W_b.bias)),
         "H_f": tuple(c(t) for t in (m.H_f[0].weight, m.H_f[0].bias, m.H_f[1].weight, m.H_f[1].bias)),
         "H_b": tuple(c(t) for t in (m.H_b[0].weight, m.H_b[0].bias, m.H_b[1].weight, m.H_b[1].bias))}
    if m.upsampling_factor == 2:
        p["W_pre"] = (c(m.W_pre.weight), c(m.W_pre.bias))
    return p


def test_context_gather_golden(lpb, dev, golden):
    g = golden("mhcrnn")
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import get_context_from_sequence

    out = get_context_from_sequence(T(g["ctx_in_seq"]).to(dev), 5)
    close(out, g["ctx_out_windows"], atol=0, rtol=0)


@pytest.mark.parametrize("tag,arch,uf", [("vit", "vits_dino", 1), ("resnet", "resnet50", 2)])
def test_mhcrnn_head_golden(lpb, dev, golden, tag, arch, uf):
    """HeatmapMHCRNNHead.forward against the outputs of the reference's own module (heads/heatmap_mhcrnn.py), and the
    fused video form against the reference call form on materialised windows."""
    g = golden("mhcrnn")
    head = _load_mhcrnn(g, tag, arch, 64, uf, dev)
    feats = T(g[f"{tag}_in_features"]).to(dev)
    sf, mf = head(feats, torch.Size([3, 5, 3, 64, 96]), False)
    close(sf, g[f"{tag}_out_sf"], atol=1e-8)
    close(mf, g[f"{tag}_out_mf"], atol=1e-8)
    close(mf.sum((2, 3)), torch.ones(3, 5), atol=1e-5)
    # video form: T = 9 frames -> 5 valid outputs; equals the call form on get_context_from_sequence(...)[2:-2]
    torch.manual_seed(6)
    seq = torch.randn(9, 64, 4, 6, device=dev)
    sf_s, mf_s = head.forward_sequence(seq)
    win = lpb.context_gather(seq, 5)[2:-2]  # (5, 5, C, h, w)
    sf_w, mf_w = head(win.permute(0, 2, 3, 4, 1).contiguous(), torch.Size([9, 3, 64, 96]), False)
    close(sf_s, sf_w, atol=0, rtol=0)
    close(mf_s, mf_w, atol=1e-9, rtol=1e-6)


@pytest.mark.parametrize("tag,arch,uf", [("vit", "vits_dino", 1), ("resnet", "resnet50", 2)])
def test_mhcrnn_backward_vs_oracle_autograd(lpb, dev, golden, tag, arch, uf):
    g = golden("mhcrnn")
    head = _load_mhcrnn(g, tag, arch, 64, uf, dev)
    p = _mhcrnn_oracle_params(head)
    leaves = []
    for key, tup in p.items():
        p[key] = tuple(t.requires_grad_(True) for t in tup)
        leaves += list(p[key])
    torch.manual_seed(9)
    seq = torch.randn(8, 64, 4, 6)
    gout = torch.randn(4, 5, 16 if uf == 1 else 32, 24 if uf == 1 else 48)
    f_ref = seq.clone().requires_grad_(True)
    win = O.context_windows(f_ref, 5)[2:-2]  # (4, 5, C, h, w) -> frames first
    mf_ref = O.mhcrnn_multiframe(win.permute(1, 0, 2, 3, 4), p, uf)
    (mf_ref * gout).sum().backward()
    f = seq.to(dev).requires_grad_(True)
    _, mf = head.forward_sequence(f)
    close(mf, mf_ref, atol=1e-8)
    (mf * gout.to(dev)).sum().backward()
    close(f.grad, f_ref.grad, atol=1e-7, rtol=2e-3)
    m = head.head_mf
    mods = {"W_f": [m.W_f], "W_b": [m.W_b], "H_f": [m.H_f[0], m.H_f[1]], "H_b": [m.H_b[0], m.H_b[1]]}
    if uf == 2:
        mods["W_pre"] = [m.W_pre]
    for key, ms in mods.items():
        got = [t for mod in ms for t in (mod.weight.grad, mod.bias.grad)]
        for a, b in zip(got, p[key]):
            close(a, b.grad, atol=2e-6, rtol=2e-3)


def test_mhcrnn_bf16_real_shape_and_tracker(lpb, dev):
    """config 3: ViT-S features (384, 16, 16) of a 256x256 clip, bf16: the video form's shapes, one semi-supervised step and predict_step."""
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import SemiSupervisedHeatmapTrackerMHCRNN
    from lightning_pose_b200.losses.factory import LossFactory

    torch.manual_seed(21)
    k, t = 17, 12

    class Feats(torch.nn.Module):  # stands in for ViT-S: (n, 3, 256, 256) -> (n, 384, 16, 16) bf16
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 384, 16, stride=16)

        def forward(self, x):
            return self.conv(x).bfloat16()

    tr = SemiSupervisedHeatmapTrackerMHCRNN(
        k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
        loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": 5.0, "epsilon": 5.0, "prob_threshold": 0.05}}, None),
        backbone=Feats(), backbone_arch="vits_dino", num_fc_input_features=384).to(dev)
    frames = torch.randn(t, 3, 256, 256, device=dev)
    with torch.no_grad():
        feats = tr.backbone(frames)
        sf, mf = tr.head.forward_sequence(feats)
    assert sf.shape == mf.shape == (t - 4, k, 64, 64)  # the heatmaps against float64: test_context_train_gpu.py
    # one semi-supervised step runs end to end and reaches the backbone
    bbox = torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=dev).repeat(t, 1)
    loss = tr.evaluate_unlabeled({"frames": frames, "transforms": torch.tensor([-1.0], device=dev), "bbox": bbox, "is_multiview": False}, "train", 1.0)
    loss.backward()
    assert torch.isfinite(loss) and tr.backbone.conv.weight.grad is not None and torch.isfinite(tr.backbone.conv.weight.grad).all()
    kp, cf = tr.predict_step({"frames": frames, "bbox": bbox}, 0)
    assert kp.shape == (t - 4, 2 * k) and cf.shape == (t - 4, k)


def test_multiview_transformer_tracker_config4(lpb, dev):
    """config 4: 4 views x 384x384 -> per-view ViT token grids (384, 24, 24) -> the SAME head on views * batch maps ->
    heatmaps folded to (batch, 4 * 17, 96, 96) (reference heatmap_tracker_multiview.py:143-258); bf16 banded kernels
    against the fp32 oracle on identical features, then one supervised + multi-view step end to end."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    torch.manual_seed(17)
    k, v, b, d, img = 17, 4, 2, 384, 384

    class Patch(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Conv2d(3, d, 16, stride=16)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class Mix(torch.nn.Module):  # stands in for the attention blocks: mixes tokens ACROSS views
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(d, d)

        def forward(self, t):
            return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()

    tr = HeatmapTrackerMultiviewTransformer(k, v, Patch(), Mix(), d, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)).to(dev)
    for layer in list(tr.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    images = torch.randn(b, v, 3, img, img, device=dev)
    with torch.no_grad():
        feats = tr.forward_vit(images.reshape(-1, 3, img, img))
        hm = tr(images)
    assert feats.shape == (b * v, d, 24, 24) and feats.dtype == torch.bfloat16 and hm.shape == (b, v * k, 96, 96)
    dc = list(tr.head.upsampling_layers)[1]
    ref = O.head_forward(feats.float().cpu(), [dc.weight.detach().cpu().bfloat16().float()], [dc.bias.detach().cpu()]).reshape(b, v * k, 96, 96)
    rel = ((hm.cpu() - ref).abs() / (ref.abs() + 1e-7)).flatten()
    assert float(rel.max()) < 3e-2 and float((rel > 1e-2).float().mean()) < 1e-4
    # view mixing really happened: changing view 3 of example 0 changes view 0's heatmaps of example 0 only
    images2 = images.clone()
    images2[0, 3] += 1.0
    with torch.no_grad():
        hm2 = tr(images2)
    assert float((hm2[0, :k] - hm[0, :k]).abs().max()) > 0 and float((hm2[1] - hm[1]).abs().max()) == 0
    kp = torch.rand(b, v * k * 2, device=dev) * img
    targets = lpb.generate_heatmaps(kp.reshape(b, v * k, 2), img, img, (96, 96))
    bbox = torch.tensor([[0.0, 0.0, 400.0, 420.0] * v], device=dev).repeat(b, 1)
    loss = tr.evaluate_labeled({"images": images, "keypoints": kp.clone(), "heatmaps": targets, "bbox": bbox, "num_views": torch.full((b,), v, device=dev)}, "train", 1.0)
    loss.backward()
    assert torch.isfinite(loss) and tr.view_embeddings.grad is not None and float(tr.view_embeddings.grad.abs().max()) > 0
    assert tr.patch_embed.proj.weight.grad is not None and torch.isfinite(tr.patch_embed.proj.weight.grad).all()


def test_kernel_variants_agree(lpb, dev):
    """LPB_TUNE_SOFTMAX_SPLIT (key 7) selects a different implementation of the SAME stage: the plane softmax as two
    launches parallel over (frame, band) (2: always) or one per-frame two-pass kernel (0: never split); results must agree
    to rounding (same math in a different order), and the default (which splits below one wave: 6 frames) with both."""
    from lightning_pose_b200._lib import lib

    head = make_head(2048, (17, 17), seed=41, gain=4.0)
    feats = features(6, 2048, 12, 12, 42, torch.bfloat16)
    gk = torch.randn(6, 34, device=dev, generator=gen(43))

    def run():
        head.zero_grad()
        f = feats.clone().requires_grad_(True)
        hm, kp, cf = head.forward_with_keypoints(f)
        ((kp * gk).sum() * 1e-3 + (hm * hm).sum()).backward()
        return hm.detach().clone(), kp.detach().clone(), cf.detach().clone(), f.grad.float().clone(), list(head.upsampling_layers)[1].weight.grad.clone()

    cur = run()  # the default
    with softmax_split(lib, 2):
        new = run()
    with softmax_split(lib, 0):
        old = run()
    close(new[0], old[0], atol=1e-9, rtol=2e-5)   # heatmaps
    close(new[1], old[1], atol=2e-3, rtol=1e-5)   # keypoints (T = 1000 amplifies the last ulp of a heatmap)
    close(new[2], old[2], atol=1e-5, rtol=1e-4)   # confidences
    for a, b in zip(new[3:] + cur[3:], old[3:] + old[3:]):
        assert float((a - b).abs().max()) <= 2e-3 * float(b.abs().max()) + 1e-12
    close(cur[0], old[0], atol=1e-9, rtol=2e-5)
    close(cur[1], old[1], atol=2e-3, rtol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("decoupled,wd", [(False, 0.0), (False, 0.01), (True, 0.05)])
def test_fused_adam_matches_torch(lpb, dev, decoupled, wd):
    """lpb_adam_step vs torch.optim.Adam / AdamW (the optimizers of configure_optimizers, models/base.py:458-477):
    same trajectories over several steps, shared step counter, state keys of torch's own Adam."""
    from lightning_pose_b200.optim import FusedAdam

    g = torch.Generator().manual_seed(7)
    shapes = [(512, 17, 3, 3), (17,), (17, 17, 3, 3), (17,)]
    ours = [torch.nn.Parameter(torch.randn(s, generator=g).to(dev)) for s in shapes]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in ours]
    opt = FusedAdam(ours, lr=3e-3, weight_decay=wd, decoupled_weight_decay=decoupled)
    topt = (torch.optim.AdamW if decoupled else torch.optim.Adam)(ref, lr=3e-3, weight_decay=wd)
    for it in range(6):
        for p, q in zip(ours, ref):
            gr = torch.randn(p.shape, generator=g).to(dev) * (1.0 + it)
            p.grad, q.grad = gr.clone(), gr.clone()
        opt.step()
        topt.step()
    for p, q in zip(ours, ref):
        close(p, q, atol=1e-6, rtol=2e-5)
    assert float(opt.state[ours[0]]["step"]) == 6.0 and opt.state[ours[1]]["step"] is opt.state[ours[0]]["step"]
    close(opt.state[ours[2]]["exp_avg_sq"], topt.state[ref[2]]["exp_avg_sq"], atol=1e-9, rtol=1e-5)


@pytest.mark.gpu
def test_fused_adam_graph_replay(lpb, dev):
    """The step counter lives on the device: a captured step replays as consecutive optimizer steps."""
    from lightning_pose_b200.optim import FusedAdam

    g = torch.Generator().manual_seed(3)
    p = torch.nn.Parameter(torch.randn(1000, generator=g).to(dev))
    q = torch.nn.Parameter(p.detach().clone())
    gr = torch.randn(1000, generator=g).to(dev)
    p.grad, q.grad = gr.clone(), gr.clone()
    opt, topt = FusedAdam([p], lr=1e-2), torch.optim.Adam([q], lr=1e-2)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        opt.step()  # state allocation outside the capture
    torch.cuda.current_stream(dev).wait_stream(side)
    topt.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    topt.step()  # capture only records: ours = 1 eager + 3 replays, torch = 4 eager steps
    for _ in range(3):
        graph.replay()
    for _ in range(2):
        topt.step()
    torch.cuda.synchronize(dev)
    assert float(opt.state[p]["step"]) == 4.0
    close(p, q, atol=1e-6, rtol=2e-5)
