"""GPU: calibrated multi-view 3-D losses (csrc/cameras.cu) against tests/golden/cameras.npz (the reference's own
data/cameras.py and frame_to_model_batch, float64 autograd), run-to-run reproducibility, the pairwise-projection loss
kernel against the torch formula, and the calibrated config-4 tracker step (eager, backward, CUDA graph)."""
import math

import numpy as np
import pytest
import torch

import cameras_oracle as O

pytestmark = pytest.mark.gpu

RIGS = ("fly", "ring2", "ring3", "ring4", "ring6")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


def rig(g, name, dev):
    t = lambda k: torch.from_numpy(g[f"{name}_in_{k}"]).to(dev)
    return t("points"), t("K"), t("E"), t("dist"), t("bbox"), tuple(int(x) for x in g[f"{name}_in_model_hw"]), t("points3d")


def match(got, ref, rtol=1e-4):
    """NaN exactly where the reference has NaN; elsewhere |got - ref| <= rtol |ref| + 1e-6 max|ref|."""
    got = got.detach().cpu().double().numpy()
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=1e-6 * np.abs(ref[fin]).max())


def match_grad(got, ref):
    """float64 autograd gradients: NaN-input entries (NaN in the reference) get a zero gradient here."""
    got = got.detach().cpu().double().numpy()
    ref = np.asarray(ref, dtype=np.float64)
    nan = np.isnan(ref)
    assert (got[nan] == 0).all() and np.isfinite(got).all()
    np.testing.assert_allclose(got[~nan], ref[~nan], rtol=1e-4, atol=1e-6 * np.abs(ref[~nan]).max())


@pytest.mark.parametrize("name", RIGS)
def test_forward_matches_golden(lpb, dev, golden, name):
    from lightning_pose_b200.data.bboxes import frame_to_model_batch
    from lightning_pose_b200.data.cameras import project_3d_to_2d, project_camera_pairs_to_3d

    g = golden("cameras")
    pts, K, E, D, bbox, hw, p3n = rig(g, name, dev)
    p3d = project_camera_pairs_to_3d(pts, K, E, D)
    match(p3d, g[f"{name}_out_p3d"])
    match(project_3d_to_2d(p3n, K, E, D), g[f"{name}_out_p2d"])
    bd = {"images": torch.zeros(pts.shape[0], pts.shape[1], 3, *hw, device=dev), "bbox": bbox}
    match(frame_to_model_batch(bd, pts), g[f"{name}_out_frame_to_model"])
    match(lpb.project_points(p3d, K, E, D, mean_over_pairs=True, bbox=bbox, model_size=hw), g[f"{name}_out_reproj"])


@pytest.mark.parametrize("name", RIGS)
def test_gradients_match_golden(lpb, dev, golden, name):
    from lightning_pose_b200.data.cameras import project_3d_to_2d, project_camera_pairs_to_3d

    g = golden("cameras")
    pts, K, E, D, bbox, hw, p3n = rig(g, name, dev)
    g3, g2 = (torch.from_numpy(g[f"{name}_in_{k}"]).to(dev) for k in ("g3", "g2"))
    x = pts.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(project_camera_pairs_to_3d(x, K, E, D), x, g3)
    match_grad(gx, g[f"{name}_out_grad_points_tri"])
    y = p3n.clone().requires_grad_(True)
    (gy,) = torch.autograd.grad(project_3d_to_2d(y, K, E, D), y, g2)
    match_grad(gy, g[f"{name}_out_grad_points3d"])
    x = pts.clone().requires_grad_(True)
    rep = lpb.project_points(project_camera_pairs_to_3d(x, K, E, D), K, E, D, mean_over_pairs=True, bbox=bbox, model_size=hw)
    (gx,) = torch.autograd.grad(rep, x, g2)
    match_grad(gx, g[f"{name}_out_grad_points_reproj"])


def _ring(v, b, p, seed, img=384, spread=0.3, arc=2 * math.pi):
    gen = torch.Generator().manual_seed(seed)
    K = torch.zeros(b, v, 3, 3)
    E = torch.zeros(b, v, 3, 4)
    for j in range(v):
        K[:, j, 0, 0] = K[:, j, 1, 1] = 800.0 + torch.randn(b, generator=gen) * 50
        K[:, j, 0, 2], K[:, j, 1, 2], K[:, j, 2, 2] = img / 2, img / 2, 1.0
        a = j / v * arc
        E[:, j] = torch.tensor([[math.cos(a), 0.0, -math.sin(a), 0.0], [0.0, 1.0, 0.0, 0.0], [math.sin(a), 0.0, math.cos(a), 2.0]])
    D = torch.randn(b, v, p, generator=gen) * 0.05
    X = torch.randn(b, 9, 3, generator=gen) * spread
    pts = O.project_3d_to_2d(X.double(), K.double(), E.double(), D.double()).float() + torch.randn(b, v, 9, 2, generator=gen) * 0.5
    pts[0, v - 1, 4] = float("nan")
    return pts, K, E, D


def test_eight_views_match_oracle(lpb, dev):
    """V = 8 (28 pairs), P = 12: forward and the pair-mean reprojection against the float64 oracle."""
    from lightning_pose_b200.data.cameras import project_camera_pairs_to_3d

    pts, K, E, D = _ring(8, 3, 12, 91)
    p3d = project_camera_pairs_to_3d(*(t.to(dev) for t in (pts, K, E, D)))
    ref = O.project_camera_pairs_to_3d(*(t.double() for t in (pts, K, E, D)))
    assert p3d.shape == (3, 28, 9, 3)
    match(p3d, ref.numpy())
    rep = lpb.project_points(p3d, *(t.to(dev) for t in (K, E, D)), mean_over_pairs=True)
    match(rep, O.project_3d_to_2d(ref.mean(1), *(t.double() for t in (K, E, D))).numpy())


@pytest.mark.parametrize("name", ["ring4", "ring6"])
def test_forward_backward_bit_identical(lpb, dev, golden, name):
    from lightning_pose_b200.data.cameras import project_camera_pairs_to_3d

    g = golden("cameras")
    pts, K, E, D, bbox, hw, _ = rig(g, name, dev)
    g2 = torch.from_numpy(g[f"{name}_in_g2"]).to(dev)
    outs = []
    for _ in range(2):
        x = pts.clone().requires_grad_(True)
        p3d = project_camera_pairs_to_3d(x, K, E, D)
        rep = lpb.project_points(p3d, K, E, D, mean_over_pairs=True, bbox=bbox, model_size=hw)
        loss = lpb.pairwise_projections_loss(torch.randn(p3d.shape[0], p3d.shape[2], 3, generator=torch.Generator().manual_seed(3)).to(dev), p3d)
        (gx,) = torch.autograd.grad((rep * g2).nansum() + loss, x)
        outs.append((p3d.detach(), rep.detach(), loss.detach(), gx))
    for a, b in zip(*outs):
        assert torch.equal(a.nan_to_num(123.0), b.nan_to_num(123.0))


def test_pairwise_projection_loss_matches_torch_formula(lpb, dev):
    from lightning_pose_b200.losses.losses import PairwiseProjectionsLoss

    gen = torch.Generator().manual_seed(8)
    targ = torch.randn(4, 17, 3, generator=gen)
    pred = targ[:, None] + torch.randn(4, 6, 17, 3, generator=gen) * 0.1
    targ[0, 2] = float("nan")
    pred[1, 3, 5, 1] = float("nan")
    pred[2, :, 7] = float("nan")
    targ, pred = targ.to(dev), pred.to(dev)
    loss_fn = PairwiseProjectionsLoss(log_weight=0.5)
    p1 = pred.clone().requires_grad_(True)
    ours, logs = loss_fn(keypoints_targ_3d=targ, keypoints_pred_3d=p1, stage="train")
    (g1,) = torch.autograd.grad(ours, p1)
    p2 = pred.clone().requires_grad_(True)
    ref = loss_fn.reduce_loss(loss_fn.remove_nans(loss_fn.compute_loss(targets=targ, predictions=p2)), "mean")
    (g2,) = torch.autograd.grad(ref, p2)
    torch.testing.assert_close(ours, ref, rtol=1e-5, atol=0)
    # dropped entries: the torch formula's norm backward at the zeroed vectors is 0/0 = NaN there; the kernel gives 0
    dropped = torch.isnan(g2)
    assert torch.isfinite(g1).all() and (g1[dropped] == 0).all()
    assert (g1[0, :, 2] == 0).all() and (g1[2, :, 7] == 0).all() and (g1[1, 3, 5] == 0).all()  # every dropped entry
    torch.testing.assert_close(g1[~dropped], g2[~dropped], rtol=1e-5, atol=1e-9)
    assert logs[0]["name"] == "train_supervised_pairwise_projections_loss"
    # nothing kept: 0 with a zero gradient
    p3 = torch.full_like(pred, float("nan")).requires_grad_(True)
    v, _ = loss_fn(keypoints_targ_3d=targ, keypoints_pred_3d=p3)
    (g3,) = torch.autograd.grad(v, p3)
    assert float(v) == 0.0 and float(g3.abs().max()) == 0.0


# ---- the calibrated config-4 tracker step --------------------------------------------------------------------------
K_, V_, B_, D_, IMG = 17, 4, 2, 384, 384


def _tracker(dev, losses):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    torch.manual_seed(17)

    class Patch(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Conv2d(3, D_, 16, stride=16)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class Mix(torch.nn.Module):  # stands in for the attention blocks: mixes tokens across views
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(D_, D_)

        def forward(self, t):
            return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()

    fac = LossFactory(losses, None)
    tr = HeatmapTrackerMultiviewTransformer(K_, V_, Patch(), Mix(), D_, loss_factory=fac).to(dev)
    for layer in list(tr.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return tr, fac


LOSSES_3D = {
    "heatmap_mse": {"log_weight": 0.0},
    "supervised_pairwise_projections": {"log_weight": 0.0},
    "supervised_reprojection_heatmap_mse": {"log_weight": 0.0, "original_image_height": IMG, "original_image_width": IMG,
                                            "downsampled_image_height": IMG // 4, "downsampled_image_width": IMG // 4},
}


def _calibrated_batch(lpb, dev):
    """Cameras on a half circle (no two facing each other) and bboxes of 4 x 4 frame pixels around each principal point:
    whatever the untrained head decodes, the rays stay near the optical axes and triangulate near the origin, in front of
    every camera, as a trained model's would."""
    pts, K, E, D = _ring(V_, B_, 5, 33, arc=math.pi)
    gen = torch.Generator().manual_seed(34)
    kp3 = torch.randn(B_, K_, 3, generator=gen) * 0.3
    kp3[0, 3] = float("nan")
    kp3[1, 11] = float("nan")
    kp = torch.rand(B_, V_ * K_ * 2, generator=gen) * IMG
    return {
        "images": torch.randn(B_, V_, 3, IMG, IMG, generator=gen).to(dev),
        "keypoints": kp.to(dev),
        "heatmaps": lpb.generate_heatmaps(kp.to(dev).reshape(B_, V_ * K_, 2), IMG, IMG, (IMG // 4, IMG // 4)),
        "bbox": torch.tensor([[IMG / 2 - 2, IMG / 2 - 2, 4.0, 4.0] * V_], device=dev).repeat(B_, 1),
        "is_multiview": True,
        "keypoints_3d": kp3.to(dev),
        "intrinsic_matrix": K.to(dev),
        "extrinsic_matrix": E.to(dev),
        "distortions": D.to(dev),
    }


def test_calibrated_config4_loss_inputs_equal_oracle(lpb, dev):
    tr, _ = _tracker(dev, LOSSES_3D)
    bd = _calibrated_batch(lpb, dev)
    with torch.no_grad():
        data = tr.get_loss_inputs_labeled(bd)
    for key in ("keypoints_targ_3d", "keypoints_pred_3d", "keypoints_pred_2d_reprojected"):
        assert data[key] is not None, key
    assert data["keypoints_pred_3d"].shape == (B_, 6, K_, 3) and data["keypoints_pred_2d_reprojected"].shape == (B_, V_ * K_, 2)
    assert data["keypoints_targ_3d"] is bd["keypoints_3d"]
    cams = [bd[k].cpu().double() for k in ("intrinsic_matrix", "extrinsic_matrix", "distortions")]
    kp = data["keypoints_pred"].cpu().double().reshape(B_, V_, K_, 2)  # the same decoded keypoints, frame pixels
    p3d = O.project_camera_pairs_to_3d(kp, *cams)
    match(data["keypoints_pred_3d"], p3d.numpy())
    rep = O.frame_to_model_batch(O.project_3d_to_2d(p3d.mean(1), *cams), bd["bbox"].cpu().double(), IMG, IMG)
    match(data["keypoints_pred_2d_reprojected"], rep.reshape(B_, V_ * K_, 2).numpy())


def test_calibrated_config4_backpropagates_into_head(lpb, dev):
    tr, _ = _tracker(dev, LOSSES_3D)
    bd = _calibrated_batch(lpb, dev)
    loss = tr.evaluate_labeled(bd, "train", 1.0)
    loss.backward()
    assert torch.isfinite(loss)
    for p in list(tr.head.parameters()) + [tr.view_embeddings]:
        assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().max()) > 0
    names = {d["name"] for d in tr.last_logs}
    assert {"train_supervised_pairwise_projections_loss", "train_supervised_reprojection_heatmap_mse_loss"} <= names
    # the two 3-D losses on their own reach the head
    tr3, fac3 = _tracker(dev, {k: v for k, v in LOSSES_3D.items() if k != "heatmap_mse"})
    data = tr3.get_loss_inputs_labeled(_calibrated_batch(lpb, dev))
    l3, _ = fac3(stage="train", **data)
    grads = torch.autograd.grad(l3, list(tr3.head.parameters()) + [tr3.view_embeddings])
    assert all(torch.isfinite(g_).all() for g_ in grads) and float(grads[0].abs().max()) > 0


def test_calibrated_config4_step_replays_in_cuda_graph(lpb, dev):
    """The labeled step with the two 3-D losses, captured once and replayed, equals the eager step: nothing on the
    path synchronises with the host."""
    tr, fac = _tracker(dev, LOSSES_3D)
    bd = _calibrated_batch(lpb, dev)
    kp0 = bd["keypoints"].clone()
    params = list(tr.head.parameters()) + [tr.view_embeddings]
    weights = {n: inst.weight.to(dev) for n, inst in fac.loss_instance_dict.items()}

    def step():
        bd["keypoints"].copy_(kp0)  # model_to_frame_batch rewrites the targets in place
        data = tr.get_loss_inputs_labeled(bd)
        total = sum(weights[n] * inst(stage="train", **data)[0] for n, inst in fac.loss_instance_dict.items())
        grads = torch.autograd.grad(total, params)
        return [total.detach(), data["keypoints_pred_3d"].detach(), data["keypoints_pred_2d_reprojected"].detach(), *grads]

    eager = [t.clone() for t in step()]
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
    graph.replay()
    torch.cuda.synchronize(dev)
    for a, b in zip(eager[:3], out[:3]):
        assert torch.equal(a.nan_to_num(123.0), b.nan_to_num(123.0))
    # gradients: the one-deconv head's bias gradient is summed with float atomics (DESIGN.md), so to rounding
    for a, b in zip(eager[3:], out[3:]):
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max())
