"""GPU: ``SemiSupervisedHeatmapTrackerMultiviewTransformer`` (reference ``models/heatmap_tracker_multiview.py:370-484``).

Two shapes: config 4 (4 views, 17 keypoints, 384 x 384 model frames) and a small odd one (3 views, 5 keypoints,
192 x 256 model frames from views of different non-square sizes), both on the stand-in transformer of
``test_gpu_parity.py::test_multiview_transformer_tracker_config4`` (patch convolution + one token-mixing layer, bf16
tokens).  The unlabeled batches are ``dlc``-augmented by ``frames_to_unlabeled_batch`` with a seeded generator.

* the unlabeled keypoints against a float64 staging of the reference's order (decode of the kernel's heatmaps, per-view
  ``undo_affine_transform_batch``, ``model_to_frame_batch``), for every transform shape the tracker accepts and for an
  unaugmented batch;
* the unsupervised losses (fused temporal + both PCA losses, temporal heatmap MSE) against the oracle on the folded
  tensors, and the step's total;
* the gradients of one semi-supervised step at the head's parameters, the view embeddings and the encoder's output
  against float64, by the rules of ``head_support.py``;
* the whole step (augmented ingest, masking, both branches, backward) captured into one CUDA graph: three replays equal
  three eager steps on the same draws, and the anneal weight changed between replays changes the unsupervised part of
  the total only."""
import pytest
import torch

import scale_oracle as S
from head_support import F64, WORST, check_grads, head_params, ref_grads, report_headroom
from oracle import lp_oracle as O

pytestmark = pytest.mark.gpu

D = 384
# name: (views, keypoints, model frame (H, W), source view sizes, unlabeled frames T, labeled examples B)
CASES = {
    "config4": (4, 17, (384, 384), [(420, 400), (390, 410), (400, 400), (384, 450)], 6, 2),
    "odd": (3, 5, (192, 256), [(200, 300), (240, 180), (150, 260)], 5, 2),
}
LOG_W = {"temporal": 0.5, "pca_multiview": 1.0, "pca_singleview": 1.5, "temporal_heatmap_mse": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


class Patch(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = torch.nn.Conv2d(3, D, 16, stride=16)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class Mix(torch.nn.Module):
    """Stands in for the attention blocks: mixes tokens across views; keeps each output, with its gradient."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(D, D)
        self.outs = []

    def forward(self, t):
        y = (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()
        if y.requires_grad:
            y.retain_grad()
        self.outs.append(y)
        return y


def pca_fit_data(v, k, n=64, seed=3):
    """(n, 2 v k) frame-pixel keypoints of n random 3-D poses seen by v affine cameras: rank-3 views for the PCA fit."""
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, k, 3, generator=g, dtype=F64) * 40
    cams = torch.randn(v, 2, 3, generator=g, dtype=F64)
    offs = 150 + torch.rand(1, v, 1, 2, generator=g, dtype=F64) * 50
    return (torch.einsum("vij,nkj->nvki", cams, pts) + offs).reshape(n, -1).float()


def unsup_params(v, k):
    sel = list(range(min(k, 6)))
    return {
        "temporal": {"log_weight": LOG_W["temporal"], "epsilon": 1.0, "prob_threshold": 0.0},
        "pca_multiview": {"loss_name": "pca_multiview", "log_weight": LOG_W["pca_multiview"], "epsilon": 2.0, "components_to_keep": 3,
                          "mirrored_column_matches": [[i * k + j for j in sel] for i in range(v)]},
        "pca_singleview": {"loss_name": "pca_singleview", "log_weight": LOG_W["pca_singleview"], "epsilon": 1.0, "components_to_keep": 3,
                           "columns_for_singleview_pca": [j + k for j in sel]},
        "temporal_heatmap_mse": {"loss_name": "temporal_heatmap_mse", "log_weight": LOG_W["temporal_heatmap_mse"], "epsilon": 0.0, "prob_threshold": 0.0},
    }


def tracker(dev, case, masker=None):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import SemiSupervisedHeatmapTrackerMultiviewTransformer

    v, k = CASES[case][:2]
    torch.manual_seed(17)
    tr = SemiSupervisedHeatmapTrackerMultiviewTransformer(
        k, v, Patch(), Mix(), D, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
        loss_factory_unsupervised=LossFactory(unsup_params(v, k), pca_fit_data(v, k)), patch_masker=masker).to(dev)
    for layer in list(tr.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return tr


def source_views(dev, case, seed=5):
    g = torch.Generator(device=dev).manual_seed(seed)
    t = CASES[case][4]
    return [torch.randint(0, 256, (t, h, w, 3), dtype=torch.uint8, device=dev, generator=g) for h, w in CASES[case][3]]


def unlabeled_batch(dev, case, seed=9, imgaug="dlc"):
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    return frames_to_unlabeled_batch(source_views(dev, case), CASES[case][2], imgaug=imgaug,
                                     generator=torch.Generator(device=dev).manual_seed(seed))


def labeled_batch(dev, case, seed=11):
    from lightning_pose_b200 import ops

    v, k, (h, w), _, _, b = CASES[case]
    g = torch.Generator(device=dev).manual_seed(seed)
    kp = torch.rand(b, v * k, 2, device=dev, generator=g) * torch.tensor([w, h], device=dev, dtype=torch.float32)
    return {"images": torch.randn(b, v, 3, h, w, device=dev, generator=g), "keypoints": kp.reshape(b, -1),
            "heatmaps": ops.generate_heatmaps(kp, h, w, (h // 4, w // 4)),
            "bbox": torch.tensor([[3.0, 5.0, h * 1.1, w * 0.9] * v], device=dev).repeat(b, 1), "is_multiview": True}


def remap_ref(kp_aug, transforms, bbox, h, w, v):
    """float64, differentiable: per-view undo of the augmentation (A^-1 (p - t), data/utils.py:142-234), then model ->
    frame pixels with the view's bbox [x, y, h, w] (data/bboxes.py:222-288)."""
    n = kp_aug.shape[0]
    p = kp_aug.to(F64).reshape(n, v, -1, 2)
    if transforms is not None:
        m = transforms.to(F64).reshape(v, 2, 3)
        a_inv = torch.linalg.inv(m[:, :, :2])
        p = torch.einsum("vij,nvkj->nvki", a_inv, p - m[None, :, None, :, 2])
    bb = bbox.to(F64).reshape(n, v, 1, 4)
    return torch.stack([p[..., 0] / w * bb[..., 3] + bb[..., 0], p[..., 1] / h * bb[..., 2] + bb[..., 1]], -1).reshape(n, -1)


def unsup_ref(tr, kp_frame, hm, conf):
    """Each unsupervised loss of the tracker's factory in float64 (the oracle) on the given folded tensors."""
    insts = tr.loss_factory_unsup.loss_instance_dict
    mv, sv = insts["pca_multiview"], insts["pca_singleview"]
    return {
        "temporal": S.temporal_loss_ref(kp_frame, conf, 1.0, 0.0),
        "pca_multiview": S.pca_multiview_ref(kp_frame, mv.pca.mirrored_column_matches, mv.pca.parameters["mean"],
                                             mv.pca.parameters["kept_eigenvectors"], float(mv.epsilon)),
        "pca_singleview": S.pca_singleview_ref(kp_frame, sv.pca.columns_for_singleview_pca, None, sv.pca.parameters["mean"],
                                               sv.pca.parameters["kept_eigenvectors"], float(sv.epsilon)),
        "temporal_heatmap_mse": O.temporal_heatmap_loss(hm.to(F64), conf.to(F64), "mse", 0.0, 0.0),
    }


# ---- 1. keypoints of the unlabeled branch -----------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["v,1,2,3", "1,v,2,3", "v,2,3", "unaugmented"])
@pytest.mark.parametrize("case", list(CASES))
def test_unlabeled_keypoints_equal_float64_staging(dev, case, shape):
    v, k, (h, w) = CASES[case][:3]
    tr = tracker(dev, case)
    bd = unlabeled_batch(dev, case, imgaug=None if shape == "unaugmented" else "dlc")
    tf = bd["transforms"]
    if shape == "unaugmented":
        assert tf.shape == (v, 1)
    else:
        assert tf.shape == (v, 1, 2, 3)
        bd["transforms"] = {"v,1,2,3": tf, "1,v,2,3": tf.reshape(1, v, 2, 3), "v,2,3": tf.reshape(v, 2, 3)}[shape]
    with torch.no_grad():
        d = tr.get_loss_inputs_unlabeled(bd)
    t = bd["frames"].shape[0]
    hm = d["heatmaps_pred"]
    assert hm.shape == (t, v * k, h // 4, w // 4) and d["keypoints_pred"].shape == d["keypoints_pred_augmented"].shape == (t, 2 * v * k)
    assert d["confidences"].shape == (t, v * k)
    preds, _, _, _ = S.decode_ref(hm, 2, 1000.0)
    aug = d["keypoints_pred_augmented"].to(F64)
    assert bool(((aug - preds).abs() <= 2e-3 + 1e-4 * preds.abs()).all()), float((aug - preds).abs().max())
    ref = remap_ref(preds, None if shape == "unaugmented" else tf, bd["bbox"], h, w, v)
    err = (d["keypoints_pred"].to(F64) - ref).abs()
    # the decode's bar (above) through the undo (row sums of A^-1 below 1.45 at +-10 degrees and scale >= 0.8) and the
    # bbox scale (below 1.25 here): within 4 times it, plus fp32 rounding
    bar = 4 * (2e-3 + 1e-4 * float(preds.abs().max()))
    assert bool((err <= bar + 1e-5 * ref.abs()).all()), float(err.max())
    # the same remap from the kernel's own decoded keypoints: to fp32 rounding
    mine = remap_ref(aug, None if shape == "unaugmented" else tf, bd["bbox"], h, w, v)
    assert bool(((d["keypoints_pred"].to(F64) - mine).abs() <= 1e-4 + 1e-5 * mine.abs()).all())


# ---- 2. the unsupervised losses ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_unsupervised_losses_equal_oracle(dev, case):
    tr = tracker(dev, case)
    bd = unlabeled_batch(dev, case)
    tr.total_unsupervised_importance.fill_(0.7)
    with torch.no_grad():
        d = tr.get_loss_inputs_unlabeled(bd)
        total, logs = tr.loss_factory_unsup.total_on_device("train", tr.total_unsupervised_importance, **d)
        eager, _ = tr.loss_factory_unsup(stage="train", anneal_weight=0.7, **d)
    ref = unsup_ref(tr, d["keypoints_pred"], d["heatmaps_pred"], d["confidences"])
    got = {e["name"]: e["value"] for e in logs}
    for name, r in ref.items():
        assert float(r) > 0, name  # an untrained model: every loss is active
        torch.testing.assert_close(got[f"train_{name}_loss"].to(F64), r.to(F64), rtol=1e-4, atol=1e-6, msg=name)
    want = sum(0.7 * O.loss_weight(LOG_W[n]) * r.to(F64) for n, r in ref.items())
    torch.testing.assert_close(total.to(F64), want, rtol=1e-4, atol=0)
    torch.testing.assert_close(total, eager.to(total.device), rtol=1e-6, atol=0)  # __call__ sums the same values


# ---- 3. gradients of one semi-supervised step ------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_training_step_gradients_equal_float64(dev, case):
    """The float64 loss gradient at the kernels' heatmaps (labeled: heatmap MSE; unlabeled: the keypoint losses through
    the remap and the soft-argmax, plus the temporal heatmap loss), then back through the head in float64 on the
    encoder's bf16 output, and from there through the stand-in encoder to the view embeddings."""
    v, k, (h, w) = CASES[case][:3]
    tr = tracker(dev, case)
    anneal = 0.6
    tr.total_unsupervised_importance.fill_(anneal)
    calls = []
    fwk = tr.forward_with_keypoints

    def recorded(images):
        out = fwk(images)
        calls.append([x.detach() for x in out])
        return out

    tr.forward_with_keypoints = recorded
    labeled, unlabeled = labeled_batch(dev, case), unlabeled_batch(dev, case)
    targets = labeled["heatmaps"]
    tr.zero_grad(set_to_none=True)
    tr.training_step({"labeled": labeled, "unlabeled": unlabeled}, 0)["loss"].backward()
    case_name = f"semi-supervised step, {case}"
    (hm_l, _, _), (hm_u, _, conf_u) = calls

    # the losses' gradient at the kernels' heatmaps, float64
    _, g_l = S.heatmap_loss_ref(targets, hm_l, "mse", with_grad=True)
    g_l = O.loss_weight(0.0) * g_l  # heatmap MSE is not annealed
    preds, _, _, _ = S.decode_ref(hm_u, 2, 1000.0)
    kp = preds.detach().requires_grad_(True)
    hm64 = hm_u.to(F64).requires_grad_(True)
    ref = unsup_ref(tr, remap_ref(kp, unlabeled["transforms"], unlabeled["bbox"], h, w, v), hm64, conf_u)
    loss_u = anneal * sum(O.loss_weight(LOG_W[n]) * r for n, r in ref.items())
    g_kp, g_hm_direct = torch.autograd.grad(loss_u, [kp, hm64])
    g_u = S.decode_grad_ref(hm_u, 2, 1000.0, g_kp) + g_hm_direct

    # back through the head, on the encoder's output rows (view-major within an example, as forward_vit orders them)
    ws, bs = head_params(tr.head)
    hh, ww = h // 16, w // 16
    as_map = lambda y: y.reshape(-1, hh, ww, D).permute(0, 3, 1, 2)  # noqa: E731  (B, V*N, D) tokens -> (B*V, D, h, w)
    out_l, out_u = tr.encoder.outs
    refs = [ref_grads(as_map(o.detach()), ws, bs, g.reshape(-1, k, h // 4, w // 4), True, hm.reshape(-1, k, h // 4, w // 4))
            for o, g, hm in ((out_l, g_l, hm_l), (out_u, g_u, hm_u))]
    dc = list(tr.head.upsampling_layers)[1]
    got = {"dw1": dc.weight.grad, "db1": dc.bias.grad}
    check_grads(got, {n: refs[0][0][n] + refs[1][0][n] for n in got}, {"db1": refs[0][1]["db1"] + refs[1][1]["db1"]},
                f"{case_name}: head", rel=2e-2, global_scale=("dw1",))
    for o, (r, _), name in ((out_l, refs[0], "labeled"), (out_u, refs[1], "unlabeled")):
        assert o.grad is not None and float(o.grad.abs().max()) > 0, f"{case_name}: no gradient at the encoder's output ({name})"
        check_grads({"dfeat": as_map(o.grad)}, {"dfeat": r["dfeat"]}, {}, f"{case_name}: encoder output, {name} batch", rel=2e-2)

    # the view embeddings: the encoder's output gradient (held to float64 above) back through the stand-in (linear +
    # token mean) in float64, summed per view over examples and tokens; fp32 sums on the way
    lin_w = tr.encoder.lin.weight.detach().to(F64)
    d_view = torch.zeros(v, D, dtype=F64, device=dev)
    for o in (out_l, out_u):
        g = o.grad.to(F64)  # (example, view * N, D)
        d_tok = g @ lin_w + g.sum(1, keepdim=True) / g.shape[1]
        d_view += d_tok.reshape(g.shape[0], v, -1, D).sum((0, 2))
    err = (tr.view_embeddings.grad.to(F64) - d_view).abs().amax(1)
    assert bool((err <= 1e-3 * d_view.abs().amax(1)).all()), (err / d_view.abs().amax(1)).tolist()


# ---- 4. the whole step in one CUDA graph ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_semisupervised_step_replays_in_cuda_graph(dev, case):
    """Augmented ingest from a seeded generator, masking (steps 0, 1, 2 of a curriculum starting at step 1), both
    branches and the gradients of the head and view embeddings, captured once: three replays equal three eager steps
    on the same draws; then a new anneal weight between replays changes the unsupervised part of the total only."""
    from lightning_pose_b200.callbacks import PatchMasker
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    masker = PatchMasker({"init_step": 1, "final_step": 3, "init_ratio": 0.2, "final_ratio": 0.6}, patch_seed=11)
    tr = tracker(dev, case, masker=masker)
    size = CASES[case][2]
    views = source_views(dev, case)
    labeled = labeled_batch(dev, case)
    images0, kp0 = labeled["images"], labeled["keypoints"].clone()
    params = list(tr.head.parameters()) + [tr.view_embeddings]
    gen = torch.Generator(device=dev)

    def weighted(logs):
        return sum(e["value"] for e in logs if e["name"].endswith("_loss_weighted"))

    def step():
        labeled["images"] = images0  # training_step replaces the batch's images with the masked ones
        labeled["keypoints"].copy_(kp0)  # model_to_frame_batch rewrites the targets in place
        unlabeled = frames_to_unlabeled_batch(views, size, imgaug="dlc", generator=gen)
        loss = tr.training_step({"labeled": labeled, "unlabeled": unlabeled}, 0)["loss"]
        grads = torch.autograd.grad(loss, params)
        tr.encoder.outs.clear()
        # total, labeled part (heatmap MSE: not annealed), unsupervised part before the anneal weight
        return [loss.detach(), weighted(tr.last_logs), weighted(tr.last_logs_unsup), tr.current_patch_mask,
                unlabeled["transforms"], *grads]

    gen.manual_seed(21)
    eager = [[x.clone() for x in step()] for _ in range(3)]
    assert tr.global_step.item() == 3
    masked = [int((e[3] == 0).sum(-1).unique().item()) for e in eager]
    assert masked == [masker.patches_to_mask(s, eager[0][3].shape[-1]) for s in range(3)] and 0 == masked[0] < masked[1] < masked[2]
    assert not torch.equal(eager[0][4], eager[1][4]) and not torch.equal(eager[1][4], eager[2][4])  # fresh draws
    for e in eager:
        assert torch.isfinite(e[0]) and all(torch.isfinite(g_).all() and float(g_.abs().max()) > 0 for g_ in e[5:])
        torch.testing.assert_close(e[0], e[1] + e[2], rtol=1e-6, atol=0)  # anneal weight 1
    assert all(not d["value"].requires_grad for d in tr.last_logs + tr.last_logs_unsup)

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    graph.register_generator_state(gen)
    with torch.cuda.graph(graph):
        out = step()
    tr.global_step.zero_()
    gen.manual_seed(21)
    for i in range(3):
        graph.replay()
        got = [x.clone() for x in out]
        for j in (3, 4):  # patch mask and augmentation: the same draws
            assert torch.equal(eager[i][j], got[j]), (i, j)
        for j in range(3):
            torch.testing.assert_close(got[j], eager[i][j], rtol=1e-6, atol=0, msg=f"replay {i}, value {j}")
        # gradients: the head's bias gradient and the loss kernels' keypoint gradients are summed with float atomics
        for a, b in zip(eager[i][5:], got[5:]):
            assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()), i
    torch.cuda.synchronize(dev)
    assert tr.global_step.item() == 3

    # the anneal weight is read by the replay: the same draws with weight 0.25 move the unsupervised part only
    tr.global_step.fill_(2)
    gen.manual_seed(21)
    graph.replay()
    base = [x.clone() for x in out[:3]]
    tr.global_step.fill_(2)
    gen.manual_seed(21)
    tr.total_unsupervised_importance.fill_(0.25)
    graph.replay()
    torch.cuda.synchronize(dev)
    for j in (1, 2):  # the labeled part and the unsupervised part before the anneal weight
        torch.testing.assert_close(out[j], base[j], rtol=1e-6, atol=0)
    torch.testing.assert_close(base[0], base[1] + base[2], rtol=1e-6, atol=0)
    torch.testing.assert_close(out[0], base[1] + 0.25 * base[2], rtol=1e-6, atol=0)
    assert float((out[0] - base[0]).abs()) > 1e-3 * float(base[2].abs())


# ---- 5. the labeled branch is the labeled step -----------------------------------------------------------------------------
def test_labeled_branch_equals_the_labeled_training_step(dev):
    """The semi-supervised step's labeled part (heatmap MSE, not annealed) is what HeatmapTrackerMultiviewTransformer's
    own training_step returns for the same labeled batch and weights, whatever the anneal weight."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    case = "config4"
    v, k = CASES[case][:2]
    semi = tracker(dev, case)
    semi.total_unsupervised_importance.fill_(0.3)
    torch.manual_seed(17)
    plain = HeatmapTrackerMultiviewTransformer(k, v, Patch(), Mix(), D, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)).to(dev)
    plain.load_state_dict(semi.state_dict())
    want = plain.training_step(labeled_batch(dev, case), 0)["loss"].detach()
    semi.training_step({"labeled": labeled_batch(dev, case), "unlabeled": unlabeled_batch(dev, case)}, 0)
    assert [e["name"] for e in semi.last_logs] == [e["name"] for e in plain.last_logs]
    assert torch.equal(semi.last_logs[-1]["value"], want) and semi.last_logs[-1]["name"] == "train_heatmap_mse_loss_weighted"
    assert plain.global_step.item() == semi.global_step.item() == 1
