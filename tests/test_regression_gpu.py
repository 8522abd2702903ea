"""GPU: the regression head, losses, trackers and predictors against float64 references (tests/regression_oracle.py,
checked against the reference's own outputs on the CPU)."""
import numpy as np
import pytest
import torch
from torch import nn

import regression_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = {torch.bfloat16: 8e-3, torch.float16: 1e-3, torch.float32: 1e-5}  # the d-feature store's rounding


def _features(b, c, h, w, dtype, channels_last, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(b, c, h, w, generator=g) * 2 + 0.5).to(dtype)
    x = x.to(DEV)
    return x.to(memory_format=torch.channels_last) if channels_last else x


def _close(got, want, rel, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err, scale = float(np.abs(got - want).max()), float(np.abs(want).max())
    assert err <= rel * scale + 1e-12, (what, err, scale)


@pytest.mark.parametrize("k", [17, 51])
@pytest.mark.parametrize("b", [3, 300])  # 300 frames: past one wave of the 132 SMs on the frame axis
@pytest.mark.parametrize("c,h,w", [(256, 12, 12), (256, 1, 1), (100, 7, 5)])  # (100, 7, 5): the scalar (unvectorised) paths
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_head_forward_and_gradients(dtype, channels_last, c, h, w, b, k):
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead

    torch.manual_seed(1)
    head = LinearRegressionHead(c, 2 * k).to(DEV)
    x = _features(b, c, h, w, dtype, channels_last).requires_grad_(True)
    y = head(x)
    g = torch.randn(b, 2 * k, device=DEV)
    y.backward(g)
    wt, bs = head.linear_layer.weight.detach().cpu().numpy(), head.linear_layer.bias.detach().cpu().numpy()
    want, pooled = O.head_forward(x.detach().float().cpu().numpy(), wt, bs)
    _close(y.detach().cpu(), want, 1e-5, "out")
    dx, dw, db = O.head_backward(g.cpu().numpy(), pooled, wt, (b, c, h, w))
    assert x.grad.dtype == dtype and x.grad.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    _close(x.grad.float().cpu(), dx, TOL[dtype], "d features")
    _close(head.linear_layer.weight.grad.cpu(), dw, 1e-5, "d weight")
    _close(head.linear_layer.bias.grad.cpu(), db, 1e-5, "d bias")
    # fixed-order sums: the same bits again
    grads = [x.grad.clone(), head.linear_layer.weight.grad.clone(), head.linear_layer.bias.grad.clone()]
    x.grad = None
    head.zero_grad(set_to_none=True)
    y2 = head(x)
    y2.backward(g)
    assert torch.equal(y2, y)
    for a, b_ in zip(grads, [x.grad, head.linear_layer.weight.grad, head.linear_layer.bias.grad]):
        assert torch.equal(a, b_)


@pytest.mark.parametrize("case", ["clean", "whole_pairs", "x_only_shift", "mixed", "all_nan"])
def test_losses_against_the_reference(golden, case):
    from lightning_pose_b200 import ops

    g = golden("regression")
    t = torch.from_numpy(g[f"loss_{case}_targ"]).float().to(DEV)
    p = torch.from_numpy(g[f"loss_{case}_pred"]).float().to(DEV).requires_grad_(True)
    mse, kept, rmse, pairs = ops.regression_losses(t, p)
    want_mse, n_kept = O.regression_mse(t.cpu().numpy(), p.detach().cpu().numpy())
    np.testing.assert_allclose(float(mse), want_mse, rtol=1e-6, equal_nan=True)
    np.testing.assert_allclose(float(mse), float(g[f"loss_{case}_mse"]), rtol=1e-5, equal_nan=True)
    np.testing.assert_allclose(float(rmse), O.regression_rmse(t.cpu().numpy(), p.detach().cpu().numpy()), rtol=1e-6, equal_nan=True)
    assert int(kept) == n_kept and int(pairs) == n_kept // 2
    mse.backward()
    tt, pp = t.double().cpu(), p.detach().double().cpu()
    keep = ~torch.isnan(tt)
    want = torch.where(keep, 2 * (pp - torch.nan_to_num(tt)) / max(n_kept, 1), torch.zeros_like(pp))
    torch.testing.assert_close(p.grad.double().cpu(), want, rtol=1e-5, atol=1e-7)


def test_losses_past_one_chunk_and_at_the_edges():
    """Many chunks of the single-CTA scan with x-only / y-only NaNs carrying a pair across chunk edges; a NaN prediction
    at a kept entry makes both losses NaN; an odd kept count makes the RMSE NaN (the reference raises there)."""
    from lightning_pose_b200 import ops

    torch.manual_seed(3)
    t = torch.rand(300, 34, device=DEV) * 384
    p = t + torch.randn_like(t) * 4
    drop = torch.rand_like(t) < 0.1
    t[drop] = float("nan")
    if int((~torch.isnan(t)).sum()) % 2:
        t.view(-1)[torch.nonzero(~torch.isnan(t.view(-1)))[0]] = float("nan")
    mse, kept, rmse, _ = ops.regression_losses(t, p)
    np.testing.assert_allclose(float(mse), O.regression_mse(t.cpu().numpy(), p.cpu().numpy())[0], rtol=1e-6)
    np.testing.assert_allclose(float(rmse), O.regression_rmse(t.cpu().numpy(), p.cpu().numpy()), rtol=1e-6)
    p2 = p.clone()
    p2.view(-1)[torch.nonzero(~torch.isnan(t.view(-1)))[5]] = float("nan")
    out = ops.regression_losses(t, p2)
    assert torch.isnan(out[0]) and torch.isnan(out[2])
    t3 = t.clone()
    t3.view(-1)[torch.nonzero(~torch.isnan(t.view(-1)))[0]] = float("nan")
    out = ops.regression_losses(t3, p)
    assert torch.isfinite(out[0]) and torch.isnan(out[2]) and int(out[1]) % 2 == 1
    # nothing kept: NaN loss, zero gradient (the reference's empty masked mean)
    pe = p.clone().requires_grad_(True)
    out = ops.regression_losses(torch.full_like(t, float("nan")), pe)
    out[0].backward()
    assert torch.isnan(out[0]) and int(out[1]) == 0 and float(pe.grad.abs().max()) == 0.0


class _Stem(nn.Module):
    """A stand-in backbone: (B, 3, 64, 64) -> (B, 128, 4, 4)."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 128, 16, stride=16)

    def forward(self, x):
        return torch.tanh(self.conv(x))


def _tracker(semi):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.regression_tracker import RegressionTracker, SemiSupervisedRegressionTracker

    sup = LossFactory({"regression": {"log_weight": 0.0}}, None)
    kw = dict(backbone=_Stem(), num_fc_input_features=128, loss_factory=sup)
    if semi:
        unsup = LossFactory({"temporal": {"log_weight": 1.0, "epsilon": 0.01}}, None)
        return SemiSupervisedRegressionTracker(17, loss_factory_unsupervised=unsup, **kw).to(DEV)
    return RegressionTracker(17, **kw).to(DEV)


def _batches(seed=5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    images = torch.randn(8, 3, 64, 64, device=DEV, generator=g)
    kp = torch.rand(8, 34, device=DEV, generator=g) * 64
    kp[1, 4:6] = float("nan")
    kp[3, 7] = float("nan")  # x-only NaN ...
    kp[5, 10] = float("nan")  # ... and y-only: the RMSE re-pairs between them
    frames = torch.randn(6, 3, 64, 64, device=DEV, generator=g)
    tf = torch.tensor([[1.05, -0.1, 3.0], [0.08, 0.95, -2.0]], device=DEV)
    return {"images": images, "keypoints": kp}, {"frames": frames, "transforms": tf}


def _oracle_b(tr, labeled, unlabeled):
    """The reference's tracker restated in float64 torch: backbone + avgpool + LinearRegressionHead, RegressionMSELoss
    (masked_select mean), RegressionRMSELoss, undo_affine_transform and TemporalLoss without confidences, summed with
    the loss factory's weights 1 / (2 exp(log_weight))."""
    import copy

    bb = copy.deepcopy(tr.backbone).double()
    lin = copy.deepcopy(tr.head.linear_layer).double()
    params = list(bb.parameters()) + list(lin.parameters())

    def forward(x):
        f = bb(x.double())
        return lin(torch.nn.functional.adaptive_avg_pool2d(f, 1).reshape(f.shape[0], -1))

    pred = forward(labeled["images"])
    t = labeled["keypoints"].double()
    keep = ~torch.isnan(t)
    mse = torch.mean((torch.masked_select(t, keep) - torch.masked_select(pred, keep)) ** 2)
    d2 = (torch.masked_select(t, keep) - torch.masked_select(pred, keep)).reshape(-1, 2) ** 2
    rmse = torch.mean(torch.sqrt(d2.mean(1)))
    total = 0.5 * mse
    if unlabeled is not None:
        kp = forward(unlabeled["frames"]).reshape(6, -1, 2)
        m = unlabeled["transforms"].double()
        a_inv = torch.linalg.inv(m[:, :2])
        kp = ((kp - m[:, 2]) @ a_inv.T).reshape(6, -1)
        d = torch.diff(kp, dim=0).reshape(5, -1, 2)
        temporal = torch.relu(torch.linalg.norm(d, dim=-1) - 0.01).mean()
        total = total + 1.0 / (2.0 * np.exp(1.0)) * temporal
    grads = torch.autograd.grad(total, params)
    return total, rmse, grads


@pytest.fixture
def deterministic_cudnn():
    """The stand-in backbone's convolutions are torch's: their weight gradient is reproducible only with cuDNN's
    deterministic algorithms.  Everything else in the step is this package's fixed-order kernels."""
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
        yield


@pytest.mark.parametrize("semi", [False, True])
def test_training_step_against_oracle_b_graph_and_bits(semi, deterministic_cudnn):
    torch.manual_seed(0)
    tr = _tracker(semi)
    labeled, unlabeled = _batches()
    params = list(tr.backbone.parameters()) + list(tr.head.parameters())

    def step():
        batch = {"labeled": labeled, "unlabeled": unlabeled} if semi else labeled
        loss = tr.training_step(batch, 0)["loss"]
        return [loss.detach(), tr.last_rmse.detach(), *torch.autograd.grad(loss, params)]

    eager = step()
    total, rmse, grads = _oracle_b(tr, labeled, unlabeled if semi else None)
    torch.testing.assert_close(eager[0].double().cpu(), total.detach().cpu(), rtol=1e-5, atol=0)
    torch.testing.assert_close(eager[1].double().cpu(), rmse.detach().cpu(), rtol=1e-5, atol=0)
    for a, b in zip(eager[2:], grads):
        _close(a.cpu(), b.cpu(), 1e-4, "gradient")
    again = step()
    for a, b in zip(eager, again):
        assert torch.equal(a, b)  # bit-identical run to run

    # the whole step, augmented ingest included, captured into one graph and replayed
    from lightning_pose_b200 import ops

    gen = torch.Generator(device=DEV)
    u8 = torch.randint(0, 256, (6, 80, 80, 3), device=DEV, dtype=torch.uint8)

    def graph_step():
        if semi:
            prm, seeds = ops.draw_dlc_params(1, DEV, generator=gen)
            unlabeled["frames"], unlabeled["transforms"] = ops.frames_augment_normalize(u8, (64, 64), prm[0], seeds[:1])
            return [*step(), unlabeled["transforms"]]
        return step()

    gen.manual_seed(7)
    ref = [[x.clone() for x in graph_step()] for _ in range(2)]
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        for _ in range(2):
            graph_step()
    torch.cuda.current_stream(DEV).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    graph.register_generator_state(gen)
    with torch.cuda.graph(graph):
        out = graph_step()
    gen.manual_seed(7)
    for i in range(2):
        graph.replay()
        for a, b in zip(ref[i], out):
            assert torch.equal(a, b), i
    if semi:
        assert not torch.equal(ref[0][-1], ref[1][-1]) and not torch.equal(ref[0][0], ref[1][0])  # fresh draws per replay


def test_predictors_against_predict_step(deterministic_cudnn):
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead
    from lightning_pose_b200.models.regression_tracker import RegressionTracker
    from lightning_pose_b200.utils.predictions import BatchedPredictor, FramePredictor

    # video: streamed features (the head's kernels treat every frame alone, so chunking cannot change a bit)
    torch.manual_seed(2)
    tr = RegressionTracker(17, backbone=nn.Identity(), num_fc_input_features=128).to(DEV).eval()
    frames = torch.randn(10, 128, 4, 4, device=DEV).bfloat16()
    with torch.no_grad():
        kp, cf = tr.predict_step({"frames": frames}, 0)
    assert cf.device == kp.device and float(cf.abs().max()) == 0.0
    want = torch.stack([kp[:, 0::2], kp[:, 1::2], cf], -1).reshape(10, -1)
    pred = BatchedPredictor(tr.head, 17, n_frames=10, chunk=4, image_hw=(64, 64))
    for i in range(0, 12, 4):
        chunk = frames[i : i + 4]
        pred.feed(torch.cat([chunk, chunk[-1:].expand(4 - chunk.shape[0], -1, -1, -1)]) if chunk.shape[0] < 4 else chunk)
    assert torch.equal(pred.table, want)
    assert isinstance(tr.head, LinearRegressionHead)
    with pytest.raises(ValueError, match="multiview"):
        BatchedPredictor(tr.head, 17, n_frames=10, chunk=4, image_hw=(64, 64), num_views=2)
    with pytest.raises(ValueError, match="model pixels"):
        pred.feed(frames[:4], torch.zeros(4, 4, device=DEV))

    tr = _tracker(False).eval()

    # one frame: the reference's predict_frame maps the model-pixel keypoints to the frame and reports confidence 1.0
    from lightning_pose_b200 import ops

    u8 = torch.randint(0, 256, (90, 120, 3), dtype=torch.uint8)
    fp = FramePredictor(tr.head, 17, (64, 64), tr.backbone)
    res = fp.predict_frame(u8.numpy(), bbox=(10, 5, 80, 70))
    x, box = ops.frames_crop_resize_cv2(u8.to(DEV)[None], (64, 64), torch.tensor([10, 5, 80, 70], dtype=torch.int32, device=DEV))
    with torch.no_grad():
        kp1, _ = tr.predict_step({"images": x}, 0)
        kp1 = ops.remap_keypoints(kp1, None, box, 64, 64)
    # the stand-in backbone is torch's convolution, run from a graph on one side and eagerly on the other
    np.testing.assert_allclose(res["keypoints"], kp1.cpu().numpy().reshape(17, 2), rtol=1e-5, atol=1e-5)
    assert np.all(res["confidence"] == 1.0)
