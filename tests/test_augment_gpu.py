"""GPU: augmented unlabeled-video ingest (csrc/ingest.cu, augment_kernel) against the float64 oracle
(tests/augment_oracle.py): frames and transform, identity against the plain ingest, geometry end to end through the
remap, the shot-noise distribution, determinism, CUDA-graph replay and both semi-supervised trackers."""
import numpy as np
import pytest
import torch

import augment_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LAYOUTS = [(torch.float32, False), (torch.bfloat16, False), (torch.bfloat16, True)]


def fchw(x):
    """(F, 3, h, w) or channels-last (F, h, w, 3) -> float64 FCHW numpy."""
    x = x.float()
    return (x.permute(0, 3, 1, 2) if x.shape[-1] == 3 else x).double().cpu().numpy()


def params_dev(p):
    return torch.tensor(np.asarray(p, np.float32), device=DEV)


def seed_dev(s):
    return torch.tensor([s], dtype=torch.int64, device=DEV)


def random_params(rng, factor=0.0):
    lo, hi = np.array([-10, 0.8, 0.8, 0.75, 0.75, 0.0]), np.array([10, 1.2, 1.2, 1.25, 1.25, 10.0])
    p = (lo + (hi - lo) * rng.random(6)).astype(np.float32)
    p[5] = factor
    return p


@pytest.mark.parametrize("dtype,channels_last", LAYOUTS)
@pytest.mark.parametrize("src,size", [((100, 140), (64, 96)), ((50, 70), (64, 64)), ((406, 396), (384, 384))])
def test_parity_with_oracle(src, size, dtype, channels_last):
    from lightning_pose_b200 import ops

    rng = np.random.default_rng(hash((src, size)) % 2**32)
    views = [rng.integers(0, 256, size=(3, *src, 3), dtype=np.uint8) for _ in range(2)]
    for v, u8 in enumerate(views):  # two views, each with its own draw
        p = random_params(rng)
        frames, tf = ops.frames_augment_normalize(torch.from_numpy(u8).to(DEV), size, params_dev(p), seed_dev(v),
                                                  channels_last=channels_last, dtype=dtype)
        want, m = O.augment(u8, size, p.astype(np.float64))
        assert frames.shape == ((3, *size, 3) if channels_last else (3, 3, *size)) and frames.dtype == dtype
        np.testing.assert_allclose(tf.cpu().numpy(), m, rtol=1e-6, atol=1e-6 * np.abs(m).max())
        if dtype == torch.float32:
            np.testing.assert_allclose(fchw(frames), want, atol=2e-4, rtol=0)
        else:  # the plain ingest's bf16 tolerance (test_video_ingest_boundary)
            np.testing.assert_allclose(fchw(frames), want, atol=2e-2, rtol=1e-2)


@pytest.mark.parametrize("dtype,channels_last", LAYOUTS)
@pytest.mark.parametrize("size", [(64, 96), (100, 140)])
def test_identity_parameters_give_the_plain_ingest(size, dtype, channels_last):
    from lightning_pose_b200 import ops

    u8 = torch.randint(0, 256, (4, 100, 140, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).to(DEV)
    plain = ops.frames_normalize(u8, size=size, channels_last=channels_last, dtype=dtype)
    aug, tf = ops.frames_augment_normalize(u8, size, params_dev([0, 1, 1, 1, 1, 0]), seed_dev(1), channels_last=channels_last, dtype=dtype)
    assert tf.tolist() == [[1, 0, 0], [0, 1, 0]]
    # only step 5's fp32 rounding, (v - 0.5) + 0.5, separates the two: one ulp of 255 after normalisation
    tol = 1e-6 if dtype == torch.float32 else 1e-2
    np.testing.assert_allclose(fchw(aug), fchw(plain), atol=tol, rtol=tol)


def blob_frames(n, h, w, centres, sigma):
    """uint8 (n, h, w, 3) Gaussian blobs on black, one frame per row of centres (x, y)."""
    yy, xx = np.meshgrid(np.arange(h) + 0.0, np.arange(w) + 0.0, indexing="ij")
    out = np.zeros((n, h, w), np.float64)
    for i in range(n):
        for cx, cy in centres[i]:
            out[i] += 250 * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * sigma**2))
    return np.repeat(np.round(np.minimum(out, 255)).astype(np.uint8)[..., None], 3, axis=-1)


def centroids(img, guesses, radius):
    """Intensity centroids (x, y) of channel 0 of (h, w) image inside a box of +- radius around each guess."""
    h, w = img.shape
    yy, xx = np.meshgrid(np.arange(h) + 0.0, np.arange(w) + 0.0, indexing="ij")
    res = []
    for gx, gy in guesses:
        m = (np.abs(xx - gx) <= radius) & (np.abs(yy - gy) <= radius)
        wgt = img * m
        res.append([(wgt * xx).sum() / wgt.sum(), (wgt * yy).sum() / wgt.sum()])
    return np.array(res)


def to_255(frames):
    """normalised fp32 FCHW -> 0..255 channel 0."""
    return (fchw(frames)[:, 0] * O.STD[0] + O.MEAN[0]) * 255.0


def test_geometry_end_to_end():
    """Blob centroids move by the returned transform (DALI's half-pixel convention), and the remap of the augmented
    centroids is the reference's undo + model_to_frame of them.  The reference undo inverts M on raw coordinates, so
    it returns c + (I - A^-1) (0.5, 0.5) rather than the plain centroid c: that bias is the reference's own and is part
    of the expected value."""
    from lightning_pose_b200 import ops

    rng = np.random.default_rng(11)
    src, size, n = (300, 420), (150, 210), 3
    # three blobs per frame in resized coordinates (x, y), >= 50 px apart and clear of the border after any draw
    cen = [np.array([[60.0, 50.0], [150.0, 50.0], [105.0, 100.0]]) + rng.uniform(-4, 4, size=(3, 2)) for _ in range(n)]
    u8 = blob_frames(n, *src, [c * 2.0 + 0.5 for c in cen], sigma=8.0)  # resized centre c <-> source 2 c + 0.5
    x = torch.from_numpy(u8).to(DEV)
    plain = to_255(ops.frames_normalize(x, size=size))
    views = []
    for v in range(2):
        p = random_params(rng)
        p[3:5] = 1.0
        frames, tf = ops.frames_augment_normalize(x, size, params_dev(p), seed_dev(v))
        aug = to_255(frames)
        m = tf.double().cpu().numpy()
        a, t = m[:, :2], m[:, 2]
        kp_aug = []
        for i in range(n):
            c = centroids(plain[i], cen[i], 16)
            want = (c + 0.5) @ a.T + t - 0.5
            got = centroids(aug[i], want, 16)
            np.testing.assert_allclose(got, want, atol=0.05, rtol=0)
            kp_aug.append(got)
            bias = O.undo_then_model_to_frame(got[None], m, np.array([[0, 0, size[0], size[1]]]), *size)[0] - c
            np.testing.assert_allclose(bias, np.broadcast_to((np.eye(2) - np.linalg.inv(a)) @ [0.5, 0.5], bias.shape), atol=0.05)
        views.append((np.stack(kp_aug), tf, m))
    bbox_np = np.array([[3.0, 5.0, 300.0, 420.0]]).repeat(n, 0)
    bbox = torch.tensor(bbox_np, dtype=torch.float32, device=DEV)
    kp0, tf0, m0 = views[0]
    got = ops.remap_keypoints(torch.tensor(kp0.reshape(n, -1), dtype=torch.float32, device=DEV), tf0, bbox, *size)
    want = O.undo_then_model_to_frame(kp0, m0, bbox_np, *size)
    np.testing.assert_allclose(got.cpu().numpy().reshape(n, -1, 2), want, atol=2e-3, rtol=0)
    # two views: (V, 1, 2, 3) transforms, bbox (n, 8), view v's keypoints in its own column block
    kp = np.concatenate([views[0][0], views[1][0]], axis=1)
    tfs = torch.stack([views[0][1], views[1][1]])[:, None]
    bb2 = np.concatenate([bbox_np, bbox_np + [1, 2, 0, 0]], axis=1)
    got = ops.remap_keypoints(torch.tensor(kp.reshape(n, -1), dtype=torch.float32, device=DEV), tfs,
                              torch.tensor(bb2, dtype=torch.float32, device=DEV), *size, is_multiview=True, num_views=2)
    want = np.concatenate([O.undo_then_model_to_frame(views[v][0], views[v][2], bb2[:, 4 * v : 4 * v + 4], *size) for v in range(2)], axis=1)
    np.testing.assert_allclose(got.cpu().numpy().reshape(n, -1, 2), want, atol=2e-3, rtol=0)


@pytest.mark.parametrize("lam", [0.3, 3.0, 30.0, 300.0, 3e4])
def test_shot_noise_distribution(lam):
    from scipy import stats

    from lightning_pose_b200 import ops

    level = 150.0
    factor = np.float32(level / lam)
    lam32 = float(np.float32(level) / factor)
    u8 = torch.full((2, 96, 128, 3), int(level), dtype=torch.uint8, device=DEV)
    frames, _ = ops.frames_augment_normalize(u8, (96, 128), params_dev([0, 1, 1, 1, 1, factor]), seed_dev(1234))
    out = (fchw(frames) * O.STD[None, :, None, None] + O.MEAN[None, :, None, None]) * 255.0  # (2, 3, h, w) in 0..255
    k = np.round(out / float(factor))
    assert np.abs(k - out / float(factor)).max() < 0.05
    s = k.reshape(-1)
    n = s.size
    se_mean = (lam32 / n) ** 0.5
    se_var = ((lam32 + 2 * lam32**2) / n) ** 0.5
    assert abs(s.mean() - lam32) < 5 * se_mean, (s.mean(), lam32)
    assert abs(s.var() - lam32) < 5 * se_var, (s.var(), lam32)
    if lam <= 30:
        # bins k <= lo, lo < k < hi one by one, k >= hi: both tails merged until they expect >= 5 samples
        ks = np.arange(1000)
        lo = int(np.argmax(stats.poisson.cdf(ks, lam32) * n >= 5))
        hi = int(np.argmax(stats.poisson.sf(ks - 1, lam32) * n < 5)) - 1
        obs = np.bincount(np.clip(s.astype(np.int64), lo, hi) - lo, minlength=hi - lo + 1)
        exp = np.concatenate([[stats.poisson.cdf(lo, lam32)], stats.poisson.pmf(ks[lo + 1 : hi], lam32), [stats.poisson.sf(hi - 1, lam32)]]) * n
        assert exp.min() >= 5 and obs.sum() == n
        assert stats.chisquare(obs, exp).pvalue > 1e-4
    frames_k = k.reshape(2, 3, -1)
    m = frames_k.shape[-1]
    bound = 5 / m**0.5
    assert abs(np.corrcoef(frames_k[0, 0], frames_k[1, 0])[0, 1]) < bound
    assert abs(np.corrcoef(frames_k[0, 0], frames_k[0, 1])[0, 1]) < bound
    assert abs(np.corrcoef(frames_k[0, 1], frames_k[0, 2])[0, 1]) < bound


def test_determinism_and_seeds():
    from lightning_pose_b200 import ops

    u8 = torch.randint(0, 256, (4, 100, 140, 3), dtype=torch.uint8, device=DEV)
    p = params_dev([3.0, 1.1, 0.9, 1.1, 0.8, 4.0])
    a, ta = ops.frames_augment_normalize(u8, (64, 96), p, seed_dev(7))
    b, tb = ops.frames_augment_normalize(u8, (64, 96), p, seed_dev(7))
    c, _ = ops.frames_augment_normalize(u8, (64, 96), p, seed_dev(8))
    assert torch.equal(a, b) and torch.equal(ta, tb)
    assert float((a != c).float().mean()) > 0.5


def test_graph_capture_replays_fresh_draws():
    """draw + augmented ingest + remap captured in one graph: every replay draws new parameters in the reference's
    ranges, and its frames are those of an eager call with the parameters read back from that replay."""
    from lightning_pose_b200 import ops

    size = (64, 96)
    u8 = torch.randint(0, 256, (4, 100, 140, 3), dtype=torch.uint8, device=DEV)
    kp = torch.rand(4, 10, device=DEV) * 60
    bbox = torch.tensor([[0.0, 0.0, 100.0, 140.0]], device=DEV).repeat(4, 1)

    def step():
        params, seeds = ops.draw_dlc_params(1, DEV)
        frames, tf = ops.frames_augment_normalize(u8, size, params[0], seeds[0:1])
        return params, seeds, frames, tf, ops.remap_keypoints(kp, tf, bbox, *size)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static = step()
    seen = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        params, seeds, frames, tf, remapped = [t.clone() for t in static]
        for cols, lo, hi in ops.DLC_PARAM_RANGES:
            assert bool((params[:, cols] >= lo).all() and (params[:, cols] <= hi).all())
        eager, eager_tf = ops.frames_augment_normalize(u8, size, params[0], seeds[0:1])
        assert torch.equal(frames, eager) and torch.equal(tf, eager_tf)
        assert torch.equal(remapped, ops.remap_keypoints(kp, eager_tf, bbox, *size))
        seen.append(params)
    assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2])


def test_unlabeled_batch_surface():
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    u8 = torch.randint(0, 256, (5, 100, 140, 3), dtype=torch.uint8, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(3)
    bd = frames_to_unlabeled_batch(u8, (64, 96), imgaug="dlc", generator=gen)
    assert bd["frames"].shape == (5, 3, 64, 96) and bd["transforms"].shape == (2, 3) and bd["is_multiview"] is False
    assert bd["bbox"].tolist() == [[0.0, 0.0, 100.0, 140.0]] * 5
    again = frames_to_unlabeled_batch(u8, (64, 96), imgaug="dlc", generator=torch.Generator(device=DEV).manual_seed(3))
    assert torch.equal(again["frames"], bd["frames"]) and torch.equal(again["transforms"], bd["transforms"])
    mv = frames_to_unlabeled_batch([u8, u8.flip(0)[:, :90]], (64, 96), imgaug="dlc-top-down", dtype=torch.bfloat16, channels_last=True)
    assert mv["frames"].shape == (5, 2, 64, 96, 3) and mv["frames"].dtype == torch.bfloat16 and mv["is_multiview"] is True
    assert mv["transforms"].shape == (2, 1, 2, 3) and not torch.equal(mv["transforms"][0], mv["transforms"][1])
    assert mv["bbox"].tolist() == [[0.0, 0.0, 100.0, 140.0, 0.0, 0.0, 90.0, 140.0]] * 5
    for imgaug in ("default", None, "dlc-lr"):
        plain = frames_to_unlabeled_batch(u8, (64, 96), imgaug=imgaug)
        assert plain["transforms"].tolist() == [-1.0] and torch.equal(plain["frames"], frames_to_unlabeled_batch(u8, (64, 96))["frames"])


def test_semisupervised_trackers_on_augmented_batches():
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import SemiSupervisedHeatmapTracker
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import SemiSupervisedHeatmapTrackerMHCRNN

    torch.manual_seed(4)
    k = 5
    sup = LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)
    unsup = LossFactory({"temporal": {"log_weight": 1.0, "epsilon": 1.0, "prob_threshold": 0.0}}, None)
    model = SemiSupervisedHeatmapTracker(k, loss_factory=sup, loss_factory_unsupervised=unsup, backbone="resnet18").to(DEV)
    model.train(False)
    imgs = torch.randn(4, 3, 64, 96, device=DEV)
    kps = torch.rand(4, k, 2, device=DEV) * torch.tensor([96.0, 64.0], device=DEV)
    labeled = {"images": imgs, "keypoints": kps.reshape(4, -1), "heatmaps": torch.rand(4, k, 16, 24, device=DEV),
               "bbox": torch.tensor([[0.0, 0.0, 64.0, 96.0]], device=DEV).repeat(4, 1)}
    u8 = torch.randint(0, 256, (6, 100, 140, 3), dtype=torch.uint8, device=DEV)
    unlabeled = frames_to_unlabeled_batch(u8, (64, 96), imgaug="dlc")
    out = model.training_step({"labeled": labeled, "unlabeled": unlabeled}, 0)
    out["loss"].backward()
    assert torch.isfinite(out["loss"]) and torch.isfinite(model.backbone[0].weight.grad).all()
    with torch.no_grad():
        d = model.get_loss_inputs_unlabeled(unlabeled)
    aug = d["keypoints_pred_augmented"].double().cpu().numpy().reshape(6, k, 2)
    want = O.undo_then_model_to_frame(aug, unlabeled["transforms"].double().cpu().numpy(), unlabeled["bbox"].double().cpu().numpy(), 64, 96)
    np.testing.assert_allclose(d["keypoints_pred"].cpu().numpy().reshape(6, k, 2), want, atol=2e-3, rtol=1e-5)

    class Feats(torch.nn.Module):  # a stand-in ViT-S: (n, 3, 256, 256) -> (n, 384, 16, 16) bf16
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 384, 16, stride=16)

        def forward(self, x):
            return self.conv(x).bfloat16()

    tr = SemiSupervisedHeatmapTrackerMHCRNN(
        k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
        loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": 5.0, "epsilon": 5.0, "prob_threshold": 0.05}}, None),
        backbone=Feats(), backbone_arch="vits_dino", num_fc_input_features=384).to(DEV)
    labeled = {"images": torch.randn(2, 5, 3, 256, 256, device=DEV), "keypoints": torch.rand(2, 2 * k, device=DEV) * 256,
               "heatmaps": torch.rand(2, k, 64, 64, device=DEV), "bbox": torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=DEV).repeat(2, 1)}
    seq = torch.randint(0, 256, (16, 300, 280, 3), dtype=torch.uint8, device=DEV)  # dali.context.train.batch_size
    unlabeled = frames_to_unlabeled_batch(seq, (256, 256), imgaug="dlc")
    out = tr.training_step({"labeled": labeled, "unlabeled": unlabeled}, 0)
    out["loss"].backward()
    assert torch.isfinite(out["loss"]) and torch.isfinite(tr.backbone.conv.weight.grad).all()
