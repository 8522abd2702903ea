"""GPU: multi-view video prediction.  The one-launch ingest (lpb_frames_normalize_views) against per-view
lpb_frames_normalize and a float64 restatement of the resize; BatchedPredictor's multi-view mode against the CPU oracle,
against the trackers' own predict_step on the batches frames_to_unlabeled_batch builds, over split frame ranges, and
its launch count."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def float64_ingest(u8, size):
    """uint8 (F, H, W, 3) -> (F, 3, h, w) float64: bilinear, half-pixel centres, no antialiasing, then /255 + ImageNet."""
    from lightning_pose_b200 import ops

    x = u8.cpu().permute(0, 3, 1, 2).double()
    if tuple(x.shape[-2:]) != tuple(size):
        x = F.interpolate(x, size=size, mode="bilinear", align_corners=False, antialias=False)
    mean = torch.tensor(ops.IMAGENET_MEAN, dtype=torch.float64).view(1, 3, 1, 1)
    std = torch.tensor(ops.IMAGENET_STD, dtype=torch.float64).view(1, 3, 1, 1)
    return (x / 255.0 - mean) / std


@pytest.mark.parametrize("size", [(384, 384), (256, 320)])
@pytest.mark.parametrize("dtype,channels_last", [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False), (torch.bfloat16, True)])
def test_ingest_views_matches_per_view_normalize(size, dtype, channels_last):
    from lightning_pose_b200 import ops

    gen = torch.Generator(device=DEV).manual_seed(5)
    shapes = [(1024, 1280), (720, 1280), (406, 396), size, (300, 333)]  # one view already at the model size, one odd width
    views = [torch.randint(0, 256, (3, h, w, 3), dtype=torch.uint8, device=DEV, generator=gen) for h, w in shapes]
    out = ops.frames_normalize_views(views, size, channels_last=channels_last, dtype=dtype)
    assert out.shape == ((3, 5, *size, 3) if channels_last else (3, 5, 3, *size)) and out.dtype == dtype
    tol = dict(atol=2e-3, rtol=0) if dtype == torch.float32 else dict(atol=2e-2, rtol=1e-2)
    for v, u8 in enumerate(views):
        mine = out[:, v]
        assert torch.equal(mine, ops.frames_normalize(u8, size=size, channels_last=channels_last, dtype=dtype)), v
        got = (mine.permute(0, 3, 1, 2) if channels_last else mine).double().cpu()
        np.testing.assert_allclose(got.numpy(), float64_ingest(u8, size).numpy(), **tol)


def test_ingest_views_past_2_31_elements():
    """4,900 frame-views of 384 x 384 in bf16: 2.17e9 output elements (4.3 GB), from small source frames."""
    from lightning_pose_b200 import ops

    gen = torch.Generator(device=DEV).manual_seed(6)
    f, size = 2450, (384, 384)
    views = [torch.randint(0, 256, (f, h, w, 3), dtype=torch.uint8, device=DEV, generator=gen) for h, w in ((12, 16), (9, 7))]
    out = ops.frames_normalize_views(views, size, dtype=torch.bfloat16)
    assert out.numel() > 2**31
    for v, u8 in enumerate(views):
        assert torch.equal(out[:, v], ops.frames_normalize(u8, size=size, dtype=torch.bfloat16)), v
    # the last frames lie past element 2^31 of the output: check them against the float64 restatement too
    got = out[-2:].float().cpu()
    for v, u8 in enumerate(views):
        np.testing.assert_allclose(got[:, v].double().numpy(), float64_ingest(u8[-2:], size).numpy(), atol=2e-2, rtol=1e-2)


def make_head(c, k, seed, arch="resnet50"):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead(arch, c, k)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return head


@pytest.mark.parametrize("views", [2, 3, 4])
def test_multiview_predictor_matches_oracle(views):
    """Features in, (N, 3 V K) table out; N = 20 in chunks of 8 (the last one padded), graph and eager."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor
    from oracle import lp_oracle as O

    k, n, chunk, c, fh, img = 17, 20, 8, 512, 4, 128
    head = make_head(c, k, 10 + views)
    feats = torch.randn(n * views, c, fh, fh) * 0.5
    sizes = torch.tensor([[200.0, 260.0], [150.0, 180.0], [480.0, 640.0], [128.0, 128.0]])[:views]
    bbox = torch.cat([torch.cat([torch.tensor([[3.0 * v, 5.0]]).repeat(n, 1) + torch.arange(n)[:, None], sizes[v].repeat(n, 1)], 1)
                      for v in range(views)], 1)
    deconvs = list(head.upsampling_layers)[1:]
    hm = O.head_forward(feats, [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs])
    kp_ref, cf_ref = O.decode_softargmax(hm, 2, 1000.0)
    kp_ref = O.model_to_frame(kp_ref.reshape(n, -1), bbox, img, img, num_views=views)
    cf_ref = cf_ref.reshape(n, -1)
    head = head.to(DEV).eval()
    pad = (-n) % chunk
    f_dev = torch.cat([feats, feats[-views:].repeat(pad, 1, 1, 1)]).to(DEV)
    b_dev = torch.cat([bbox, bbox[-1:].repeat(pad, 1)]).to(DEV)
    tables = []
    for use_graph in (True, False):
        bp = BatchedPredictor(head, k, n, chunk, (img, img), use_graph=use_graph, num_views=views)
        bp.run((f_dev[i * views : (i + chunk) * views], b_dev[i : i + chunk]) for i in range(0, n + pad, chunk))
        kp, cf = bp.results()
        assert kp.shape == (n, 2 * views * k) and cf.shape == (n, views * k)
        np.testing.assert_allclose(kp.cpu().numpy(), kp_ref.numpy(), rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(cf.cpu().numpy(), cf_ref.numpy(), rtol=1e-4, atol=1e-5)
        assert int(bp.cursor) == n + pad
        vt = bp.view_tables()
        assert len(vt) == views and all(torch.equal(vt[v], bp.table[:, 3 * k * v : 3 * k * (v + 1)]) for v in range(views))
        tables.append(bp.table.clone())
    assert torch.equal(tables[0], tables[1])


class Patch(torch.nn.Module):  # the stand-in patch embedding of scripts/bench_configs.py
    def __init__(self):
        super().__init__()
        self.proj = torch.nn.Conv2d(3, 384, 16, stride=16)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class Mix(torch.nn.Module):  # the stand-in encoder of scripts/bench_configs.py
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(384, 384)

    def forward(self, t):
        return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()


def make_tracker(kind, k, views):
    """(model, features_of, model_type) on the device, eval."""
    if kind == "transformer":
        from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

        model = HeatmapTrackerMultiviewTransformer(k, views, Patch(), Mix(), 384).to(DEV).eval()
        return model, model.forward_vit, "heatmap_multiview_transformer"
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    model = HeatmapTracker(k, backbone=torch.nn.Conv2d(3, 512, 32, stride=32), num_fc_input_features=512)
    for layer in list(model.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    model = model.to(DEV).eval()
    return model, model.get_representations, "heatmap"


def video_views(n, shapes, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=DEV, generator=gen) for h, w in shapes]


def chunked(views, chunk):
    """The views cut into chunks of ``chunk`` frames, the last one padded with the final frame."""
    n = views[0].shape[0]
    pad = (-n) % chunk
    full = [torch.cat([v, v[-1:].repeat(pad, 1, 1, 1)]) for v in views]
    return [[v[i : i + chunk] for v in full] for i in range(0, n + pad, chunk)]


SHAPES = [(150, 200), (128, 128), (97, 131), (240, 180)]


@pytest.mark.parametrize("kind", ["heatmap", "transformer"])
def test_multiview_predictor_matches_predict_step(kind):
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch
    from lightning_pose_b200.utils.predictions import BatchedPredictor, PredictionHandler

    k, n, chunk, img, views = 17, 20, 8, 128, 4
    model, features_of, model_type = make_tracker(kind, k, views)
    vids = video_views(n, SHAPES, 21)
    bp = BatchedPredictor(model.head, k, n, chunk, (img, img), features_of=features_of, num_views=views)
    preds = []
    for i, ch in enumerate(chunked(vids, chunk)):
        bp.feed(ch)
        with torch.no_grad():
            preds.append(model.predict_step(frames_to_unlabeled_batch(ch, resize_dims=(img, img)), i))
    assert int(bp.cursor) == 24
    kp_ref = torch.cat([p[0] for p in preds])[:n]
    cf_ref = torch.cat([p[1] for p in preds])[:n]
    kp, cf = bp.results()
    np.testing.assert_allclose(kp.cpu().numpy(), kp_ref.cpu().numpy(), rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(cf.cpu().numpy(), cf_ref.cpu().numpy(), rtol=1e-4, atol=1e-5)

    names, view_names = [f"bp{j}" for j in range(k)], ["top", "side", "front", "back"]
    ph = PredictionHandler(names, n, model_type=model_type, view_names=view_names)
    from_table = ph.dataframes(bp.table)
    from_step = ph(preds, is_multiview_video=True)
    from_results = ph([(kp, cf)], is_multiview_video=True)
    assert list(from_table) == list(from_step) == view_names
    for v in view_names:  # the table's frames hold its fp32 values, the reference call form's float64 copies of them
        np.testing.assert_array_equal(from_table[v].to_numpy(), from_results[v].to_numpy())
        assert from_table[v].columns.equals(from_results[v].columns) and from_table[v].columns.equals(from_step[v].columns)
        assert from_table[v].columns[0][0] == f"{model_type}_tracker"
        np.testing.assert_allclose(from_table[v].to_numpy(), from_step[v].to_numpy(), rtol=1e-4, atol=2e-3)


def test_multiview_predictor_rank_split():
    """Two predictors over frame_range_for_rank(N, r, 2), one after the other, give the single predictor's table."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor, frame_range_for_rank

    k, n, chunk, img, views = 17, 32, 8, 128, 3
    model, features_of, _ = make_tracker("heatmap", k, views)
    vids = video_views(n, SHAPES[:views], 22)
    whole = BatchedPredictor(model.head, k, n, chunk, (img, img), features_of=features_of, num_views=views)
    whole.run(chunked(vids, chunk))
    parts = []
    for r in range(2):
        a, b = frame_range_for_rank(n, r, 2)
        bp = BatchedPredictor(model.head, k, b - a, chunk, (img, img), features_of=features_of, num_views=views)
        bp.run(chunked([v[a:b] for v in vids], chunk))
        parts.append(bp.table)
    assert torch.equal(torch.cat(parts), whole.table)


def test_multiview_predictor_launch_count():
    """uint8 views in: one launch more than the same predictor fed the normalised (T, V, 3, h, w) frames, the ingest."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    k, n, chunk, img, views = 17, 16, 8, 128, 4
    model, features_of, _ = make_tracker("transformer", k, views)
    vids = video_views(n, SHAPES, 23)
    ch = chunked(vids, chunk)
    u8 = BatchedPredictor(model.head, k, n, chunk, (img, img), features_of=features_of, num_views=views)
    fr = BatchedPredictor(model.head, k, n, chunk, (img, img), features_of=features_of, num_views=views)
    for c in ch:
        u8.feed(c)
        boxes = torch.tensor([[0.0, 0.0, float(h), float(w)] for h, w in SHAPES], device=DEV).reshape(1, -1).repeat(chunk, 1)
        fr.feed(ops.frames_normalize_views(c, (img, img)), boxes)
    assert u8.launches_per_chunk == fr.launches_per_chunk + 1, (u8.launches_per_chunk, fr.launches_per_chunk)
    assert torch.equal(u8.table, fr.table)
