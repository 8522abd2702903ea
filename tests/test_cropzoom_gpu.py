"""GPU: crop-zoom inference kernels (csrc/cropzoom.cu) against tests/golden/cropzoom.npz, which holds the reference's
own outputs, and the crop mode of BatchedPredictor against the eager composition of its parts."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cropzoom_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CROP = [c[0] for c in O.CROP_CASES]


def t(a, **kw):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, **kw)


@pytest.mark.parametrize("name", CROP)
def test_crop_matches_golden(golden, name):
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.bboxes import crop_and_resize_frames
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    g = golden("cropzoom")
    want, want_boxes = g[f"crop_{name}_out_frames"], g[f"crop_{name}_out_boxes"]
    size = [int(v) for v in g[f"crop_{name}_in_size"]]
    rows = t(g[f"crop_{name}_in_rows"])
    # fp32 normalised frames, the reference function's own input and signature (a DataFrame of rows)
    import pandas as pd

    df = pd.DataFrame(g[f"crop_{name}_in_rows"].astype(np.float64), columns=["x", "y", "h", "w"])
    out, boxes = crop_and_resize_frames(t(g[f"crop_{name}_in_f32"]), df, size)
    np.testing.assert_allclose(out.cpu().numpy(), want, atol=1e-5, rtol=1e-4)
    np.testing.assert_array_equal(boxes.cpu().numpy(), want_boxes)
    # uint8 surface, crop + resize + normalise in one launch
    u8 = t(g[f"crop_{name}_in_u8"])
    bd = frames_to_unlabeled_batch(u8, resize_dims=size, bbox=rows)
    np.testing.assert_allclose(bd["frames"].cpu().numpy(), want, atol=1e-5, rtol=1e-4)
    np.testing.assert_array_equal(bd["bbox"].cpu().numpy(), want_boxes)
    assert bd["is_multiview"] is False and bd["transforms"].tolist() == [-1.0]
    # bf16 outputs, FCHW and FHWC
    fchw, b1 = ops.frames_crop_normalize(u8, rows, size, dtype=torch.bfloat16)
    fhwc, b2 = ops.frames_crop_normalize(u8, rows, size, dtype=torch.bfloat16, channels_last=True)
    np.testing.assert_allclose(fchw.float().cpu().numpy(), want, atol=1e-2, rtol=1e-2)
    np.testing.assert_allclose(fhwc.float().permute(0, 3, 1, 2).cpu().numpy(), want, atol=1e-2, rtol=1e-2)
    assert torch.equal(b1, b2) and torch.equal(b1.cpu(), torch.from_numpy(want_boxes))
    # two runs are bit-identical
    again, again_boxes = ops.frames_crop_normalize(u8, rows, size)
    assert torch.equal(again, bd["frames"]) and torch.equal(again_boxes, bd["bbox"])


def test_row_cursor_and_last_row_padding():
    """N = 10 rows read in chunks of 4: rows 0-3, 4-7, then 8, 9, 9, 9 (the reference pads with the final row)."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch

    rows = torch.tensor([[i, 2 * i, 5 + i, 7 + i] for i in range(10)], dtype=torch.float32, device=DEV)
    frames = torch.randint(0, 256, (4, 40, 40, 3), dtype=torch.uint8, device=DEV)
    cursor = torch.zeros(1, dtype=torch.int64, device=DEV)
    want = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 9, 9]]
    for chunk in want:
        _, boxes = ops.frames_crop_normalize(frames, rows, (16, 16), cursor=cursor)
        assert torch.equal(boxes, rows[chunk]), (chunk, boxes)
        cursor += 4
    for r0, chunk in zip((0, 4, 8), want):
        assert torch.equal(frames_to_unlabeled_batch(frames, resize_dims=(16, 16), bbox=rows, bbox_row0=r0)["bbox"], rows[chunk])


def test_cases_the_reference_rejects_do_not_fault():
    """An origin past the far edge is a one-pixel crop at the last pixel; a NaN (or inf) row is the whole frame."""
    from lightning_pose_b200 import ops

    h, w = 30, 44
    frames = torch.randint(0, 256, (5, h, w, 3), dtype=torch.uint8, device=DEV)
    rows = torch.tensor([[50.0, 3.0, 10.0, 10.0], [5.0, 31.0, 10.0, 10.0], [1e12, -1e12, 5.0, 5.0],
                         [float("nan"), 2.0, 3.0, 4.0], [1.0, 2.0, float("inf"), 4.0]], device=DEV)
    out, boxes = ops.frames_crop_normalize(frames, rows, (8, 12))
    torch.cuda.synchronize()
    assert boxes.tolist() == [[w - 1, 3, 10, 1], [5, h - 1, 1, 10], [w - 1, 0, 1, 1], [0, 0, h, w], [0, 0, h, w]]
    full = ops.frames_normalize(frames, size=(8, 12))
    np.testing.assert_allclose(out[3:].cpu().numpy(), full[3:].cpu().numpy(), atol=1e-5, rtol=1e-4)
    px = ops.frames_normalize(frames[:1, 3:13, w - 1 :].contiguous(), size=(8, 12))  # the last column, resized
    np.testing.assert_allclose(out[:1].cpu().numpy(), px.cpu().numpy(), atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("name", [c[0] for c in O.BBOX_CASES])
def test_compute_bboxes_matches_golden_exactly(golden, name):
    from lightning_pose_b200.utils.cropzoom import compute_bboxes

    g = golden("cropzoom")
    tab = t(g[f"bbox_{name}_in_table"])
    ratio, (ch, cw) = float(g[f"bbox_{name}_in_ratio"]), [int(v) for v in g[f"bbox_{name}_in_hw"]]
    kw = {"crop_ratio": ratio} if ratio > 0 else {"crop_height": ch, "crop_width": cw}
    anchors = [int(a) for a in g[f"bbox_{name}_in_anchors"]]
    want = torch.from_numpy(g[f"bbox_{name}_out"]).float()
    from_table = compute_bboxes(tab, anchors, **kw)  # the (N, 3K) prediction table, read in place
    kp = tab.reshape(tab.shape[0], -1, 3)[:, :, :2].contiguous()
    from_kp = compute_bboxes(kp, anchors, **kw)
    assert torch.equal(from_table.cpu(), want) and torch.equal(from_kp.cpu(), want)
    assert torch.equal(compute_bboxes(tab, anchors, **kw), from_table)  # bit-identical rerun


def test_compute_bboxes_nan_anchor_gives_nan_row():
    from lightning_pose_b200.utils.cropzoom import compute_bboxes

    kp = torch.rand(3, 4, 2, device=DEV) * 100
    kp[1, 2, 0] = float("nan")
    out = compute_bboxes(kp, crop_ratio=1.5)
    assert torch.isnan(out[1]).all() and torch.isfinite(out[[0, 2]]).all()
    assert torch.isfinite(compute_bboxes(kp, [0, 1], crop_ratio=1.5)).all()  # the NaN keypoint is not an anchor


@pytest.mark.parametrize("name", [c[0] for c in O.SMOOTH_CASES])
def test_smooth_bboxes_matches_golden_exactly(golden, name):
    from lightning_pose_b200.utils.cropzoom import smooth_bboxes

    g = golden("cropzoom")
    boxes = t(g[f"smooth_{name}_in_boxes"].astype(np.float32))
    window = int(g[f"smooth_{name}_in_window"])
    out = smooth_bboxes(boxes, window=window)
    assert torch.equal(out.cpu(), torch.from_numpy(g[f"smooth_{name}_out"]).float())
    assert torch.equal(smooth_bboxes(boxes, window=window), out)


def test_smooth_bboxes_skips_nan():
    import pandas as pd

    from lightning_pose_b200.utils.cropzoom import smooth_bboxes

    b = np.array([[1, 5, 0, 2], [2, np.nan, 0, 3], [np.nan, np.nan, 0, 4], [4, np.nan, 0, 6], [3, np.nan, 1, 1],
                  [np.nan, np.nan, 1, 1]], np.float32)
    for window in (1, 2, 4, 5):
        want = pd.DataFrame(b.astype(np.float64)).rolling(window=window, center=True, min_periods=1).median().round(0).to_numpy()
        np.testing.assert_array_equal(smooth_bboxes(t(b), window=window).cpu().numpy(), want.astype(np.float32))


def _crop_predictor_setup():
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(11)
    k, c, img = 7, 512, 128
    head = HeatmapHead("resnet50", c, k)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    head = head.to(DEV).eval()
    channel, scale = torch.arange(c, device=DEV) % 3, torch.randn(c, device=DEV)[None, :, None, None]

    def features_of(frames):  # a stand-in backbone of elementwise ops only: (T, 3, 128, 128) -> (T, 512, 4, 4)
        return (F.avg_pool2d(frames.float(), 32)[:, channel] * scale).contiguous()

    return head, k, img, features_of


def test_batched_predictor_crop_mode_graph_equals_eager_and_composition():
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.bboxes import crop_and_resize_frames
    from lightning_pose_b200.utils.cropzoom import compute_bboxes, smooth_bboxes
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head, k, img, features_of = _crop_predictor_setup()
    n, chunk, fh, fw = 22, 8, 240, 320
    gen = torch.Generator(device=DEV).manual_seed(5)
    video = torch.randint(0, 256, (n, fh, fw, 3), dtype=torch.uint8, device=DEV, generator=gen)
    detector = torch.rand(n, 5, 2, device=DEV, generator=gen) * torch.tensor([fw, fh], device=DEV) * 0.6 + 20
    boxes = smooth_bboxes(compute_bboxes(detector, crop_ratio=1.3), window=5)
    pad = (-n) % chunk
    padded = torch.cat([video, video[-1:].repeat(pad, 1, 1, 1)])
    tables = {}
    for use_graph in (True, False):
        bp = BatchedPredictor(head, k, n, chunk, (img, img), features_of=features_of, use_graph=use_graph, bboxes=boxes, frame_hw=(fh, fw))
        bp.run(padded[i : i + chunk] for i in range(0, n + pad, chunk))
        torch.cuda.synchronize()
        assert int(bp.cursor) == n + pad
        tables[use_graph] = bp.table.clone()
        if use_graph:
            assert bp.launches_per_chunk is not None and bp.launches_per_chunk >= 4
    assert torch.equal(tables[True], tables[False])
    # the eager composition: normalise -> crop_and_resize_frames -> head -> decode -> remap with the clamped boxes
    rows = torch.cat([boxes, boxes[-1:].repeat(pad, 1)])
    kps, cfs = [], []
    with torch.no_grad():
        for i in range(0, n + pad, chunk):
            full = ops.frames_normalize(padded[i : i + chunk])
            crops, clamped = crop_and_resize_frames(full, rows[i : i + chunk], [img, img])
            kp, cf = head.run_subpixelmaxima(head(features_of(crops)))
            kps.append(ops.remap_keypoints(kp, None, clamped, img, img))
            cfs.append(cf)
    kp, cf = torch.cat(kps)[:n], torch.cat(cfs)[:n]
    got = tables[False].reshape(n, k, 3)
    np.testing.assert_allclose(got[:, :, :2].reshape(n, 2 * k).cpu().numpy(), kp.cpu().numpy(), rtol=1e-4, atol=2e-2)
    np.testing.assert_allclose(got[:, :, 2].cpu().numpy(), cf.cpu().numpy(), rtol=1e-3, atol=1e-4)


def test_batched_predictor_crop_mode_adds_one_launch():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head, k, img, features_of = _crop_predictor_setup()
    n, chunk = 8, 8
    video = torch.randint(0, 256, (n, 200, 200, 3), dtype=torch.uint8, device=DEV)
    boxes = torch.tensor([[10.0, 20.0, 150.0, 150.0]], device=DEV).repeat(n, 1)
    crop = BatchedPredictor(head, k, n, chunk, (img, img), features_of=features_of, bboxes=boxes, frame_hw=(200, 200))
    crop.feed(video)
    plain = BatchedPredictor(head, k, n, chunk, (img, img), features_of=features_of)  # model-size frames streamed in
    plain.feed(torch.randn(n, 3, img, img, device=DEV))
    assert crop.launches_per_chunk == plain.launches_per_chunk + 1, (crop.launches_per_chunk, plain.launches_per_chunk)
    with pytest.raises(ValueError, match="uint8"):
        crop.feed(video.float())
