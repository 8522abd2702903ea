"""GPU: the single-frame ingest (lpb_frames_crop_resize_cv2) against OpenCV's own outputs (tests/golden/frame_resize.npz)
and the numpy restatement of its rule, and FramePredictor: graph replay against the eager body and against the
trackers' get_loss_inputs_labeled path, keypoints against the float64 head and decode, the context selection, and the
graph's state across calls."""
import numpy as np
import pytest
import torch

import frame_resize_oracle as O
import head_support as HS
import scale_oracle as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F64 = torch.float64
GOLDEN = np.load(__file__.rsplit("/", 1)[0] + "/golden/frame_resize.npz")
CASES = sorted(k[: -len("_frames")] for k in GOLDEN.files if k.endswith("_frames"))
K, IMG = 9, 128


def _ingest(frames, box, size, channels_last=False, dtype=torch.float32):
    from lightning_pose_b200 import ops

    b = None if box is None else torch.tensor(box, dtype=torch.int32, device=DEV)
    return ops.frames_crop_resize_cv2(torch.from_numpy(frames).to(DEV), size, b, channels_last=channels_last, dtype=dtype)


# ------------------------------------------------------------------------------------------------
# the ingest
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channels_last", [False, True], ids=["fchw", "channels_last"])
@pytest.mark.parametrize("case", CASES)
def test_ingest_equals_opencv_golden(case, channels_last):
    """Bit-identical to cv2.resize + numpy normalisation in fp32; bf16 / fp16 are that result rounded; the bbox row is
    [x, y, actual_h, actual_w]."""
    box = GOLDEN[f"{case}_box"]
    box = None if box[0] < 0 else tuple(int(v) for v in box)
    want = torch.from_numpy(GOLDEN[f"{case}_f32"]).to(DEV)
    if channels_last:
        want = want.permute(0, 2, 3, 1).contiguous()
    size = GOLDEN[f"{case}_u8"].shape[1:3]
    for dtype, cast in ((torch.float32, lambda t: t), (torch.bfloat16, torch.Tensor.bfloat16), (torch.float16, torch.Tensor.half)):
        out, bbox = _ingest(GOLDEN[f"{case}_frames"], box, size, channels_last, dtype)
        torch.cuda.synchronize()
        assert out.dtype == dtype and out.shape == want.shape
        assert torch.equal(out.view(torch.int16 if dtype != torch.float32 else torch.int32),
                           cast(want).view(torch.int16 if dtype != torch.float32 else torch.int32)), (case, dtype)
        assert bbox.cpu().numpy().tolist() == [GOLDEN[f"{case}_bbox"].tolist()], case


@pytest.mark.parametrize("src,dst", [((1024, 1280), (384, 384)), ((720, 1280), (384, 384)), ((406, 396), (256, 256)),
                                     ((1024, 1024), (512, 512)), ((37, 1000), (384, 384)), ((250, 250), (384, 384)),
                                     ((200, 300), (123, 77))])
def test_ingest_equals_oracle_at_production_sizes(src, dst):
    """Camera-frame sizes (1024 x 1280 -> 384 x 384 among them), an exact 2x downscale, upscales and an output that is
    not a multiple of 8, against the numpy rule that equals cv2 byte for byte."""
    frames = np.random.default_rng(src[0] + dst[1]).integers(0, 256, (1, *src, 3), dtype=np.uint8)
    _, want, _ = O.crop_resize_normalize(frames, None, *dst)
    out, _ = _ingest(frames, None, dst)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------------
# the models: a single-frame tracker and a context tracker on stand-in backbones
# ------------------------------------------------------------------------------------------------
class _Backbone(torch.nn.Module):
    """(n, 3, 128, 128) -> (n, C, 128 / stride, 128 / stride) in ``dtype``: one strided convolution, deterministic."""

    def __init__(self, c, stride, dtype):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, c, stride, stride=stride)
        self.dtype = dtype

    def forward(self, x):
        return (self.conv(x.float()) * 0.5).to(self.dtype)


def frame_tracker(dtype):
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    torch.manual_seed(3)
    tr = HeatmapTracker(K, backbone=_Backbone(512, 32, dtype), num_fc_input_features=512)
    tr.head = HS.make_head(512, (K, K), seed=4)
    return tr.to(DEV).eval()


def context_tracker():
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import HeatmapTrackerMHCRNN
    from test_context_train_gpu import make_context_head

    torch.manual_seed(5)
    tr = HeatmapTrackerMHCRNN(K, backbone=_Backbone(384, 16, torch.bfloat16), backbone_arch="vits_dino", num_fc_input_features=384)
    tr.head = make_context_head("vits_dino", 384, K, 1, seed=6)
    return tr.to(DEV).eval()


def predictor(tr, **kw):
    from lightning_pose_b200.utils.predictions import FramePredictor

    return FramePredictor(tr.head, K, (IMG, IMG), features_of=tr.backbone, **kw)


def frames(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def labeled_path(tr, frame, box):
    """The reference's predict_frame composed from existing parts: the ingest, then get_loss_inputs_labeled on the
    (1, 3, h, w) or (1, 5, 3, h, w) batch (which remaps to the frame), then for a context model the selection."""
    x, bbox = _ingest(frame if frame.ndim == 4 else frame[None], box, (IMG, IMG))
    images = x[None] if frame.ndim == 4 else x
    batch = {"images": images, "keypoints": torch.zeros(1, 2 * K, device=DEV), "bbox": bbox,
             "heatmaps": torch.zeros(1, K, 1, 1, device=DEV)}
    with torch.no_grad():
        res = tr.get_loss_inputs_labeled(batch)
    kp, cf = res["keypoints_pred"].reshape(-1, K, 2), res["confidences"]
    if frame.ndim == 4:
        pick = torch.gt(cf[1:], cf[:1])
        kp, cf = torch.where(pick[..., None], kp[1:], kp[:1]), torch.where(pick, cf[1:], cf[:1])
    return kp[0].cpu().numpy(), cf[0].cpu().numpy()


def assert_same(a, b, what=""):
    assert np.array_equal(a["keypoints"].view(np.uint32), b["keypoints"].view(np.uint32)), what
    assert np.array_equal(a["confidence"].view(np.uint32), b["confidence"].view(np.uint32)), what


# ------------------------------------------------------------------------------------------------
# predict_frame
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
def test_predict_frame_graph_eager_and_labeled_path(dtype):
    tr = frame_tracker(dtype)
    graph, eager = predictor(tr), predictor(tr, use_graph=False)
    frame = frames((150, 190, 3), 1)
    for box in (None, (20, 11, 97, 120), (150, 100, 80, 80)):
        g = graph.predict_frame(frame, bbox=box)
        assert g["keypoints"].shape == (K, 2) and g["confidence"].shape == (K,) and g["keypoints"].dtype == np.float32
        assert_same(g, eager.predict_frame(frame, bbox=box), f"eager {box}")
        assert_same(g, graph.predict_frame(torch.from_numpy(frame).to(DEV), bbox=box), f"device frame {box}")
        kp, cf = labeled_path(tr, frame, box)
        assert_same(g, {"keypoints": kp, "confidence": cf}, f"labeled path {box}")
    assert graph.launches_per_call is not None and graph.launches_per_call >= 4


def test_predict_frame_context_graph_eager_and_labeled_path():
    tr = context_tracker()
    graph, eager = predictor(tr), predictor(tr, use_graph=False)
    clip = frames((5, 140, 170, 3), 2)
    for box in (None, (9, 13, 120, 100), (100, 90, 200, 200)):
        g = graph.predict_frame(clip, bbox=box)
        assert_same(g, eager.predict_frame(clip, bbox=box), f"eager {box}")
        kp, cf = labeled_path(tr, clip, box)
        assert_same(g, {"keypoints": kp, "confidence": cf}, f"labeled path {box}")
    assert graph.launches_per_call is not None


@pytest.mark.parametrize("dtype,bar", [(torch.bfloat16, 0.05), (torch.float16, 0.1), (torch.float32, 0.05)], ids=["bf16", "fp16", "fp32"])
def test_predict_frame_keypoints_against_float64(dtype, bar):
    """The head and decode in float64 on the features the predictor's backbone made: keypoints within ``bar`` model
    pixels on the planes the reference is confident in, after the float64 remap."""
    tr = frame_tracker(dtype)
    fp = predictor(tr)
    frame, box = frames((150, 190, 3), 3), (20, 11, 97, 120)
    got = fp.predict_frame(frame, bbox=box)
    x, bbox = _ingest(frame[None], box, (IMG, IMG))
    with torch.no_grad():
        feats = tr.backbone(x)
    ws, bs = HS.head_params(tr.head)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, operands=HS._operands(feats))
    kp_ref, cf_ref, _, _ = S.decode_ref(hm_ref, tr.head.downsample_factor)
    bb = bbox.to(F64)[0]
    scale = torch.stack([bb[3] / IMG, bb[2] / IMG]).cpu().numpy()
    frame_ref = kp_ref.reshape(K, 2).cpu().numpy() * scale + bb[:2].cpu().numpy()
    d = (np.abs(got["keypoints"] - frame_ref) / scale).max(-1)
    confident = cf_ref[0].cpu().numpy() > 0.5
    assert confident.any()
    assert (d[confident] < bar).all(), (d, confident)


def test_context_selection_rule_of_the_predictor_call():
    """lpb_pack_context_predictions as FramePredictor calls it (one frame, a five-row table, frame0 = 4, step 1): every
    row holds mf where conf_mf > conf_sf and sf otherwise, a NaN on either side keeping sf, remapped with the box."""
    from lightning_pose_b200 import ops

    k = 6
    kp_sf = torch.arange(2 * k, dtype=torch.float32, device=DEV)[None] * 3.0
    kp_mf = kp_sf + 100.0
    cf_sf = torch.tensor([[0.2, 0.9, float("nan"), 0.5, 0.4, float("nan")]], device=DEV)
    cf_mf = torch.tensor([[0.8, 0.1, 0.7, float("nan"), 0.4, float("nan")]], device=DEV)
    bbox = torch.tensor([[10.0, 20.0, 64.0, 32.0]], device=DEV)
    table = torch.full((5, 3 * k), -1.0, device=DEV)
    ops.pack_context_predictions(kp_sf, cf_sf, kp_mf, cf_mf, bbox, 128.0, 128.0, table, 1, frame0=4)
    mf = np.array([True, False, False, False, False, False])
    kp = np.where(mf[:, None], kp_mf.cpu().numpy().reshape(k, 2), kp_sf.cpu().numpy().reshape(k, 2))
    want = np.stack([kp[:, 0] * np.float32(1 / 128.0) * 32 + 10, kp[:, 1] * np.float32(1 / 128.0) * 64 + 20,
                     np.where(mf, cf_mf.cpu().numpy()[0], cf_sf.cpu().numpy()[0])], -1).astype(np.float32)
    for row in table.cpu().numpy().reshape(5, k, 3):
        np.testing.assert_array_equal(row, want)


# ------------------------------------------------------------------------------------------------
# the graph's state
# ------------------------------------------------------------------------------------------------
def test_consecutive_calls_shape_change_and_allocations():
    tr = frame_tracker(torch.bfloat16)
    fp, eager = predictor(tr), predictor(tr, use_graph=False)
    seq = [(frames((150, 190, 3), 10 + i), box) for i, box in enumerate([(3, 4, 50, 60), None, (100, 0, 400, 30), (0, 149, 1, 1)])]
    for frame, box in seq:  # each call sees its own frame and box: nothing stale in the staging buffers
        assert_same(fp.predict_frame(frame, bbox=box), eager.predict_frame(frame, bbox=box), str(box))
    first = fp._graph
    other = frames((97, 211, 3), 20)
    assert_same(fp.predict_frame(other, bbox=(5, 5, 90, 90)), eager.predict_frame(other, bbox=(5, 5, 90, 90)), "new shape")
    assert fp._graph is not first and fp._key == (True, (1, 97, 211, 3))
    assert_same(fp.predict_frame(*seq[0]), eager.predict_frame(*seq[0]), "back to the first shape")
    torch.cuda.synchronize()
    before = torch.cuda.memory_stats(DEV)["allocation.all.allocated"]
    for i in range(100):
        fp.predict_frame(seq[i % 4][0], bbox=seq[i % 4][1])
    assert torch.cuda.memory_stats(DEV)["allocation.all.allocated"] == before


def test_value_errors():
    tr, ctx = frame_tracker(torch.bfloat16), context_tracker()
    fp, fc = predictor(tr), predictor(ctx)
    frame = frames((60, 80, 3), 0)
    bad = [
        (fp, frame.astype(np.float32), None, "uint8"),
        (fp, torch.from_numpy(frame).to(DEV).float(), None, "uint8"),
        (fp, frame[..., :2], None, "shape"),
        (fp, frame[0], None, "shape"),
        (fp, np.zeros((0, 80, 3), np.uint8), None, "empty"),
        (fp, np.stack([frame] * 5), None, "single-frame model"),
        (fc, frame, None, "context model"),
        (fc, np.stack([frame] * 3), None, "5 frames"),
        (fp, frame, (-1, 0, 10, 10), "origin"),
        (fp, frame, (0, -3, 10, 10), "origin"),
        (fp, frame, (0, 0, 0, 10), "positive"),
        (fp, frame, (0, 0, 10, -2), "positive"),
        (fp, frame, (80, 0, 10, 10), "empty crop"),
        (fp, frame, (0, 60, 10, 10), "empty crop"),
        (fc, np.stack([frame] * 5), (0, 70, 10, 10), "empty crop"),
    ]
    for p, f, box, what in bad:
        with pytest.raises(ValueError):
            p.predict_frame(f, bbox=box)
        del what
