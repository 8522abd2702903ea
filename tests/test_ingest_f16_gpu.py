"""GPU: fp16 frame ingest and BatchedPredictor on fp16 features.

The ingest kernels compute each pixel in fp32 and round it once on the way out, so their fp16 output is the same call's
fp32 output .half() bit for bit, in every entry, layout and input type.  BatchedPredictor then runs all four chunk bodies
on fp16 (a stand-in backbone that keeps the frames' dtype, as autocast(float16) would): its graph replays equal eager
runs bit for bit, and its tables agree with the same predictor on fp32 features within the fp16 head's keypoint bar
(test_head_f16_gpu.py, 0.1 px)."""
import functools

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _u8(*shape, seed=1):
    return torch.randint(0, 256, shape, dtype=torch.uint8, device=DEV, generator=_gen(seed))


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("size", [(64, 96), (40, 52)])  # resized, as is
def test_normalize_f16_is_f32_half(channels_last, size):
    from lightning_pose_b200 import ops

    frames = _u8(3, 64, 96, 3)
    f32 = ops.frames_normalize(frames, size, channels_last=channels_last)
    f16 = ops.frames_normalize(frames, size, channels_last=channels_last, dtype=torch.float16)
    assert f16.dtype == torch.float16 and torch.equal(f16.view(torch.int16), f32.half().view(torch.int16))
    views = [_u8(3, 64, 96, 3, seed=2), _u8(3, 50, 70, 3, seed=3), _u8(3, *size, 3, seed=4)]
    v32 = ops.frames_normalize_views(views, size, channels_last=channels_last)
    v16 = ops.frames_normalize_views(views, size, channels_last=channels_last, dtype=torch.float16)
    assert torch.equal(v16.view(torch.int16), v32.half().view(torch.int16))


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("in_f32", [False, True])
def test_crop_f16_is_f32_half(channels_last, in_f32):
    from lightning_pose_b200 import ops

    frames = _u8(4, 80, 120, 3, seed=5)
    if in_f32:
        frames = ops.frames_normalize(frames)
    boxes = torch.tensor([[3.0, 5.0, 40.0, 60.0], [0.0, 0.0, 80.0, 120.0], [70.0, 10.0, 30.0, 30.0], [-5.0, 60.0, 100.0, 90.0]], device=DEV)
    a, ba = ops.frames_crop_normalize(frames, boxes, (48, 64), channels_last=channels_last)
    b, bb = ops.frames_crop_normalize(frames, boxes, (48, 64), channels_last=channels_last, dtype=torch.float16)
    assert torch.equal(b.view(torch.int16), a.half().view(torch.int16)) and torch.equal(ba, bb)


def test_augment_refuses_f16():
    from lightning_pose_b200 import ops

    params, seeds = ops.draw_dlc_params(1, DEV)
    with pytest.raises(ValueError, match="float32 or bfloat16"):
        ops.frames_augment_normalize(_u8(2, 32, 32, 3), (32, 32), params[0], seeds[:1], dtype=torch.float16)


# ---- BatchedPredictor ----------------------------------------------------------------------------------------------
K, C, IMG = 7, 512, 128


def _head(seed=11):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead("resnet50", C, K)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return head.to(DEV).eval().requires_grad_(False)


@functools.lru_cache(maxsize=None)
def _stand_in():
    """the stand-in backbone's constants, made once, before any graph capture"""
    return torch.arange(C, device=DEV) % 3, torch.randn(C, device=DEV, generator=_gen(12))[None, :, None, None]


def features_of(frames):
    """stand-in backbone of elementwise ops, in fp32, returning the frames' dtype: (T, 3, 128, 128) -> (T, 512, 4, 4)"""
    ch, scale = _stand_in()
    return (F.avg_pool2d(frames.float(), 32)[:, ch] * scale).to(frames.dtype).contiguous()


def _run(make, chunks):
    tables = {}
    for use_graph in (False, True):
        bp = make(use_graph)
        bp.run(chunks)
        torch.cuda.synchronize()
        tables[use_graph] = bp.table.clone()
    assert torch.equal(tables[True], tables[False])
    return tables[True]


def _agree(t16, t32, views=1):
    """fp16 and fp32 tables: every keypoint within 0.1 px, confidences within 1e-2.  The stand-in backbone's heatmaps are
    flat (no keypoint is confident), where the soft-argmax is most sensitive to the operands' rounding, so every keypoint
    is held to the bar the head's tests apply to confident ones."""
    a, b = t16.reshape(t16.shape[0], views * K, 3), t32.reshape(t32.shape[0], views * K, 3)
    d = (a[..., :2] - b[..., :2]).abs().amax(-1)
    assert float(d.max()) < 0.1, float(d.max())
    assert float((a[..., 2] - b[..., 2]).abs().max()) < 1e-2


def test_predictor_f16_frames_and_crop():
    """Single-frame (features streamed in) and crop (uint8 frames, crop_dtype=float16) chunks on fp16."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = _head()
    n, chunk = 24, 8
    frames = _u8(n, 200, 240, 3, seed=20)
    boxes = torch.tensor([[20.0, 30.0, 150.0, 170.0]], device=DEV).repeat(n, 1) + torch.arange(n, device=DEV)[:, None]
    tabs = {}
    for dtype in (torch.float16, torch.float32):
        x = ops.frames_normalize(frames, (IMG, IMG), dtype=dtype)
        feats = features_of(x)
        assert feats.dtype == dtype
        tabs["frames", dtype] = _run(lambda g: BatchedPredictor(head, K, n, chunk, (IMG, IMG), use_graph=g),
                                     [feats[i : i + chunk] for i in range(0, n, chunk)])
        tabs["crop", dtype] = _run(lambda g: BatchedPredictor(head, K, n, chunk, (IMG, IMG), features_of=features_of, use_graph=g, bboxes=boxes,
                                                              frame_hw=(200, 240), crop_dtype=dtype),
                                   [frames[i : i + chunk] for i in range(0, n, chunk)])
    for form in ("frames", "crop"):
        _agree(tabs[form, torch.float16], tabs[form, torch.float32])


def test_predictor_f16_views():
    """4-view uint8 chunks normalised to fp16 in one launch (crop_dtype=float16)."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head, v, n, chunk = _head(seed=13), 4, 16, 8
    views = [_u8(n, 120 + 8 * i, 160, 3, seed=30 + i) for i in range(v)]
    tabs = {}
    for dtype in (torch.float16, torch.float32):
        tabs[dtype] = _run(lambda g: BatchedPredictor(head, K, n, chunk, (IMG, IMG), features_of=features_of, use_graph=g, num_views=v, crop_dtype=dtype),
                           [[x[i : i + chunk] for x in views] for i in range(0, n, chunk)])
    assert tabs[torch.float16].shape == (n, 3 * K * v)
    _agree(tabs[torch.float16], tabs[torch.float32], views=v)


def test_predictor_f16_context():
    """Context (MHCRNN) chunks of fp16 features."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    torch.manual_seed(17)
    head = HeatmapMHCRNNHead("resnet50", C, K).to(DEV).eval().requires_grad_(False)
    for m in head.modules():
        if isinstance(m, torch.nn.ConvTranspose2d) and m.weight.shape[-1] == 3:
            torch.nn.init.xavier_uniform_(m.weight, gain=3.0)
    n, chunk = 21, 8
    frames = _u8(n + 3, 128, 128, 3, seed=40)  # padded to whole chunks
    tabs = {}
    for dtype in (torch.float16, torch.float32):
        from lightning_pose_b200 import ops

        feats = features_of(ops.frames_normalize(frames, dtype=dtype))
        tabs[dtype] = _run(lambda g: BatchedPredictor(head, K, n, chunk, (IMG, IMG), use_graph=g),
                           [feats[i : i + chunk] for i in range(0, n + 3, chunk)])
    _agree(tabs[torch.float16], tabs[torch.float32])
