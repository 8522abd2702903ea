"""GPU: FramePredictor.push_frame, a live stream of one frame per call through a context (MHCRNN) model, against the
composition of the existing parts on frames t - 4 .. t, against predict_frame on the five-frame stack, against the
float64 head and decode, and the stream's state across pushes, resets, predict_frame calls and new input forms."""
import numpy as np
import pytest
import torch

import scale_oracle as S
from test_context_train_gpu import head_tensors
from test_predict_frame_gpu import DEV, IMG, K, _ingest, assert_same, context_tracker, frames

pytestmark = pytest.mark.gpu
F64 = torch.float64
N = 12
SHAPE = (140, 170, 3)


def clip(seed, shape=SHAPE, n=N):
    return frames((n, *shape), seed)


def boxes(mode, n=N, seed=0):
    """Per-frame (x, y, w, h) boxes: none, one fixed box, or a different box for every frame (some past the far edges,
    which clip)."""
    if mode == "none":
        return [None] * n
    if mode == "fixed":
        return [(9, 13, 120, 100)] * n
    rng = np.random.default_rng(seed)
    return [tuple(int(v) for v in (rng.integers(0, 40), rng.integers(0, 30), rng.integers(60, 150), rng.integers(60, 130)))
            for _ in range(n)]


def stream_predictor(tr, **kw):
    from lightning_pose_b200.utils.predictions import FramePredictor

    return FramePredictor(tr.head, K, (IMG, IMG), features_of=kw.pop("features_of", tr.backbone), **kw)


def push_all(fp, video, bxs, device=False):
    out = []
    for f, b in zip(video, bxs):
        out.append(fp.push_frame(torch.from_numpy(f).to(DEV) if device else f, bbox=b))
    return out


def composed(tr, video, bxs, t):
    """Frame t - 2 of the stream from existing parts: each frame of t - 4 .. t ingested with its own box and through the
    backbone alone; HeatmapTrackerMHCRNN.forward's head call on the (1, 5, 3, h, w) form; both decodes; the strict-greater
    selection; remap_keypoints with frame t - 2's box."""
    from lightning_pose_b200 import ops

    ins = [_ingest(video[i][None], bxs[i], (IMG, IMG)) for i in range(t - 4, t + 1)]
    with torch.no_grad():
        feats = torch.cat([tr.backbone(x) for x, _ in ins])
        reps = torch.permute(feats.reshape(1, 5, *feats.shape[1:]), (0, 2, 3, 4, 1))
        sf, mf = tr.head(reps, (1, 5, 3, IMG, IMG), False)
        kp_sf, cf_sf = tr.head.run_subpixelmaxima(sf)
        kp_mf, cf_mf = tr.head.run_subpixelmaxima(mf)
        pick = torch.gt(cf_mf, cf_sf)
        kp = torch.where(pick[..., None], kp_mf.reshape(1, K, 2), kp_sf.reshape(1, K, 2)).reshape(1, 2 * K)
        cf = torch.where(pick, cf_mf, cf_sf)
        kp = ops.remap_keypoints(kp, None, ins[2][1], IMG, IMG)
    return {"keypoints": kp.reshape(K, 2).cpu().numpy(), "confidence": cf[0].cpu().numpy()}


def assert_stream(results, tr, video, bxs, what=""):
    for t, r in enumerate(results):
        if t < 4:
            assert r == {"keypoints": None, "confidence": None, "frame": None}, (what, t)
            continue
        assert r["frame"] == t - 2 and r["keypoints"].shape == (K, 2) and r["keypoints"].dtype == np.float32
        assert_same(r, composed(tr, video, bxs, t), f"{what} t={t}")


# ------------------------------------------------------------------------------------------------
# results
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["none", "fixed", "per_frame"])
def test_push_equals_composition(mode):
    tr = context_tracker()
    video, bxs = clip(1), boxes(mode, seed=3)
    fp = stream_predictor(tr)
    assert_stream(push_all(fp, video, bxs), tr, video, bxs, mode)
    assert fp.launches_per_push is not None and fp.launches_per_push >= 8


def test_push_against_predict_frame():
    """With one box for the stream, push t equals predict_frame on frames t - 4 .. t.  Bit for bit when the stand-in
    backbone gives a frame the same features alone and in a batch of five; otherwise within 0.05 model pixels on the
    planes whose confidence is above 0.5.  On the H100 the bf16 stand-in's features agreed bit for bit."""
    tr = context_tracker()
    video, box = clip(2), (9, 13, 120, 100)
    stream, single = stream_predictor(tr), stream_predictor(tr)
    x, _ = _ingest(video[:5], box, (IMG, IMG))
    with torch.no_grad():
        batch_free = torch.equal(tr.backbone(x), torch.cat([tr.backbone(x[i : i + 1]) for i in range(5)]))
    for t, r in enumerate(push_all(stream, video, [box] * N)):
        if t < 4:
            continue
        want = single.predict_frame(video[t - 4 : t + 1], bbox=box)
        if batch_free:
            assert_same(r, want, f"t={t}")
        else:
            confident = want["confidence"] > 0.5
            d = (np.abs(r["keypoints"] - want["keypoints"]) * IMG / np.array([box[2], box[3]])).max(-1)
            assert (d[confident] < 0.05).all(), (t, d, confident)


def test_push_keypoints_against_float64():
    """The single-frame and context heads and both decodes in float64 on the features the stream's backbone made for
    frames t - 4 .. t, the float64 selection and remap: keypoints within 0.05 model pixels (test_predict_frame's bar for
    bf16 features) on the planes whose selected confidence is above 0.5 and whose two confidences are more than 1e-3
    apart (so that both sides select the same head).  The stand-in's features are scaled by 3: at scale 1 its heatmaps
    on random frames are flat (confidences near 0.002), at 3 both heads have confident planes."""
    tr = context_tracker()

    def features_of(x):
        return (tr.backbone(x).float() * 3.0).to(torch.bfloat16)

    video, bxs = clip(4), boxes("per_frame", seed=5)
    res = push_all(stream_predictor(tr, features_of=features_of), video, bxs)
    ws, bs, p = head_tensors(tr.head)
    ds, uf = tr.head.downsample_factor, tr.head.head_mf.upsampling_factor
    idx = torch.arange(5, device=DEV, dtype=torch.int32)[None]
    checked = 0
    for t in range(4, N):
        ins = [_ingest(video[i][None], bxs[i], (IMG, IMG)) for i in range(t - 4, t + 1)]
        with torch.no_grad():
            feats = torch.cat([features_of(x) for x, _ in ins])
        f64 = feats.to(F64)  # bf16 values: the references' operand rounding leaves them as they are
        sf = S.head_ref_chunked(f64[2:3], ws, bs, softmax=True, operands=feats.dtype)
        mf, _, _ = S.context_ref(f64, p, uf, idx, operands=feats.dtype)
        kp_sf, cf_sf, _, _ = S.decode_ref(sf, ds)
        kp_mf, cf_mf, _, _ = S.decode_ref(mf.detach(), ds)
        pick = (cf_mf > cf_sf)[0]
        kp = torch.where(pick[:, None], kp_mf.reshape(K, 2), kp_sf.reshape(K, 2))
        cf = torch.where(pick, cf_mf[0], cf_sf[0])
        bb = ins[2][1].to(F64)[0]
        scale = torch.stack([bb[3] / IMG, bb[2] / IMG])
        want = (kp * scale + bb[:2]).cpu().numpy()
        d = (np.abs(res[t]["keypoints"] - want) / scale.cpu().numpy()).max(-1)
        keep = ((cf > 0.5) & ((cf_mf[0] - cf_sf[0]).abs() > 1e-3)).cpu().numpy()
        assert (d[keep] < 0.05).all(), (t, d, keep)
        checked += int(keep.sum())
    assert checked >= N


def test_one_backbone_pass_per_push_and_every_form_same_bits():
    """Eager: features_of sees one call with one frame per push.  Graph and eager, host and device frames: same bits."""
    tr = context_tracker()
    video, bxs = clip(6), boxes("per_frame", seed=7)
    seen = []

    def counting(x):
        seen.append(tuple(x.shape))
        return tr.backbone(x)

    eager = stream_predictor(tr, features_of=counting, use_graph=False)
    ref = []
    for t, (f, b) in enumerate(zip(video, bxs)):
        ref.append(eager.push_frame(f, bbox=b))
        assert seen == [(1, 3, IMG, IMG)] * (t + 1), seen
    runs = {"graph host": push_all(stream_predictor(tr), video, bxs),
            "graph device": push_all(stream_predictor(tr), video, bxs, device=True),
            "eager device": push_all(stream_predictor(tr, use_graph=False), video, bxs, device=True)}
    for what, got in runs.items():
        for t in range(4, N):
            assert got[t]["frame"] == ref[t]["frame"], (what, t)
            assert_same(got[t], ref[t], f"{what} t={t}")


# ------------------------------------------------------------------------------------------------
# the stream's state
# ------------------------------------------------------------------------------------------------
def test_reset_restarts_the_stream():
    tr = context_tracker()
    video, bxs = clip(8), boxes("per_frame", seed=9)
    fp = stream_predictor(tr)
    first = push_all(fp, video[:9], bxs[:9])
    fp.reset_stream()
    again = push_all(fp, video[:9], bxs[:9])
    fp.reset_stream()
    other = push_all(fp, video[3:], bxs[3:])  # a new stream starting at a different frame: the old ring is not read
    for t in range(4, 9):
        assert again[t]["frame"] == t - 2
        assert_same(again[t], first[t], f"t={t}")
    assert_stream(other, tr, video[3:], bxs[3:], "after reset")


def test_predict_frame_calls_between_pushes_change_nothing():
    tr = context_tracker()
    video, bxs = clip(10), boxes("per_frame", seed=11)
    alone = push_all(stream_predictor(tr), video, bxs)
    fp = stream_predictor(tr)
    stacks = clip(12, shape=(97, 211, 3), n=5)
    mixed = []
    for t, (f, b) in enumerate(zip(video, bxs)):
        if t % 3 == 1:
            fp.predict_frame(stacks, bbox=(5, 5, 90, 90))
        mixed.append(fp.push_frame(f, bbox=b))
        if t % 3 == 2:
            fp.predict_frame(torch.from_numpy(video[:5]).to(DEV))
    for t in range(4, N):
        assert_same(mixed[t], alone[t], f"t={t}")


def test_new_frame_shape_and_source_keep_the_stream():
    """A frame shape or source (host / device) change recaptures the push graph; the ring carries over."""
    tr = context_tracker()
    a, b = clip(13), clip(14, shape=(97, 211, 3))
    video = [a[0], a[1], a[2], b[3], b[4], b[5], a[6], a[7], b[8], b[9], a[10], a[11]]
    bxs = boxes("per_frame", seed=15)  # origins inside both shapes
    fp = stream_predictor(tr)
    res, graphs = [], []
    for t, (f, box) in enumerate(zip(video, bxs)):
        res.append(fp.push_frame(torch.from_numpy(f).to(DEV) if t in (6, 7) else f, bbox=box))
        graphs.append(fp._push_graph)
    assert graphs[3] is not graphs[2] and graphs[6] is not graphs[5] and graphs[8] is not graphs[7]
    assert graphs[4] is graphs[3] and graphs[7] is graphs[6]
    assert_stream(res, tr, video, bxs, "mixed shapes")


def test_steady_state_pushes_allocate_nothing():
    tr = context_tracker()
    video, bxs = clip(16), boxes("per_frame", seed=17)
    fp = stream_predictor(tr)
    push_all(fp, video, bxs)
    torch.cuda.synchronize()
    before = torch.cuda.memory_stats(DEV)["allocation.all.allocated"]
    for i in range(100):
        fp.push_frame(video[i % N], bbox=bxs[i % N])
    assert torch.cuda.memory_stats(DEV)["allocation.all.allocated"] == before
