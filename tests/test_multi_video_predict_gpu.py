"""GPU: BatchedPredictor over a list of videos.  Each video's rows of the list table equal, bit for bit, the table a
one-video predictor gives that video alone, fed in chunks of T with the last one padded.  Features are streamed, or the
stand-in backbone computes every frame on its own, so a frame's prediction does not depend on which chunk holds it.

The list (T = 12): a video shorter than a chunk, one that ends on a chunk boundary, two 5-frame videos inside one
chunk, and for context models (S = 16) videos with R < N - 1, R >= N and R = N - 1, the last of them spanning three
chunks."""
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
K, T = 17, 12
LENGTHS = [7, 17, 5, 5, 28, 30, 13, 25]
ENDS_ON_BOUNDARY = [11, 13]  # a context list that ends on a chunk boundary after an R = N - 1 video: one more chunk


def chunks(video, lo, hi, n_chunks, pad):
    """Frames [lo, hi) of ``video`` (a tensor, a tuple of tensors or a list of views, leading frame axis) in
    ``n_chunks`` chunks of T: past the video, ``pad`` (one item per part; None repeats the part's last frame)."""
    parts = list(video) if isinstance(video, (tuple, list)) else [video]
    pads = list(pad) if isinstance(pad, (tuple, list)) else [pad] * len(parts)
    out = []
    for x, p in zip(parts, pads):
        x = x[lo : min(hi, x.shape[0])]
        fill = x[-1:] if p is None else p[None]
        out.append(torch.cat([x, fill.expand(n_chunks * T - x.shape[0], *x.shape[1:])]))
    items = [[x[i : i + T] for x in out] for i in range(0, n_chunks * T, T)]
    if isinstance(video, list):
        return items
    return [tuple(it) if isinstance(video, tuple) else it[0] for it in items]


def split(video, lengths):
    """The per-video slices of a concatenated stream (every part of a tuple / list)."""
    starts = [sum(lengths[:i]) for i in range(len(lengths) + 1)]
    if isinstance(video, (tuple, list)):
        per = [split(x, lengths) for x in video]
        return [type(video)(p[i] for p in per) for i in range(len(lengths))]
    return [video[a:b] for a, b in zip(starts, starts[1:])]


def run(make, n, video, pad):
    bp = make(n)
    bp.run(chunks(video, *bp.feed_range, bp.n_chunks, pad))
    return bp


def assert_list_equals_one_video_tables(make, video, lengths, pad):
    """make(n_frames, video index or None for the list) -> BatchedPredictor.  Returns the list predictor."""
    lst = run(lambda n: make(n, None), lengths, video, pad)
    torch.cuda.synchronize()
    for i, (n, part, got) in enumerate(zip(lengths, split(video, lengths), lst.video_tables())):
        one = run(lambda m: make(m, i), n, part, pad)
        torch.cuda.synchronize()
        assert got.shape == one.table.shape
        bad = (got != one.table).any(1).nonzero().flatten().tolist()
        assert not bad, f"video {i} (N = {n}): rows {bad} differ"
    return lst


def frame_head(seed):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead("resnet50", 512, K)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return head.to(DEV).eval()


def conv_tracker(seed):
    """A heatmap tracker whose stand-in backbone is one stride-32 convolution: every frame on its own."""
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    torch.manual_seed(seed)
    model = HeatmapTracker(K, backbone=torch.nn.Conv2d(3, 512, 32, stride=32), num_fc_input_features=512)
    for layer in list(model.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return model.to(DEV).eval()


def context_head(seed):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    torch.manual_seed(seed)
    return HeatmapMHCRNNHead("vits_dino", 384, K, upsampling_factor=1).to(DEV).eval()


def feature_video(n, seed, c=512, hw=4, dtype=torch.bfloat16):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    feats = (torch.randn(n, c, hw, hw, device=DEV, generator=gen) * 0.5).to(dtype)
    boxes = torch.cat([torch.rand(n, 2, device=DEV, generator=gen) * 30, 200 + torch.rand(n, 2, device=DEV, generator=gen) * 200], 1)
    return feats, boxes


def test_list_shape_cases():
    from lightning_pose_b200.utils.predictions import _context_rows

    starts = [sum(LENGTHS[:i]) for i in range(len(LENGTHS) + 1)]
    assert LENGTHS[0] < T and starts[2] % T == 0  # shorter than a chunk; the second ends on a chunk boundary
    assert LENGTHS[2:4] == [5, 5] and starts[2] // T == (starts[4] - 1) // T  # two 5-frame videos inside one chunk
    rows = [(_context_rows(n, T), n) for n in LENGTHS]
    assert any(r >= n for r, n in rows) and any(r < n - 1 for r, n in rows) and any(r == n - 1 for r, n in rows)
    last = LENGTHS[-1]
    assert (starts[-1] - 1) // T - starts[-2] // T + 1 == 3 and _context_rows(last, T) == last - 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_frame_model_list(dtype):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = frame_head(3)
    feats, boxes = feature_video(sum(LENGTHS), 5, dtype=dtype)
    pad = (torch.zeros_like(feats[0]), None)
    lst = assert_list_equals_one_video_tables(lambda n, i: BatchedPredictor(head, K, n, T, (128, 128)), (feats, boxes), LENGTHS, pad)
    one = BatchedPredictor(head, K, 30, T, (128, 128))
    one.run(chunks((feats, boxes), 0, 30, 3, pad))
    assert lst.launches_per_chunk == one.launches_per_chunk


def test_regression_model_list():
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    torch.manual_seed(2)
    head = LinearRegressionHead(128, 2 * K).to(DEV).eval()
    feats, _ = feature_video(sum(LENGTHS), 6, c=128)
    assert_list_equals_one_video_tables(lambda n, i: BatchedPredictor(head, K, n, T, (64, 64)), feats, LENGTHS, None)


def test_multiview_uint8_view_list():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    model = conv_tracker(7)
    gen = torch.Generator(device=DEV).manual_seed(8)
    vids = [torch.randint(0, 256, (sum(LENGTHS), h, w, 3), dtype=torch.uint8, device=DEV, generator=gen)
            for h, w in ((150, 200), (97, 131))]
    make = lambda n, i: BatchedPredictor(model.head, K, n, T, (128, 128), features_of=model.get_representations, num_views=2)
    lst = assert_list_equals_one_video_tables(make, vids, LENGTHS, [None, None])
    assert [tuple(t.shape) for t in lst.video_tables()] == [(n, 6 * K) for n in LENGTHS]


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
def test_crop_mode_list(use_graph):
    """Every video's boxes in one (sum N, 4) table; rows past the list's end repeat its last row, as for one video."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    model = conv_tracker(9)
    side, n = 160, sum(LENGTHS)
    gen = torch.Generator(device=DEV).manual_seed(10)
    frames = torch.randint(0, 256, (n, side, side, 3), dtype=torch.uint8, device=DEV, generator=gen)
    wh = torch.randint(40, 150, (n, 2), device=DEV, generator=gen).float()
    boxes = torch.cat([(torch.rand(n, 2, device=DEV, generator=gen) * (side - wh)).floor(), wh], 1).contiguous()
    rows = split(boxes, LENGTHS)  # a one-video predictor takes that video's own rows of the box table
    make = lambda n, i: BatchedPredictor(model.head, K, n, T, (128, 128), features_of=model.get_representations,
                                         use_graph=use_graph, bboxes=boxes if i is None else rows[i].contiguous(),
                                         frame_hw=(side, side))
    assert_list_equals_one_video_tables(make, frames, LENGTHS, None)
    with pytest.raises(ValueError, match="bboxes has 10 rows"):
        BatchedPredictor(model.head, K, [4, 7], T, (128, 128), features_of=model.get_representations, bboxes=boxes[:10],
                         frame_hw=(side, side))


@pytest.mark.parametrize("lengths", [LENGTHS, ENDS_ON_BOUNDARY], ids=["mixed", "ends_on_boundary"])
def test_context_model_list(lengths):
    """Graph replay, eager and sub-chunks: one capture for the whole list, the same table three times, and each video's
    rows equal to its one-video table padded with the pad feature."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = context_head(11)
    feats, boxes = feature_video(sum(lengths), 12, c=384, hw=16)
    pad = torch.zeros_like(feats[0])
    tables, launches = {}, {}
    for name, kw in (("graph", {}), ("eager", {"use_graph": False}), ("sub", {"sub_chunk": 5})):
        make = lambda n, i: BatchedPredictor(head, K, n, T, (256, 256), pad=pad if i is None else None, **kw)
        lst = assert_list_equals_one_video_tables(make, (feats, boxes), lengths, (pad, None)) if name == "graph" else \
            run(lambda n: make(n, None), lengths, (feats, boxes), (pad, None))
        torch.cuda.synchronize()
        tables[name], launches[name] = lst.table.clone(), lst.launches_per_chunk
    assert torch.equal(tables["graph"], tables["eager"]) and torch.equal(tables["graph"], tables["sub"])
    one = run(lambda n: BatchedPredictor(head, K, n, T, (256, 256)), 30, (feats[:30], boxes[:30]), (pad, None))
    assert launches["graph"] == one.launches_per_chunk and launches["eager"] is None


def test_context_list_needs_the_pad_feature():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = context_head(11)
    feats, boxes = feature_video(22, 13, c=384, hw=16)
    bp = BatchedPredictor(head, K, [9, 13], T, (256, 256))  # 13 frames at T = 12: R = 12 = N - 1
    with pytest.raises(ValueError, match="pass `pad`"):
        bp.feed(feats[:T], boxes[:T])
    assert int(bp.cursor) == 0 and float(bp.table.abs().sum()) == 0.0
    bp = BatchedPredictor(head, K, [9, 13], T, (256, 256), pad=torch.zeros(384, 16, 16, device=DEV))  # fp32 pad, bf16 chunk
    with pytest.raises(ValueError, match="pad must be one"):
        bp.feed(feats[:T], boxes[:T])
    BatchedPredictor(head, K, [30, 27], T, (256, 256)).feed(feats[:T], boxes[:T])  # no R = N - 1 video: no pad needed


def test_context_crop_mode_list():
    """uint8 frames cropped inside the chunk: the padding frame is a zero frame, for the list as for one video."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    torch.manual_seed(11)
    k, c, img, fh, fw = 7, 128, 64, 120, 160
    lengths = [13, 5, 5, 27, 25]
    n = sum(lengths)
    head = HeatmapMHCRNNHead("vits_dino", c, k, upsampling_factor=1)
    for prm in head.head_sf.parameters():
        torch.nn.init.normal_(prm, std=0.3)
    head = head.to(DEV).eval()
    channel, scale = torch.arange(c, device=DEV) % 3, torch.randn(c, device=DEV)[None, :, None, None]

    def features_of(frames):  # elementwise stand-in backbone: (T, 3, 64, 64) -> (T, 128, 4, 4)
        return (F.avg_pool2d(frames.float(), 16)[:, channel] * scale).contiguous()

    gen = torch.Generator(device=DEV).manual_seed(5)
    video = torch.randint(0, 256, (n, fh, fw, 3), dtype=torch.uint8, device=DEV, generator=gen)
    xy = torch.rand(n, 2, device=DEV, generator=gen) * 60
    boxes = torch.cat([xy.floor(), torch.full((n, 2), 50.0, device=DEV) + torch.arange(n, device=DEV)[:, None] % 40], 1)
    rows = split(boxes, lengths)
    zero = torch.zeros(fh, fw, 3, dtype=torch.uint8, device=DEV)
    make = lambda m, i: BatchedPredictor(head, k, m, T, (img, img), features_of=features_of,
                                         bboxes=boxes if i is None else rows[i].contiguous(), frame_hw=(fh, fw))
    assert_list_equals_one_video_tables(make, video, lengths, zero)


# ---- shards ---------------------------------------------------------------------------------------------------------
def joined_shards(make, video, lengths, world, pad):
    from lightning_pose_b200.utils.predictions import fill_context_edges

    whole = run(make, (0, 1), video, pad)
    joined = torch.full_like(whole.table, float("nan"))
    for rank in range(world):
        bp = make((rank, world))
        if bp.feed_range[0] < bp.feed_range[1]:
            bp.run(chunks(video, *bp.feed_range, bp.n_chunks, pad))
        a, b = bp.rows
        joined[a:b] = bp.table[a:b]
    if whole.context:
        fill_context_edges(joined, T, world, lengths)
    torch.cuda.synchronize()
    return whole.table, joined


@pytest.mark.parametrize("world", [2, 3, 8])
def test_context_list_shards(world):
    """World 8 puts a shard's first row on a video's first frame (row 34): its halo stays in that video."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor, shard_feed_range

    assert shard_feed_range(LENGTHS, T, 2, 8, context=True)[0] == 34
    head = context_head(14)
    feats, boxes = feature_video(sum(LENGTHS), 15, c=384, hw=16)
    pad = torch.zeros_like(feats[0])
    make = lambda shard: BatchedPredictor(head, K, LENGTHS, T, (256, 256), pad=pad, shard=shard)
    whole, joined = joined_shards(make, (feats, boxes), LENGTHS, world, (pad, None))
    bad = (joined != whole).any(1).nonzero().flatten().tolist()
    assert not bad, f"world {world}: rows {bad} differ"


@pytest.mark.parametrize("world", [2, 3, 8])
def test_frame_list_shards(world):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = frame_head(16)
    feats, boxes = feature_video(sum(LENGTHS), 17)
    make = lambda shard: BatchedPredictor(head, K, LENGTHS, T, (128, 128), shard=shard)
    whole, joined = joined_shards(make, (feats, boxes), LENGTHS, world, (torch.zeros_like(feats[0]), None))
    assert torch.equal(joined, whole)


GLOO_CONTEXT = [25, 7, 13, 5]  # world 2: rank 1's first row (25) is a video's first frame; 25 and 13 have R = N - 1


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gather_worker(rank, world, port, out):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        ok = {}
        head = context_head(18)
        ctx = feature_video(sum(GLOO_CONTEXT), 19, c=384, hw=16)
        pad = torch.zeros_like(ctx[0][0])
        fhead = frame_head(20)
        frames = feature_video(sum(LENGTHS), 21)
        for name, make, vid, vpad in (
                ("context", lambda s: BatchedPredictor(head, K, GLOO_CONTEXT, T, (256, 256), pad=pad, shard=s), ctx, (pad, None)),
                ("frames", lambda s: BatchedPredictor(fhead, K, LENGTHS, T, (128, 128), shard=s), frames, (None, None))):
            whole = run(make, (0, 1), vid, vpad)
            bp = make((rank, world))
            bp.run(chunks(vid, *bp.feed_range, bp.n_chunks, vpad))
            table = bp.gather()
            torch.cuda.synchronize()
            ok[name] = bool(torch.equal(table, whole.table))
        out[rank] = ok
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_list_gather_two_ranks_gloo():
    world = 2
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_gather_worker, args=(world, _free_port(), out), nprocs=world, join=True)
        assert dict(out) == {r: {"context": True, "frames": True} for r in range(world)}
