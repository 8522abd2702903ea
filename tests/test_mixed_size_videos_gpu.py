"""GPU: a list of videos of several frame sizes through one BatchedPredictor (``frame_sizes``).

- The ragged ingest kernels, on a chunk holding a downscaled, an upscaled, an identity (copy path) and an odd-sized
  video plus the padding rows past the list's end, give every frame the bits of ``frames_normalize`` /
  ``frames_crop_normalize`` on that frame's own video alone, for every layout and output format.  The arena's slots
  and every output are first filled with 0x00, 0xFF and 0x7F (poison_support.py): bytes past a frame's end are never
  read and every output byte is written.
- Per body (frames on bf16, fp16 and fp32 features, context, regression, crop), graph replay and eager: each video's
  rows equal bit for bit the table of a one-video predictor fed that video alone through the uint8 form it has today
  (one uint8 view, or crop mode with frame_hw), padded with zero frames.  The first chunk holds one size only, so the
  capture happens before the other sizes appear; the graph is never captured again.
- Two shards over gloo on one GPU: ``gather()`` equals the one-GPU table."""
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from poison_support import PATTERNS, fill_storage, poisoned

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
K, T = 7, 12
# the first video fills the first chunk; 13 frames give R = N - 1 at T = 12, 5 frames R >= N, 28 frames R < N - 1
LENGTHS = [14, 5, 13, 7, 28, 25]
SIZES_64 = [(150, 170), (64, 64), (41, 77), (97, 131), (64, 64), (407, 395)]  # for 64 x 64 model images
SIZES_128 = [(200, 260), (128, 128), (61, 47), (407, 395), (128, 128), (150, 170)]  # for 128 x 128 model images


def make_videos(lengths, sizes, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=DEV, generator=gen) for n, (h, w) in zip(lengths, sizes)]


def fill_arena(arena, slot_bytes, frames, byte):
    """``frames`` (a list of (H, W, 3) uint8 tensors) into consecutive slots of an arena poisoned with ``byte``."""
    fill_storage(arena, byte)
    slots = arena.view(-1, slot_bytes)
    for f, x in enumerate(frames):
        slots[f, : x.numel()].copy_(x.reshape(-1))
    return arena


# ---- the kernels ------------------------------------------------------------------------------------------------------
OUT_HW = (96, 112)
KERNEL_SIZES = [(150, 200), (61, 47), OUT_HW, (407, 395)]  # downscale, upscale, identity, odd
KERNEL_LENGTHS = [3, 2, 4, 3]


def kernel_case(seed):
    from lightning_pose_b200 import ops

    videos = make_videos(KERNEL_LENGTHS, KERNEL_SIZES, seed)
    host = ops.ragged_videos(KERNEL_LENGTHS, KERNEL_SIZES)
    starts = [int(r) for r in host[:, 0]] + [sum(KERNEL_LENGTHS)]
    slot = ops.ragged_slot_bytes(KERNEL_SIZES)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    rows = []
    for n, (h, w) in zip(KERNEL_LENGTHS, KERNEL_SIZES):  # boxes partly outside the frame, and one non-finite row
        wh = torch.randint(8, max(h, w) + 20, (n, 2), device=DEV, generator=gen).float()
        xy = torch.randint(-10, max(h, w), (n, 2), device=DEV, generator=gen).float()
        rows.append(torch.cat([xy, wh], 1))
    rows[2][1, 0] = float("nan")
    return videos, host, starts, slot, rows


def frame_at(videos, starts, row):
    """(video, frame) of global row ``row``; rows past the end are zero frames of the last video."""
    v = max(i for i in range(len(videos)) if starts[i] <= row)
    a = row - starts[v]
    return v, (videos[v][a] if a < videos[v].shape[0] else torch.zeros_like(videos[v][0]))


@pytest.mark.parametrize("channels_last", [False, True], ids=["fchw", "fhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("crop", [False, True], ids=["normalize", "crop"])
def test_ragged_kernels_equal_the_one_size_kernels(channels_last, dtype, crop):
    from lightning_pose_b200 import ops

    videos, host, starts, slot, rows = kernel_case(1)
    boxes = torch.cat(rows).contiguous()
    table = host.to(DEV)
    n = sum(KERNEL_LENGTHS)
    for row0 in (0, 5):  # all four sizes from row 0; from row 5, seven padding rows past the list's end
        frames = [frame_at(videos, starts, row0 + f) for f in range(n)]
        arena = torch.empty(n * slot, dtype=torch.uint8, device=DEV)
        cursor = torch.tensor([row0], dtype=torch.int64, device=DEV)
        got = []
        for byte in PATTERNS:
            fill_arena(arena, slot, [x for _, x in frames], byte)
            with poisoned(byte):
                if crop:
                    out = ops.frames_crop_normalize_ragged(arena, slot, n, cursor, table, host, boxes, OUT_HW,
                                                           channels_last=channels_last, dtype=dtype)
                else:
                    out = ops.frames_normalize_ragged(arena, slot, n, cursor, table, host, OUT_HW, channels_last=channels_last,
                                                      dtype=dtype)
            got.append([t.clone() for t in out])
        for f, (v, x) in enumerate(frames):
            h, w = KERNEL_SIZES[v]
            if crop:  # the crop kernel on the frame's own video: its own box rows, at the frame's row in that video
                want, want_box = ops.frames_crop_normalize(x[None], rows[v], OUT_HW, row0=row0 + f - starts[v],
                                                           channels_last=channels_last, dtype=dtype)
            else:
                want = ops.frames_normalize(x[None], OUT_HW, channels_last=channels_last, dtype=dtype)
                want_box = torch.tensor([[0.0, 0.0, h, w]], device=DEV)
            for byte, (out, box) in zip(PATTERNS, got):
                assert torch.equal(out[f].view(torch.int16 if dtype != torch.float32 else torch.int32),
                                   want[0].view(torch.int16 if dtype != torch.float32 else torch.int32)), (row0, f, hex(byte))
                assert torch.equal(box[f], want_box[0]), (row0, f, hex(byte), box[f].tolist(), want_box[0].tolist())


def test_ragged_ingest_is_capturable():
    """One captured launch serves every cursor: replays at rows 0 and 5 give the eager results."""
    from lightning_pose_b200 import ops

    videos, host, starts, slot, _ = kernel_case(2)
    table, n = host.to(DEV), sum(KERNEL_LENGTHS)
    arena = torch.zeros(n * slot, dtype=torch.uint8, device=DEV)
    cursor = torch.zeros(1, dtype=torch.int64, device=DEV)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ops.frames_normalize_ragged(arena, slot, n, cursor, table, host, OUT_HW, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, boxes = ops.frames_normalize_ragged(arena, slot, n, cursor, table, host, OUT_HW, dtype=torch.bfloat16)
    for row0 in (0, 5):
        fill_arena(arena, slot, [frame_at(videos, starts, row0 + f)[1] for f in range(n)], 0x7F)
        cursor.fill_(row0)
        graph.replay()
        want = ops.frames_normalize_ragged(arena, slot, n, cursor, table, host, OUT_HW, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        assert torch.equal(out, want[0]) and torch.equal(boxes, want[1])


# ---- the predictor ----------------------------------------------------------------------------------------------------
def one_video_chunks(video, n_chunks):
    """A video's uint8 frames in chunks of T, padded with zero frames, each chunk one view."""
    pad = torch.zeros((n_chunks * T - video.shape[0], *video.shape[1:]), dtype=torch.uint8, device=DEV)
    x = torch.cat([video, pad])
    return [[x[i : i + T]] for i in range(0, n_chunks * T, T)]


def run_list(make, videos):
    from lightning_pose_b200.utils.predictions import segment_chunks

    bp = make([v.shape[0] for v in videos], [tuple(v.shape[1:3]) for v in videos], None)
    graph = None
    for chunk in segment_chunks(videos, T, bp.feed_range):
        bp.feed(chunk)
        graph = graph or bp._graph
        assert bp._graph is graph  # never captured again
    return bp


def assert_each_video_equals_its_one_video_table(make, videos):
    """make(lengths or N, sizes or None, video index or None) -> BatchedPredictor.  Returns the list predictor."""
    lst = run_list(make, videos)
    torch.cuda.synchronize()
    for i, (video, got) in enumerate(zip(videos, lst.video_tables())):
        one = make(video.shape[0], None, i)
        chunks = one_video_chunks(video, one.n_chunks)
        one.run([c[0] for c in chunks] if one.bboxes is not None else chunks)  # crop mode takes a tensor
        torch.cuda.synchronize()
        assert got.shape == one.table.shape
        bad = (got.view(torch.int32) != one.table.view(torch.int32)).any(1).nonzero().flatten().tolist()
        assert not bad, f"video {i} {tuple(video.shape[1:3])}: rows {bad} differ"
    return lst


def conv_features(seed, dtype):
    """A stride-32 convolution, every frame on its own: (T, 3, 128, 128) -> (T, 512, 4, 4) in ``dtype``."""
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(3, 512, 32, stride=32).to(DEV).eval()
    return lambda x: conv(x).to(dtype)


def pooled_features(seed, c=128):
    """An elementwise stand-in backbone: (T, 3, 64, 64) -> (T, c, 4, 4)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    channel, scale = torch.arange(c, device=DEV) % 3, torch.randn(c, device=DEV, generator=gen)[None, :, None, None]
    return lambda frames: (F.avg_pool2d(frames.float(), 16)[:, channel] * scale).contiguous()


def frame_head(seed, c=512):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead("resnet50", c, K)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    return head.to(DEV).eval()


def context_head(seed, c=128):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    torch.manual_seed(seed)
    head = HeatmapMHCRNNHead("vits_dino", c, K, upsampling_factor=1)
    for prm in head.head_sf.parameters():
        torch.nn.init.normal_(prm, std=0.3)
    return head.to(DEV).eval()


def sized(lengths, sizes, kw):
    """The list predictor takes frame_sizes; a one-video predictor (sizes None) takes its video's one uint8 view."""
    return dict(kw, frame_sizes=sizes) if sizes is not None else kw


GRAPH = pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])


@GRAPH
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
def test_frame_body(dtype, use_graph):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head, feats = frame_head(3), conv_features(4, dtype)
    videos = make_videos(LENGTHS, SIZES_128, 5)
    make = lambda n, sizes, i: BatchedPredictor(head, K, n, T, (128, 128), features_of=feats, use_graph=use_graph,
                                                **sized(n, sizes, {}))
    lst = assert_each_video_equals_its_one_video_table(make, videos)
    if use_graph:  # the launches of a same-size list predictor fed uint8 frames
        same = BatchedPredictor(head, K, [14, 10], T, (128, 128), features_of=feats)
        same.run(one_video_chunks(make_videos([24], [(200, 260)], 6)[0], 2))
        assert lst.launches_per_chunk == same.launches_per_chunk


@GRAPH
def test_context_body(use_graph):
    """Videos with R = N - 1 (13 frames: frame N - 2 reads the padding frame's maps), 5 frames and R < N - 1 (28
    frames).  The last video (25 frames) has R = N - 1 too: it reads the list's first padding row, a zero frame, as a
    one-video predictor reads its own."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor, _context_rows

    assert _context_rows(13, T) == 12 and 5 in LENGTHS and _context_rows(28, T) < 27 and _context_rows(25, T) == 24
    head, feats = context_head(7), pooled_features(8)
    videos = make_videos(LENGTHS, SIZES_64, 9)
    make = lambda n, sizes, i: BatchedPredictor(head, K, n, T, (64, 64), features_of=feats, use_graph=use_graph,
                                                **sized(n, sizes, {}))
    assert_each_video_equals_its_one_video_table(make, videos)


@GRAPH
def test_regression_body(use_graph):
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    torch.manual_seed(10)
    head = LinearRegressionHead(128, 2 * K).to(DEV).eval()
    feats = pooled_features(11)
    videos = make_videos(LENGTHS, SIZES_64, 12)
    make = lambda n, sizes, i: BatchedPredictor(head, K, n, T, (64, 64), features_of=feats, use_graph=use_graph,
                                                **sized(n, sizes, {}))
    assert_each_video_equals_its_one_video_table(make, videos)


def crop_boxes(lengths, sizes, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rows = []
    for n, (h, w) in zip(lengths, sizes):
        wh = torch.randint(16, min(h, w) + 1, (n, 2), device=DEV, generator=gen).float()
        xy = (torch.rand(n, 2, device=DEV, generator=gen) * (torch.tensor([w, h], device=DEV) - wh + 8)).floor()
        rows.append(torch.cat([xy, wh], 1).contiguous())
    return rows


@GRAPH
@pytest.mark.parametrize("context", [False, True], ids=["frames", "context"])
def test_crop_body(context, use_graph):
    """Each video's boxes in one (sum N, 4) table; frame_sizes takes the place of frame_hw."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = context_head(13) if context else frame_head(13, c=128)
    feats = pooled_features(14)
    videos = make_videos(LENGTHS, SIZES_64, 15)
    rows = crop_boxes(LENGTHS, SIZES_64, 16)
    boxes = torch.cat(rows).contiguous()

    def make(n, sizes, i):
        kw = dict(frame_sizes=sizes) if sizes is not None else dict(frame_hw=tuple(videos[i].shape[1:3]))
        return BatchedPredictor(head, K, n, T, (64, 64), features_of=feats, use_graph=use_graph,
                                bboxes=boxes if i is None else rows[i], crop_dtype=torch.bfloat16,
                                **kw)

    assert_each_video_equals_its_one_video_table(make, videos)


# ---- shards -------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gather_worker(rank, world, port, out):
    from lightning_pose_b200.utils.predictions import BatchedPredictor, segment_chunks

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        ok = {}
        videos = make_videos(LENGTHS, SIZES_64, 17)
        feats = pooled_features(18)
        for name, head in (("context", context_head(19)), ("frames", frame_head(20, c=128))):
            make = lambda s: BatchedPredictor(head, K, LENGTHS, T, (64, 64), features_of=feats, frame_sizes=SIZES_64, shard=s)
            whole = make((0, 1))
            whole.run(segment_chunks(videos, T))
            bp = make((rank, world))
            bp.run(segment_chunks(videos, T, bp.feed_range))
            table = bp.gather()
            torch.cuda.synchronize()
            ok[name] = bool(torch.equal(table, whole.table))
        out[rank] = ok
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_gather_two_ranks_gloo():
    world = 2
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_gather_worker, args=(world, _free_port(), out), nprocs=world, join=True)
        assert dict(out) == {r: {"context": True, "frames": True} for r in range(world)}
