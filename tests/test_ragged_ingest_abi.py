"""CPU: the ragged ingest entries (lpb_frames_normalize_ragged, lpb_frames_crop_normalize_ragged) refuse malformed
arguments with LPB_ERR_INVALID before they queue anything (the device pointers are fake, so a launch or a CUDA call
would show as a different code), and the host side of a BatchedPredictor built with per-video frame sizes: its segment
checks, the chunks ``segment_chunks`` cuts, and its refusals."""
import ctypes as C

import pytest
import torch

LPB_ERR_INVALID = -1
ENTRIES = ["lpb_frames_normalize_ragged", "lpb_frames_crop_normalize_ragged"]


def call(name, arena=0x1000, slot_bytes=1024, F=4, cursor=0x1000, videos=0x1000, table=((0, 8, 10), (5, 16, 20)),
         n_videos=None, boxes=0x1000, n_boxes=9, out_h=8, out_w=8, std=(0.229, 0.224, 0.225), layout=0, fmt=0, out=0x1000,
         boxes_out=0x1000):
    from lightning_pose_b200 import _lib

    host = (C.c_int64 * max(3 * len(table), 1))(*[v for row in table for v in row]) if table is not None else None
    n = len(table or ((0, 1, 1),)) if n_videos is None else n_videos
    m3, s3 = (C.c_float * 3)(0.485, 0.456, 0.406), (C.c_float * 3)(*std)
    head = [C.c_void_p(arena), slot_bytes, F, C.c_void_p(cursor), C.c_void_p(videos), C.cast(host, C.c_void_p) if host else None, n]
    tail = [out_h, out_w, m3, s3, layout, fmt, C.c_void_p(out), C.c_void_p(boxes_out), None]
    if name == "lpb_frames_crop_normalize_ragged":
        head += [C.c_void_p(boxes), n_boxes]
    return getattr(_lib.lib, name)(*head, *tail)


def refused(rc, msg):
    from lightning_pose_b200 import _lib

    err = _lib.lib.lpb_last_error().decode()
    assert rc == LPB_ERR_INVALID, (rc, err)
    assert msg in err, err


@pytest.mark.parametrize("name,arg", [(name, arg) for name in ENTRIES
                                      for arg in ("arena", "cursor", "videos", "table", "out", "boxes_out")]
                         + [("lpb_frames_crop_normalize_ragged", "boxes")])
def test_null_pointers(name, arg):
    refused(call(name, **{arg: None if arg == "table" else 0}), "null pointer")


@pytest.mark.parametrize("name", ENTRIES)
def test_empty_table(name):
    refused(call(name, table=(), n_videos=0), "the video table is empty")


@pytest.mark.parametrize("name", ENTRIES)
@pytest.mark.parametrize("table,msg", [
    (((0, 8, 10), (5, 19, 18)), "video 1's 19 x 18 frames (1026 bytes) do not fit a 1024-byte slot"),
    (((0, 8, 10), (5, 0, 20)), "video 1 has frame size 0 x 20"),
    (((1, 8, 10),), "video 0 starts at row 1"),
    (((0, 8, 10), (0, 8, 10)), "video 1 starts at row 0"),
    (((0, 8, 10), (7, 8, 10), (6, 8, 10)), "video 2 starts at row 6"),
])
def test_bad_tables(name, table, msg):
    refused(call(name, table=table), msg)


@pytest.mark.parametrize("name", ENTRIES)
@pytest.mark.parametrize("kw,msg", [
    ({"arena": 0x1008}, "the arena must be 16-byte aligned"),
    ({"videos": 0x1004}, "the table 8-byte aligned"),
    ({"slot_bytes": 1032}, "slot_bytes 1032 is not a positive multiple of 16"),
    ({"slot_bytes": 0}, "slot_bytes 0"),
    ({"F": -1}, "outside 0..65535"),
    ({"F": 65536}, "outside 0..65535"),
    ({"out_h": 0}, "bad shape/layout"),
    ({"layout": 2}, "bad shape/layout"),
    ({"fmt": 3}, "unknown output format 3"),
    ({"std": (0.229, 0.0, 0.225)}, "std must be positive"),
])
def test_bad_arguments(name, kw, msg):
    refused(call(name, **kw), msg)


def test_crop_entry_needs_a_box_row():
    refused(call("lpb_frames_crop_normalize_ragged", n_boxes=0), "bad shape/layout")


@pytest.mark.parametrize("name", ENTRIES)
def test_no_frames_is_a_no_op(name):
    assert call(name, F=0) == 0


def test_slot_arena_offsets_are_64_bit():
    """96 slots of 1080 x 1920 frames: 597 MB, past 2^31 bytes only for larger chunks, which the int64 slot size carries."""
    from lightning_pose_b200 import ops

    assert ops.ragged_slot_bytes([(1080, 1920), (720, 1280)]) == 1080 * 1920 * 3
    assert ops.ragged_slot_bytes([(407, 395), (5, 7)]) == -(-407 * 395 * 3 // 16) * 16
    assert call("lpb_frames_normalize_ragged", slot_bytes=(1 << 31) + 16, F=0) == 0


def test_ragged_wrappers_refuse_cpu_tensors():
    from lightning_pose_b200 import ops

    table = ops.ragged_videos([3, 4], [(8, 10), (16, 20)])
    assert table.tolist() == [[0, 8, 10], [3, 16, 20]]
    with pytest.raises(ValueError, match="2 videos but 1 frame sizes"):
        ops.ragged_videos([3, 4], [(8, 10)])
    cur = torch.zeros(1, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.frames_normalize_ragged(torch.zeros(4 * 960, dtype=torch.uint8), 960, 4, cur, table, table, (8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.frames_crop_normalize_ragged(torch.zeros(4 * 960, dtype=torch.uint8), 960, 4, cur, table, table,
                                         torch.ones(7, 4), (8, 8))


# ---- the predictor's host side ----------------------------------------------------------------------------------------
SIZES = [(12, 16), (8, 10), (20, 6), (9, 9)]


def videos_of(lengths, sizes=SIZES):
    return [torch.full((n, h, w, 3), i + 1, dtype=torch.uint8) for i, (n, (h, w)) in enumerate(zip(lengths, sizes))]


def layout(chunks):
    """Each chunk as (frames, H, W, first byte, last byte) per segment."""
    return [[(s.shape[0], s.shape[1], s.shape[2], int(s[0, 0, 0, 0]), int(s[-1, 0, 0, 0])) for s in c] for c in chunks]


def test_segment_chunks_short_videos_and_three_videos_in_a_chunk():
    from lightning_pose_b200.utils.predictions import segment_chunks

    # T = 8: videos of 3, 2 and 6 frames; chunk 0 spans three videos, chunk 1 holds the end of the third and the fourth
    # video (12 frames), whose end pads chunk 2 with a zero frame of its size
    chunks = list(segment_chunks(videos_of([3, 2, 6, 12]), 8))
    assert layout(chunks) == [
        [(3, 12, 16, 1, 1), (2, 8, 10, 2, 2), (3, 20, 6, 3, 3)],
        [(3, 20, 6, 3, 3), (5, 9, 9, 4, 4)],
        [(8, 9, 9, 4, 0)],
    ]
    assert sum(s.shape[0] for s in chunks[2]) == 8 and int(chunks[2][0][7:].sum()) == 0 and int(chunks[2][0][:7].min()) == 4
    assert layout(segment_chunks(videos_of([2]), 8)) == [[(8, 12, 16, 1, 0)]]  # a video shorter than a chunk


def test_segment_chunks_of_a_shard_pad_past_its_range_at_each_row_s_size():
    from lightning_pose_b200.utils.predictions import segment_chunks

    # rows [4, 9) in chunks of 4: rows 9 .. 11 lie past the range, in videos 2 and 3, and are zero frames of their sizes
    chunks = list(segment_chunks(videos_of([3, 2, 6, 13]), 4, (4, 9)))
    assert layout(chunks) == [[(1, 8, 10, 2, 2), (3, 20, 6, 3, 3)], [(3, 20, 6, 3, 0), (1, 9, 9, 0, 0)]]
    assert int(chunks[1][0][1:].sum()) == 0


def head():
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    return HeatmapHead("resnet50", 64, 3)


def test_predictor_checks_segments_against_its_videos():
    from lightning_pose_b200.utils.predictions import BatchedPredictor, segment_chunks

    lengths = [3, 2, 6, 13]
    bp = BatchedPredictor(head(), 3, lengths, 8, (64, 64), features_of=lambda x: x, device="cpu", frame_sizes=SIZES)
    assert bp.slot_bytes == 576 and bp._arena.numel() == 8 * 576 and bp.n_chunks == 3
    assert bp._videos_host.tolist() == [[0, 12, 16], [3, 8, 10], [5, 20, 6], [11, 9, 9]]
    chunks = list(segment_chunks(videos_of(lengths), 8))
    assert bp._inputs(chunks[0], None) == ("ragged", (bp._arena,))
    with pytest.raises(ValueError, match=r"from row 0 holds segments .* \[\(3, 12, 16\), \(2, 8, 10\), \(3, 20, 6\)\]"):
        bp._inputs(chunks[1], None)  # the second chunk first
    with pytest.raises(ValueError, match="in this order"):
        bp._inputs(chunks[0][::-1], None)
    with pytest.raises(ValueError, match="holds segments"):
        bp._inputs([chunks[0][0], chunks[0][1], chunks[0][2][:2]], None)  # 7 frames
    with pytest.raises(ValueError, match="holds segments"):
        bp._inputs([chunks[0][0], chunks[0][1].transpose(1, 2), chunks[0][2]], None)  # a 10 x 8 segment
    with pytest.raises(ValueError, match="must be uint8"):
        bp._inputs([s.float() for s in chunks[0]], None)
    with pytest.raises(ValueError, match="list of uint8"):
        bp._inputs(torch.zeros(8, 12, 16, 3, dtype=torch.uint8), None)
    with pytest.raises(ValueError, match="take their boxes"):
        bp._inputs(chunks[0], torch.zeros(8, 4))
    # a shard starts at its own first row
    shard = BatchedPredictor(head(), 3, lengths, 8, (64, 64), features_of=lambda x: x, device="cpu", frame_sizes=SIZES,
                             shard=(1, 2))
    first = next(segment_chunks(videos_of(lengths), 8, shard.feed_range))
    assert shard.feed_range[0] == 12 and shard._inputs(first, None)[0] == "ragged"


def test_predictor_fills_the_arena_slot_by_slot():
    from lightning_pose_b200.utils.predictions import BatchedPredictor, segment_chunks

    lengths = [3, 2, 6, 13]
    bp = BatchedPredictor(head(), 3, lengths, 8, (64, 64), features_of=lambda x: x, device="cpu", frame_sizes=SIZES)
    bp._arena.fill_(0xEE)
    segs = next(segment_chunks(videos_of(lengths), 8))
    bp._fill_arena(segs)
    slots = bp._arena.view(8, 576)
    for f, (fill, size) in enumerate([(1, 576)] * 3 + [(2, 240)] * 2 + [(3, 360)] * 3):
        assert bool((slots[f, :size] == fill).all()) and bool((slots[f, size:] == 0xEE).all()), f


def test_predictor_refusals():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    feats = lambda x: x  # noqa: E731
    with pytest.raises(ValueError, match="one \\(H >= 1, W >= 1\\) per video: 2 videos"):
        BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), features_of=feats, device="cpu", frame_sizes=[(8, 8)])
    with pytest.raises(ValueError, match="per video"):
        BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), features_of=feats, device="cpu", frame_sizes=[(8, 8), (0, 4)])
    with pytest.raises(ValueError, match="single-view"):
        BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), features_of=feats, device="cpu", frame_sizes=[(8, 8), (9, 9)],
                         num_views=2)
    with pytest.raises(ValueError, match="need features_of"):
        BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), device="cpu", frame_sizes=[(8, 8), (9, 9)])
    boxes = torch.ones(9, 4)
    with pytest.raises(ValueError, match="drop frame_hw"):
        BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), features_of=feats, device="cpu", frame_sizes=[(8, 8), (9, 9)],
                         bboxes=boxes, frame_hw=(8, 8))
    # a predictor without frame_sizes keeps its refusals: uint8 views of a new size after the first chunk
    bp = BatchedPredictor(head(), 3, [4, 5], 8, (64, 64), features_of=feats, device="cpu")
    bp._inputs([torch.zeros(8, 8, 8, 3, dtype=torch.uint8)], None)
    with pytest.raises(ValueError, match="differ from the first chunk's"):
        bp._inputs([torch.zeros(8, 9, 9, 3, dtype=torch.uint8)], None)
    assert bp.frame_sizes is None


def test_crop_mode_takes_the_sizes_in_place_of_frame_hw():
    """Without frame_hw the constructor goes on to the boxes, which must be a device table."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        BatchedPredictor(head(), 3, [3, 2, 6, 13], 8, (64, 64), features_of=lambda x: x, device="cpu", frame_sizes=SIZES,
                         bboxes=torch.ones(24, 4))
