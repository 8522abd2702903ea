"""CPU: the arithmetic of prediction over a list of videos (row rules, window tables, shard feed ranges, edge fills)
against a per-video restatement, the list predictor's input checks, and lpb_pack_context_predictions_segments'
argument checks (fake device pointers: a launch or CUDA call would show here)."""
import ctypes as C
import math
import random

import pytest
import torch

FAKE = C.c_void_p(0x1000)


def per_video_source(lengths, t):
    """Global row -> global source row, one video at a time with the one-video rule."""
    from lightning_pose_b200.utils.predictions import _context_rows, _context_source

    out, row0 = [], 0
    for n in lengths:
        r = _context_rows(n, t)
        out += [row0 + _context_source(f, n, r) for f in range(n)]
        row0 += n
    return out


def random_lists(count, seed, context=True):
    rng = random.Random(seed)
    for _ in range(count):
        lo = 5 if context else 1
        lengths = [rng.choice([lo, lo + 1, rng.randint(lo, 12), rng.randint(lo, 40)]) for _ in range(rng.randint(1, 7))]
        yield lengths, rng.choice([1, 2, 3, 4, 5, 8, 13]), rng.choice([1, 2, 3, 5, 8])


def simulate_context_list(lengths, t, world):
    """Every shard of a context list run symbolically: chunks of its feed range, the window table of each chunk, the
    writer's rule, then the gather and the edge fill.  A row is ("ok", g) when frame g's prediction came from its true
    window: the frames g - 2 .. g + 2 of its own video as fed, and the padding frame's maps in place of frame N."""
    from lightning_pose_b200.utils.predictions import (_context_rows, _context_window_index, context_edge_fill,
                                                       frame_range_for_rank, shard_feed_range)

    starts = [0]
    for n in lengths:
        starts.append(starts[-1] + n)
    total = starts[-1]
    video = [v for v, n in enumerate(lengths) for _ in range(n)]
    source = per_video_source(lengths, t)
    final = [None] * total
    for rank in range(world):
        a, b = frame_range_for_rank(total, rank, world)
        if a == b:
            continue
        lo, hi = shard_feed_range(lengths, t, rank, world, context=True)
        assert lo <= a and b <= hi <= total + 1
        fed = set(range(lo, min(hi, total)))
        rows = [None] * total
        for j in range(math.ceil((hi - lo) / t)):
            c = lo + j * t
            idx = _context_window_index(c, t, lengths)
            for o in range(t):
                g = c - 2 + o
                if not 0 <= g < total:
                    continue
                v = video[g]
                row0, n = starts[v], lengths[v]
                f = g - row0
                if not 2 <= f <= n - 2:
                    continue
                ok = True
                for s, m in enumerate(idx[o]):
                    want = g - 2 + s
                    if want < row0 + n:
                        ok &= m == o + s and want in fed  # map row o + s holds frame c - 4 + o + s = want
                    else:  # frame N: only the R = N - 1 window reads it, from the padding frame's maps
                        ok &= s == 4 and _context_rows(n, t) == n - 1 and m == t + 4
                for r in range(n):
                    if source[row0 + r] == g:
                        rows[row0 + r] = ("ok" if ok else "bad", g)
        final[a:b] = rows[a:b]
    for row, src in context_edge_fill(lengths, t, world):
        final[row] = final[src]
    return final, [("ok", s) for s in source]


@pytest.mark.parametrize("seed", range(6))
def test_context_list_shards_give_every_row_its_true_frame(seed):
    for lengths, t, world in random_lists(60, seed):
        got, want = simulate_context_list(lengths, t, world)
        assert got == want, (lengths, t, world)


def test_context_list_fixed_cases():
    # R >= N, R < N - 1, R = N - 1 (N = 9 at T = 8), N = 5 twice, a list that ends on a chunk boundary with R = N - 1
    for lengths in ([30, 27, 25, 5, 5, 9, 16], [9], [7, 9], [5, 5, 5, 5], [23, 9]):
        for world in (1, 2, 3, 8):
            got, want = simulate_context_list(lengths, 8, world)
            assert got == want, (lengths, world)


def test_context_rows_table_matches_the_one_video_rule():
    from lightning_pose_b200 import ops
    from lightning_pose_b200.utils.predictions import _context_rows

    for lengths, t, _ in random_lists(200, 1):
        seg = ops.context_segments(lengths, t).tolist()
        row0 = 0
        for (r0, n, r), length in zip(seg, lengths):
            assert (r0, n, r) == (row0, length, _context_rows(length, t))
            row0 += length


def test_edge_fill_is_every_row_whose_source_lies_in_another_shard():
    from lightning_pose_b200.utils.predictions import context_edge_fill

    for lengths, t, world in random_lists(300, 2):
        per = -(-sum(lengths) // world)
        want = [(row, src) for row, src in enumerate(per_video_source(lengths, t)) if row // per != src // per]
        assert context_edge_fill(lengths, t, world) == want, (lengths, t, world)


def test_one_video_list_edge_fill_equals_the_int_form():
    from lightning_pose_b200.utils.predictions import context_edge_fill

    for n in range(5, 60):
        for t in (1, 3, 8):
            for world in (1, 2, 5):
                assert context_edge_fill([n], t, world) == context_edge_fill(n, t, world)


def test_frame_list_feed_range_is_the_rows():
    from lightning_pose_b200.utils.predictions import frame_range_for_rank, shard_feed_range

    for lengths, t, world in random_lists(200, 3, context=False):
        for rank in range(world):
            assert shard_feed_range(lengths, t, rank, world) == frame_range_for_rank(sum(lengths), rank, world)


def test_context_list_feed_range_stays_in_its_videos():
    """The halo starts no earlier than the first row's video and ends no later than one frame past the last row's."""
    from lightning_pose_b200.utils.predictions import frame_range_for_rank, shard_feed_range

    for lengths, t, world in random_lists(300, 4):
        starts = [0]
        for n in lengths:
            starts.append(starts[-1] + n)
        for rank in range(world):
            a, b = frame_range_for_rank(starts[-1], rank, world)
            lo, hi = shard_feed_range(lengths, t, rank, world, context=True)
            if a == b:
                assert (lo, hi) == (a, b)
                continue
            first = max(s for s in starts[:-1] if s <= a)
            end = min(s for s in starts[1:] if s >= b)
            assert max(a - 2, first) == lo and b <= hi <= min(b + 2, end + 1), (lengths, t, world, rank)


def test_window_table_of_one_video_is_the_plain_table():
    from lightning_pose_b200.utils.predictions import _context_rows, _context_window_index

    for n in range(5, 40):
        for t in (1, 2, 4, 8):
            plain = [[i + s for s in range(5)] for i in range(t)]
            for start in range(0, n + 1, t):
                got = _context_window_index(start, t, [n])
                if _context_rows(n, t) == n - 1 and start <= n < start + t:  # the chunk that predicts frame N - 2
                    plain_pad = [row[:] for row in plain]
                    plain_pad[n - start][4] = t + 4
                    assert got == plain_pad
                else:
                    assert got == plain


# ---- input checks ---------------------------------------------------------------------------------------------------
def test_list_predictor_refuses_bad_lists():
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = HeatmapHead("resnet50", 64, 3)
    with pytest.raises(ValueError, match="empty"):
        BatchedPredictor(head, 3, [], 8, (64, 64), device="cpu")
    with pytest.raises(ValueError, match="at least one frame"):
        BatchedPredictor(head, 3, [4, 0, 7], 8, (64, 64), device="cpu")
    with pytest.raises(TypeError):
        BatchedPredictor(head, 3, [4, 2.5], 8, (64, 64), device="cpu")
    ctx = HeatmapMHCRNNHead("vits_dino", 32, 3, upsampling_factor=1)
    with pytest.raises(ValueError, match=r"videos \[1\] have fewer"):
        BatchedPredictor(ctx, 3, [9, 4, 5], 8, (64, 64), device="cpu")


def test_list_predictor_tables_and_ranges():
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = HeatmapHead("resnet50", 64, 3)
    bp = BatchedPredictor(head, 3, [4, 7, 1], 8, (64, 64), device="cpu")
    assert bp.table.shape == (12, 9) and bp.feed_range == (0, 12) and bp.n_chunks == 2
    assert [tuple(t.shape) for t in bp.video_tables()] == [(4, 9), (7, 9), (1, 9)]
    assert all(t.data_ptr() == bp.table[r].data_ptr() for t, r in zip(bp.video_tables(), (0, 4, 11)))
    one = BatchedPredictor(head, 3, 12, 8, (64, 64), device="cpu")
    assert len(one.video_tables()) == 1 and one.video_tables()[0] is one.table
    # a context list whose last video (N = 9, T = 8: R = 8 = N - 1) ends on a chunk boundary: one more chunk
    ctx = HeatmapMHCRNNHead("vits_dino", 32, 3, upsampling_factor=1)
    bp = BatchedPredictor(ctx, 3, [7, 9], 8, (64, 64), device="cpu")
    assert bp.feed_range == (0, 17) and bp.n_chunks == 3


def test_video_dataframes_have_the_one_video_schema():
    from lightning_pose_b200.utils.predictions import PredictionHandler

    names = ["a", "b"]
    tables = [torch.arange(n * 6, dtype=torch.float32).reshape(n, 6) for n in (3, 5)]
    dfs = PredictionHandler(names, 8).video_dataframes(tables)
    for df, table in zip(dfs, tables):
        want = PredictionHandler(names, table.shape[0]).dataframe(table)
        assert df.equals(want) and df.shape == (table.shape[0], 6)
    views = PredictionHandler(names, 8, view_names=["top", "side"]).video_dataframes([torch.zeros(4, 12)])
    assert list(views[0]) == ["top", "side"] and views[0]["side"].shape == (4, 6)


# ---- lpb_pack_context_predictions_segments: argument checks without a device ----------------------------------------
def entry(**kw):
    from lightning_pose_b200 import _lib

    seg = kw.pop("seg", [(0, 9, 8), (9, 12, 8)])
    host = (C.c_int64 * max(3 * len(seg), 1))(*[v for row in seg for v in row])
    a = dict(kp_sf=FAKE, conf_sf=FAKE, kp_mf=FAKE, conf_mf=FAKE, n=8, K=3, bbox=FAKE, mh=64.0, mw=64.0, table=FAKE,
             n_rows=21, cursor=FAKE, segments=FAKE, segments_host=host, n_segments=len(seg), step=8, window_index=FAKE)
    a.update(kw)
    return _lib.lib.lpb_pack_context_predictions_segments(*a.values(), None)


def refused(rc, msg):
    from lightning_pose_b200 import _lib

    assert rc == -1, rc
    assert msg in _lib.lib.lpb_last_error().decode()


@pytest.mark.parametrize("name", ["kp_sf", "conf_sf", "kp_mf", "conf_mf", "bbox", "table", "cursor", "segments",
                                  "segments_host"])
def test_segments_entry_refuses_null_pointers(name):
    refused(entry(**{name: None}), "pack_context_predictions_segments: null pointer")


@pytest.mark.parametrize("name,addr", [("kp_sf", 0x1002), ("table", 0x1001), ("cursor", 0x1004), ("segments", 0x1004),
                                       ("window_index", 0x1002)])
def test_segments_entry_refuses_misaligned_pointers(name, addr):
    refused(entry(**{name: C.c_void_p(addr)}), "pack_context_predictions_segments: misaligned pointer")


def test_segments_entry_refuses_bad_arguments():
    refused(entry(n=-1), "bad shape")
    refused(entry(K=0), "bad shape")
    refused(entry(step=0), "step")
    refused(entry(mh=0.0), "model dims")
    refused(entry(seg=[], n_segments=0), "no segments")


@pytest.mark.parametrize("seg,n_rows,msg", [
    ([(0, 9, 8), (9, 4, 8)], 13, "video 1 has 4 frames"),
    ([(1, 9, 8), (10, 11, 8)], 21, "segment 0"),                # does not start at row 0
    ([(0, 9, 8), (10, 11, 8)], 21, "segment 1"),                # a gap
    ([(0, 9, 8), (8, 13, 8)], 21, "segment 1"),                 # an overlap
    ([(0, 9, 8), (9, 12, 8)], 20, "segment 1"),                 # past the table's end
    ([(0, 9, 8), (9, 12, 8)], 22, "cover 21 of the table's 22 rows"),
    ([(0, 9, 9), (9, 12, 8)], 21, "gives R = 9"),               # R is not the reader's
])
def test_segments_entry_refuses_segments_that_do_not_tile_the_table(seg, n_rows, msg):
    refused(entry(seg=seg, n_rows=n_rows), msg)


def test_segments_entry_empty_call_is_a_no_op():
    assert entry(n=0, window_index=None) == 0


def test_segments_wrapper_refuses_cpu_tensors():
    from lightning_pose_b200 import ops

    kp, cf, bb = torch.zeros(4, 6), torch.zeros(4, 3), torch.ones(4, 4)
    seg = ops.context_segments([5, 5], 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.pack_context_predictions_segments(kp, cf, kp, cf, bb, 64, 64, torch.zeros(10, 9), 4, None, seg, seg)
