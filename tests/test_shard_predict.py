"""CPU: the shard arithmetic of BatchedPredictor(..., shard=(rank, world)) against a host restatement.

A context model's final table gives every row one source frame.  Here every row of the one-GPU table is labelled with
its source by ``PredictionHandler.fix_context_preds_confs`` applied to frame indices, the reference's own fix-up, on the
rows of a reader that is counted here window by window (pinned to the reference's row maps in
tests/golden/context_predict.npz), not taken from the code under test.  Each
shard is then restated at the level of frames: which frames it feeds, from where its cursor starts, which output frames
its chunks produce, and which of those see their whole 5-frame window.  The kernel writes each output frame to every row
whose source it is.  The rows each shard owns, joined and completed by ``context_edge_fill``, must hold the same source
as the one-GPU table in every row.
"""
import numpy as np
import pytest
import torch

from conftest import load_golden
from lightning_pose_b200.utils.predictions import (PredictionHandler, context_edge_fill, frame_range_for_rank,
                                                   shard_feed_range)

# R = N - 1 needs T > 3 and N = 1 (mod T): 93 and 97 give it for T = 92 and 96, and T = 8 gives it for N = 25, 33, ...
N_GRID = [*range(5, 41), 93, 97, 100_000]
T_GRID = [1, 3, 8, 92, 96]
WORLDS = [1, 2, 3, 8]
HALO, UNWRITTEN = -1, -2  # a frame predicted from the zero halo or a padded window; a row nothing wrote


def reader_rows(n: int, t: int) -> int:
    """R: the rows the reference's context reader yields, T per window of S = T + 4 frames.  With step 1 it reads one
    window per frame (``PrepareDALI.num_iters``' first branch); otherwise windows start at 0, T, 2T, ... until one
    reaches the last frame (at least one window)."""
    if t == 1:
        return n
    windows = 1
    while (windows - 1) * t + t + 4 < n:
        windows += 1
    return windows * t


def reference_sources(n: int, t: int) -> np.ndarray:
    """Source frame of each row of the reference's final table: its reader's R rows hold frames 2 .. R + 1 (trimmed to
    N), then fix_context_preds_confs shifts and fills them."""
    r = reader_rows(n, t)
    stacked = torch.arange(2, r + 2, dtype=torch.float64)[:n, None]
    fixed = PredictionHandler(["kp"], n, model_type="heatmap_mhcrnn").fix_context_preds_confs(stacked)
    return fixed[:, 0].numpy().astype(np.int64)


def kernel_sources(n: int, t: int) -> np.ndarray:
    """The row rule of pack_context_kernel (csrc/predict.cu), restated over all rows."""
    r, f = reader_rows(n, t), np.arange(n)
    return np.clip(f, 2, n - 3) if r >= n else np.where((f >= 2) & (f <= r - 1), f, 2)


def shard_rows(n: int, t: int, rank: int, world: int) -> np.ndarray:
    """The whole (N,) table of one shard after its chunks, as sources: chunks of T from lo until frame hi is fed (the
    last padded past N as the one-GPU caller pads); a chunk fed from cursor c outputs frames c - 2 .. c + T - 3.  A frame
    is right when its window f - 2 .. f + 2 was fed from the video, or from the padding after frame N - 1 as on one GPU."""
    lo, hi = shard_feed_range(n, t, rank, world, context=True)
    table = np.full(n, UNWRITTEN)
    if lo == hi:
        return table
    end = lo + -(-(hi - lo) // t) * t
    src = kernel_sources(n, t)
    out = (src >= lo - 2) & (src <= end - 3)  # the frame each row takes is output by one of this shard's chunks
    right = (src - 2 >= lo) & ((src + 2 < hi) | (hi == n))
    table[out] = np.where(right[out], src[out], HALO)
    return table


def sharded_sources(n: int, t: int, world: int) -> np.ndarray:
    joined = np.full(n, UNWRITTEN)
    for rank in range(world):
        a, b = frame_range_for_rank(n, rank, world)
        joined[a:b] = shard_rows(n, t, rank, world)[a:b]
    for row, src in context_edge_fill(n, t, world):
        joined[row] = joined[src]
    return joined


def test_reader_rows_match_the_reference_row_maps():
    """The reference's own final row maps (its reader, predict_step and fix-up run on frame labels) for each golden
    case: R = N - 1, R < N, R >= N, N = 5 and N < S."""
    g = load_golden("context_predict")
    cases = [f[: -len("_meta")] for f in g.files if f.startswith("uf1_") and f.endswith("_meta")]
    assert len(cases) >= 5
    for case in cases:
        n, s = (int(v) for v in g[f"{case}_meta"][:2])
        np.testing.assert_array_equal(reference_sources(n, s - 4), g[f"{case}_rows"], err_msg=case)


@pytest.mark.parametrize("t", T_GRID)
def test_context_shards_give_the_one_gpu_rows(t):
    for n in N_GRID:
        ref = reference_sources(n, t)
        np.testing.assert_array_equal(kernel_sources(n, t), ref, err_msg=f"row rule N={n} T={t}")
        np.testing.assert_array_equal(shard_rows(n, t, 0, 1), ref, err_msg=f"one GPU N={n} T={t}")
        assert context_edge_fill(n, t, 1) == []
        for world in WORLDS:
            np.testing.assert_array_equal(sharded_sources(n, t, world), ref, err_msg=f"N={n} T={t} world={world}")


def test_context_grid_covers_every_regime():
    seen = set()
    for n in N_GRID:
        for t in T_GRID:
            r = reader_rows(n, t)
            seen.add("R>=N" if r >= n else ("R=N-1" if r == n - 1 else "R<N-1"))
            for world in WORLDS:
                sizes = [b - a for a, b in (frame_range_for_rank(n, q, world) for q in range(world))]
                seen.update({"empty shard"} if 0 in sizes else set())
                seen.update({"shard < 3 rows"} if any(0 < s < 3 for s in sizes) else set())
                for q in range(world):
                    a, b = frame_range_for_rank(n, q, world)
                    lo, _ = shard_feed_range(n, t, q, world, context=True)
                    if a < b and lo < max(a - 2, 0):
                        seen.add("R=N-1 shard starts a frame early")
    assert seen == {"R>=N", "R=N-1", "R<N-1", "empty shard", "shard < 3 rows", "R=N-1 shard starts a frame early"}


def test_fill_rows_cross_shards_only():
    # N = 27, T = 8: R = 24 < N, rows 24-26 hold frame 2 (shard 0 of 2); rows 0 and 1 are shard 0's own
    assert context_edge_fill(27, 8, 2) == [(24, 2), (25, 2), (26, 2)]
    # N = 30, T = 8: R = 32 >= N, rows 28 and 29 hold frame 27; with 8 shards of 4 rows row 27 is in shard 6, 28-29 in 7
    assert context_edge_fill(30, 8, 8) == [(28, 27), (29, 27)]
    assert context_edge_fill(30, 8, 3) == []


@pytest.mark.parametrize("world", WORLDS)
def test_frame_model_feed_range_is_the_shard(world):
    for n in N_GRID:
        covered = []
        for rank in range(world):
            a, b = frame_range_for_rank(n, rank, world)
            for t in T_GRID:
                assert shard_feed_range(n, t, rank, world) == (a, b)
            covered.extend(range(a, b))
        assert covered == list(range(n))


def test_context_feed_range_halo():
    assert shard_feed_range(100, 16, 0, 4, context=True) == (0, 27)
    assert shard_feed_range(100, 16, 1, 4, context=True) == (23, 52)
    assert shard_feed_range(100, 16, 3, 4, context=True) == (73, 100)
    assert shard_feed_range(5, 3, 7, 8, context=True) == (5, 5)  # no rows: nothing to feed
