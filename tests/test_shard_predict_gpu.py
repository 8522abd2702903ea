"""GPU: BatchedPredictor(..., shard=(rank, world)) gives the one-GPU table bit for bit.

One process: each shard's predictor runs in turn on one GPU, fed its ``feed_range`` in chunks with the last one padded,
and its own rows are joined with ``fill_context_edges``, the code ``gather()`` runs after its all-gather.  Two
processes: ``gather()`` itself over gloo, both ranks on one GPU.  Every kernel on the chunk path works per frame and per
heatmap plane, so a frame's prediction does not depend on where in a chunk it lands, and the tables must be equal.
"""
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WORLDS = [1, 2, 3, 8]
K = 17


def chunks_of(video, lo, hi, t, zero_pad=False):
    """Frames [lo, hi) of the video in chunks of t, the last padded with zero frames or its final frame.  ``video`` is
    a tensor, a tuple (features, boxes) or a list of views, each with a leading frame axis."""
    parts = list(video) if isinstance(video, (tuple, list)) else [video]
    n_chunks = -(-(hi - lo) // t)
    padded = []
    for x in parts:
        fill = torch.zeros_like(x[:1]) if zero_pad else x[hi - 1 : hi]
        padded.append(torch.cat([x[lo:hi], fill.expand(n_chunks * t - (hi - lo), *x.shape[1:])]))
    items = [[x[i : i + t] for x in padded] for i in range(0, n_chunks * t, t)]
    if isinstance(video, list):
        return items
    return [tuple(it) if isinstance(video, tuple) else it[0] for it in items]


def assert_shards_equal_whole(make, video, n, t, zero_pad=False):
    """make(shard) -> BatchedPredictor.  The unsharded table against the shards' rows joined and edge-filled."""
    from lightning_pose_b200.utils.predictions import fill_context_edges

    whole = make((0, 1))
    assert whole.feed_range == (0, n)
    whole.run(chunks_of(video, 0, n, t, zero_pad))
    for world in WORLDS:
        joined = torch.full_like(whole.table, float("nan"))
        for rank in range(world):
            bp = make((rank, world))
            lo, hi = bp.feed_range
            if lo < hi:
                bp.run(chunks_of(video, lo, hi, t, zero_pad))
            assert int(bp.cursor) == lo + -(-(hi - lo) // t) * t
            a, b = bp.rows
            joined[a:b] = bp.table[a:b]
        if whole.context:
            fill_context_edges(joined, t, world)
        torch.cuda.synchronize()
        bad = (joined != whole.table).any(1).nonzero().flatten().tolist()
        assert not bad, f"world {world}: rows {bad} differ"


def make_head(c, seed, arch="resnet50"):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead(arch, c, K)
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


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_feature_shards(dtype, use_graph):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    n, t, img = 45, 8, 128
    head = make_head(512, 3)
    gen = torch.Generator(device=DEV).manual_seed(5)
    feats = (torch.randn(n, 512, 4, 4, device=DEV, generator=gen) * 0.5).to(dtype)
    boxes = torch.cat([torch.rand(n, 2, device=DEV, generator=gen) * 50, 100 + torch.rand(n, 2, device=DEV, generator=gen) * 300], 1)
    assert_shards_equal_whole(lambda shard: BatchedPredictor(head, K, n, t, (img, img), use_graph=use_graph, shard=shard),
                              (feats, boxes), n, t)


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
def test_uint8_view_shards(use_graph):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    n, t, img, views = 37, 8, 128, 2
    model = conv_tracker(7)
    gen = torch.Generator(device=DEV).manual_seed(8)
    vids = [torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=DEV, generator=gen) for h, w in ((150, 200), (97, 131))]
    assert_shards_equal_whole(lambda shard: BatchedPredictor(model.head, K, n, t, (img, img), features_of=model.get_representations,
                                                             use_graph=use_graph, num_views=views, shard=shard), vids, n, t)


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
def test_crop_shards(use_graph):
    """Crop mode: every shard reads its boxes from the full (N, 4) table at the global cursor."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    n, t, img, side = 41, 8, 128, 160
    model = conv_tracker(9)
    gen = torch.Generator(device=DEV).manual_seed(10)
    frames = torch.randint(0, 256, (n, side, side, 3), dtype=torch.uint8, device=DEV, generator=gen)
    wh = torch.randint(40, 150, (n, 2), device=DEV, generator=gen).float()
    xy = (torch.rand(n, 2, device=DEV, generator=gen) * (side - wh)).floor()
    boxes = torch.cat([xy, wh], 1).contiguous()
    assert_shards_equal_whole(lambda shard: BatchedPredictor(model.head, K, n, t, (img, img), features_of=model.get_representations,
                                                             use_graph=use_graph, bboxes=boxes, frame_hw=(side, side), shard=shard),
                              frames, n, t)


# config 3's context head, T = 8 new frames per chunk (sequence_length 12): R = 8 (ceil((N - 12) / 8) + 1)
CONTEXT_CASES = [("r_ge_n", 30), ("r_lt_n", 27), ("r_n_minus_1", 25), ("r_n_minus_1_early_start", 97)]


def context_video(n, seed):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    torch.manual_seed(seed)
    head = HeatmapMHCRNNHead("vits_dino", 384, K, upsampling_factor=1).to(DEV).eval()
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    feats = (torch.randn(n, 384, 16, 16, device=DEV, generator=gen) * 0.5).bfloat16()
    boxes = torch.cat([torch.rand(n, 2, device=DEV, generator=gen) * 30, 200 + torch.rand(n, 2, device=DEV, generator=gen) * 200], 1)
    return head, (feats, boxes)


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("case,n", CONTEXT_CASES, ids=[c[0] for c in CONTEXT_CASES])
def test_context_shards(case, n, use_graph):
    """Halo frames on each side, zero padding after frame N - 1 (the reference reader's), and the edge fill."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor, _context_rows, shard_feed_range

    t = 8
    r = _context_rows(n, t)
    assert {"r_ge_n": r >= n, "r_lt_n": r < n - 1, "r_n_minus_1": r == n - 1}.get(case, r == n - 1)
    if case == "r_n_minus_1_early_start":  # the shard owning row N - 2 starts a frame before its halo
        assert shard_feed_range(n, t, 7, 8, context=True) == (88, 97)
    head, video = context_video(n, 11)
    assert_shards_equal_whole(lambda shard: BatchedPredictor(head, K, n, t, (256, 256), use_graph=use_graph, shard=shard),
                              video, n, t, zero_pad=True)


def test_context_shard_rejects_multiview_and_bad_shard():
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head, _ = context_video(30, 12)
    with pytest.raises(ValueError, match="multiview"):
        BatchedPredictor(head, K, 30, 8, (256, 256), num_views=2, shard=(0, 2))
    with pytest.raises(ValueError, match="shard"):
        BatchedPredictor(head, K, 30, 8, (256, 256), shard=(2, 2))


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
        # a context video whose tail rows (R = 24 < N = 27) hold frame 2 of rank 0, and a feature video
        head, video = context_video(27, 13)
        frame_head = make_head(512, 14)
        gen = torch.Generator(device=DEV).manual_seed(15)
        feats = (torch.randn(29, 512, 4, 4, device=DEV, generator=gen) * 0.5).bfloat16()
        for name, make, vid, n, zero_pad in (
                ("context", lambda s: BatchedPredictor(head, K, 27, 8, (256, 256), shard=s), video, 27, True),
                ("frames", lambda s: BatchedPredictor(frame_head, K, 29, 8, (128, 128), shard=s), feats, 29, False)):
            whole = make((0, 1))
            whole.run(chunks_of(vid, 0, n, 8, zero_pad))
            bp = make((rank, world))
            bp.run(chunks_of(vid, *bp.feed_range, 8, zero_pad))
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
