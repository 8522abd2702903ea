"""A directory of videos of four frame sizes at config 5's shape (resized to 512x512, K = 17, chunks of 96), three ways,
alternated in the same process:

    python scripts/bench_mixed_size_videos.py [--sources stream,resnet50] [--repeats 2] [--out F]

  groups     one list predictor (``n_frames=[...]``, uint8 frames) per frame size;
  per_video  one predictor per video;
  mixed      one list predictor with ``frame_sizes``: every video in one frame stream, one capture.
Workload: 24 videos of 160 to 2,805 frames (log-uniform, seed 0) cycling through 1024x1280, 720x1280, 406x396 and
384x384.  Frame j of video i is frame (7 i + j) mod 96 of a resident pool of 96 frames of its size, gathered per chunk
(per segment in the mixed arm) in every arm.  Sources:
  stream    a stand-in backbone (16x16 average pool, then a 1x1 convolution to 2048 bf16 channels): the predictor's
            own overhead;
  resnet50  a torchvision ResNet-50 (random init, bf16, channels-last) as ``features_of``.
Per arm (best of the repeats by total_ms):
  total_ms  wall time of every construction and feed, to the last table on the device;
  feed_ms   the same without each predictor's first feed (its capture, two eager warm-up chunks and one replay);
  ms_per_chunk  feed_ms over the chunks it covers;
  backbone_frames  frames every feed pushes through the backbone (padding included); warmup_frames those of the
            captures' warm-up chunks;  launches_per_chunk  kernel nodes of the chunk graph.
Each video's table (SHA-256 of its rows) is compared between the arms.  ``kernel``: one chunk of 24 frames of each size,
``lpb_frames_normalize_ragged`` (one launch) against ``lpb_frames_normalize`` (one launch per size) on the same frames,
bf16 channels-last, CUDA events around each call with the L2 flushed before it; and a one-size chunk (96 frames of
1024x1280) through both, the cost of the per-frame lookup.  The card, its power limit and SM clocks are read in the same
run.  One JSON object on stdout (and in --out).  Changes no device setting.
"""
import argparse
import hashlib
import json
import math
import os
import random
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402
from lightning_pose_b200.utils.predictions import BatchedPredictor, _chunk_segments, _video_starts  # noqa: E402

K, T, IMG, POOL = 17, 96, 512, 96
SIZES = [(1024, 1280), (720, 1280), (406, 396), (384, 384)]


def card(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if out else {"nvidia_smi": "unavailable"}


def workload() -> tuple[list[int], list[tuple[int, int]]]:
    rng = random.Random(0)
    lengths = [int(round(math.exp(rng.uniform(math.log(160), math.log(2805))))) for _ in range(24)]
    return lengths, [SIZES[i % len(SIZES)] for i in range(len(lengths))]


def source(name: str, dev):
    """(head, features_of on normalised (T, h, w, 3) bf16 channels-last images)."""
    torch.manual_seed(0)
    head = HeatmapHead("resnet50", 2048, K).to(dev).eval()
    if name == "stream":
        proj = torch.nn.Conv2d(3, 2048, 1).to(dev, torch.bfloat16).eval()
        return head, lambda x: proj(F.avg_pool2d(x.permute(0, 3, 1, 2), 32))
    import torchvision

    trunk = torch.nn.Sequential(*list(torchvision.models.resnet50().children())[:-2])
    trunk = trunk.to(dev, torch.bfloat16).to(memory_format=torch.channels_last).eval()
    return head, lambda x: trunk(x.permute(0, 3, 1, 2))


class Stream:
    """The frames of a list of videos (indices into the workload) back to back, gathered from the resident pools."""

    def __init__(self, videos, lengths, sizes, pools, dev):
        self.videos, self.lengths = videos, [lengths[v] for v in videos]
        self.sizes, self.pools = [sizes[v] for v in videos], pools
        self.starts = _video_starts(self.lengths)
        self.ar = torch.arange(T, device=dev)

    def segments(self, row: int) -> list[torch.Tensor]:
        out, r = [], row
        for i, t in _chunk_segments(row, T, self.starts):
            idx = torch.remainder(self.ar[:t] + (7 * self.videos[i] + r - self.starts[i]), POOL)
            out.append(self.pools[self.sizes[i]].index_select(0, idx))
            r += t
        return out

    def chunk(self, row: int, ragged: bool):
        segs = self.segments(row)
        return segs if ragged else [segs[0] if len(segs) == 1 else torch.cat(segs)]


def predict(head, features_of, stream: Stream, ragged: bool, dev):
    """One predictor over ``stream`` -> (predictor, total ms, feed ms without the first feed)."""
    t0 = time.perf_counter()
    n = stream.lengths if len(stream.lengths) > 1 or ragged else stream.lengths[0]
    kw = {"frame_sizes": stream.sizes} if ragged else {}
    bp = BatchedPredictor(head, K, n, T, (IMG, IMG), features_of=features_of, crop_dtype=torch.bfloat16,
                          crop_channels_last=True, **kw)
    bp.feed(stream.chunk(0, ragged))
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    for j in range(1, bp.n_chunks):
        bp.feed(stream.chunk(j * T, ragged))
    torch.cuda.synchronize(dev)
    t2 = time.perf_counter()
    return bp, (t2 - t0) * 1e3, (t2 - t1) * 1e3


def arm(name, head, features_of, lengths, sizes, pools, dev):
    """-> (stats, per-video tables in workload order)."""
    if name == "mixed":
        groups = [list(range(len(lengths)))]
    elif name == "groups":
        groups = [[v for v in range(len(lengths)) if sizes[v] == s] for s in SIZES]
    else:
        groups = [[v] for v in range(len(lengths))]
    t0 = time.perf_counter()
    feed_ms, fed, timed, warm, launches, tables = 0.0, 0, 0, 0, None, {}
    for g in groups:
        bp, _, ms = predict(head, features_of, Stream(g, lengths, sizes, pools, dev), name == "mixed", dev)
        feed_ms += ms
        fed += bp.n_chunks * T
        timed += bp.n_chunks - 1
        warm += 2 * T
        launches = bp.launches_per_chunk
        tables.update(zip(g, bp.video_tables()))
    total_ms = (time.perf_counter() - t0) * 1e3
    return {"predictors": len(groups), "feed_ms": feed_ms, "total_ms": total_ms, "ms_per_chunk": feed_ms / timed,
            "backbone_frames": fed,
            "warmup_frames": warm, "launches_per_chunk": launches}, [tables[v] for v in range(len(lengths))]


def digests(tables) -> list[str]:
    return [hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest() for t in tables]


def time_calls(fn, flush, iters=30) -> float:
    """Mean ms of ``fn`` with the L2 flushed (a 256 MB write) before each call, CUDA events around the call."""
    fn()
    times = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return sum(times) / len(times)


def kernel_bench(pools, dev) -> dict:
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {}
    for name, per_size in (("four_sizes", [(s, T // 4) for s in SIZES]), ("one_size", [(SIZES[0], T)])):
        frames = [pools[s][:n] for s, n in per_size]
        lengths, sizes = [n for _, n in per_size], [s for s, _ in per_size]
        host = ops.ragged_videos(lengths, sizes)
        table, slot = host.to(dev), ops.ragged_slot_bytes(sizes)
        arena = torch.zeros(T * slot, dtype=torch.uint8, device=dev)
        slots, f0 = arena.view(T, slot), 0
        for x in frames:
            slots[f0 : f0 + x.shape[0], : x[0].numel()].copy_(x.reshape(x.shape[0], -1))
            f0 += x.shape[0]
        cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        ragged = lambda: ops.frames_normalize_ragged(arena, slot, T, cursor, table, host, (IMG, IMG), channels_last=True,
                                                     dtype=torch.bfloat16)
        plain = lambda: [ops.frames_normalize(x, (IMG, IMG), channels_last=True, dtype=torch.bfloat16) for x in frames]
        got, want = ragged()[0], torch.cat(plain())
        read = sum(x.numel() for x in frames)
        written = T * IMG * IMG * 3 * 2
        ms_r, ms_p = time_calls(ragged, flush), time_calls(plain, flush)
        out[name] = {"frames": lengths, "sizes": sizes, "bytes_read": read, "bytes_written": written,
                     "ragged_ms": ms_r, "normalize_ms": ms_p, "launches_normalize": len(frames),
                     "ragged_gbps": (read + written) / ms_r / 1e6, "normalize_gbps": (read + written) / ms_p / 1e6,
                     "arena_copy_bytes": read, "bit_identical": bool(torch.equal(got.view(torch.int16), want.view(torch.int16)))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", default="stream,resnet50")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lengths, sizes = workload()
    gen = torch.Generator(device=dev).manual_seed(1)
    pools = {s: torch.randint(0, 256, (POOL, *s, 3), dtype=torch.uint8, device=dev, generator=gen) for s in SIZES}
    res = {"card": card(0), "chunk": T, "keypoints": K, "image": IMG, "repeats": args.repeats, "videos": len(lengths),
           "frames": sum(lengths), "lengths": lengths, "sizes": sizes, "runs": {}}
    with torch.no_grad():
        res["kernel"] = kernel_bench(pools, dev)
        print(json.dumps({"kernel": res["kernel"]}), file=sys.stderr, flush=True)
        for src in args.sources.split(","):
            head, features_of = source(src, dev)
            arms = {"groups": [], "per_video": [], "mixed": []}
            same = True
            for _ in range(args.repeats):  # alternate the arms
                sha = {}
                for name in arms:
                    stats, tables = arm(name, head, features_of, lengths, sizes, pools, dev)
                    arms[name].append(stats)
                    sha[name] = digests(tables)
                    del tables
                same &= sha["groups"] == sha["per_video"] == sha["mixed"]
            best = {a: min(r, key=lambda x: x["total_ms"]) for a, r in arms.items()}
            res["runs"][src] = {
                **best,
                "feed_ms_all": {a: [round(x["feed_ms"], 1) for x in r] for a, r in arms.items()},
                "total_ms_all": {a: [round(x["total_ms"], 1) for x in r] for a, r in arms.items()},
                "speedup_total_vs_groups": best["groups"]["total_ms"] / best["mixed"]["total_ms"],
                "speedup_total_vs_per_video": best["per_video"]["total_ms"] / best["mixed"]["total_ms"],
                "per_video_sha256_equal": bool(same)}
            print(json.dumps({src: res["runs"][src]}), file=sys.stderr, flush=True)
            del head, features_of
            torch.cuda.empty_cache()
    res["card_after"] = card(0)
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
