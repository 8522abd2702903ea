"""A directory of videos at config 5's shape (512x512, K = 17, chunks of 96): one-video ``BatchedPredictor``s in a loop
against one list predictor (``n_frames=[N_0, N_1, ...]``), alternated in the same process.

    python scripts/bench_multi_video.py [--workloads short,mixed] [--sources head,e2e] [--repeats 2] [--out F]

Workloads: ``short`` 200 videos of 300 frames; ``mixed`` 24 lengths drawn log-uniformly from 60 to 3,000 frames
(seed 0).  Sources, as in scripts/bench_sharded_predict.py:
  head  streamed bf16 (., 2048, 16, 16) features (a resident pool of 4 chunks): the predictor's own overhead;
  e2e   uint8 512x512 frames (a resident pool of 2 chunks) through ``frames_normalize`` and a torchvision ResNet-50
        (random init, bf16, channels-last) as ``features_of``.
Frame f of the concatenated stream is pool frame f mod P in both arms (one gather per chunk, in both).  Per arm:
  feed_ms   wall time from the first timed feed to the last table on the device (the loop: the sum over videos);
  total_ms  wall time including every construction and capture (the capture is the first feed, which also runs the
            two eager warm-up chunks; its replay is then rewound and the timed run starts at frame 0);
  backbone_frames  frames pushed through the backbone by the timed feeds (padding included), and warmup_frames by the
            captures;  launches_per_chunk  kernel nodes of the chunk graph.
Each video's table (SHA-256 of its rows) is compared between the arms.  The card, its power limit and SM clocks are read
in the same run.  One JSON object on stdout (and in --out).  Changes no device setting.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_sharded_predict import e2e_source, head_source  # noqa: E402
from lightning_pose_b200.utils.predictions import BatchedPredictor  # noqa: E402

K, T, IMG = 17, 96, 512


def card(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if out else {"nvidia_smi": "unavailable"}


def workload(name: str) -> list[int]:
    if name == "short":
        return [300] * 200
    rng = random.Random(0)
    return [int(round(math.exp(rng.uniform(math.log(60), math.log(3000))))) for _ in range(24)]


def run_arm(head, features_of, pool, start, n_frames, dev, ar):
    """One predictor over ``n_frames`` (an int: one video starting at stream frame ``start``; a list from frame 0)
    -> (predictor, total ms, feed ms)."""
    t0 = time.perf_counter()
    bp = BatchedPredictor(head, K, n_frames, T, (IMG, IMG), features_of=features_of)
    chunk = lambda j: pool.index_select(0, torch.remainder(ar + (start + j * T), pool.shape[0]))
    bp.feed(chunk(0))  # capture (two eager warm-up chunks) + one replay, then rewind
    bp.cursor.fill_(bp.feed_range[0])
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    for j in range(bp.n_chunks):
        bp.feed(chunk(j))
    torch.cuda.synchronize(dev)
    t2 = time.perf_counter()
    return bp, (t2 - t0) * 1e3, (t2 - t1) * 1e3


def loop_arm(head, features_of, pool, lengths, dev, ar):
    t0 = time.perf_counter()
    feed_ms, tables, fed, launches = 0.0, [], 0, None
    row0 = 0
    for n in lengths:
        bp, _, ms = run_arm(head, features_of, pool, row0, n, dev, ar)
        feed_ms += ms
        tables.append(bp.table)
        fed += bp.n_chunks * T
        launches = bp.launches_per_chunk
        row0 += n
    total_ms = (time.perf_counter() - t0) * 1e3
    return {"feed_ms": feed_ms, "total_ms": total_ms, "backbone_frames": fed, "warmup_frames": 3 * T * len(lengths),
            "launches_per_chunk": launches}, tables


def list_arm(head, features_of, pool, lengths, dev, ar):
    bp, total_ms, feed_ms = run_arm(head, features_of, pool, 0, lengths, dev, ar)
    return {"feed_ms": feed_ms, "total_ms": total_ms, "backbone_frames": bp.n_chunks * T, "warmup_frames": 3 * T,
            "launches_per_chunk": bp.launches_per_chunk}, bp.video_tables()


def digests(tables) -> list[str]:
    return [hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest() for t in tables]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="short,mixed")
    ap.add_argument("--sources", default="head,e2e")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ar = torch.arange(T, device=dev)
    res = {"card": card(0), "chunk": T, "keypoints": K, "image": IMG, "repeats": args.repeats, "runs": {}}
    for src in args.sources.split(","):
        head, features_of, pool = {"head": head_source, "e2e": e2e_source}[src](dev)
        pool = torch.cat(pool)
        with torch.no_grad():
            for wl in args.workloads.split(","):
                lengths = workload(wl)
                arms = {"loop": [], "list": []}
                same = True
                for _ in range(args.repeats):  # alternate the arms
                    loop, loop_tables = loop_arm(head, features_of, pool, lengths, dev, ar)
                    lst, list_tables = list_arm(head, features_of, pool, lengths, dev, ar)
                    same &= digests(loop_tables) == digests(list_tables)
                    arms["loop"].append(loop)
                    arms["list"].append(lst)
                    del loop_tables, list_tables
                best = {a: min(r, key=lambda x: x["total_ms"]) for a, r in arms.items()}
                res["runs"][f"{src}/{wl}"] = {
                    "videos": len(lengths), "frames": sum(lengths), "min_len": min(lengths), "max_len": max(lengths),
                    "loop": best["loop"], "list": best["list"],
                    "feed_ms_all": {a: [round(x["feed_ms"], 1) for x in r] for a, r in arms.items()},
                    "total_ms_all": {a: [round(x["total_ms"], 1) for x in r] for a, r in arms.items()},
                    "speedup_total": best["loop"]["total_ms"] / best["list"]["total_ms"],
                    "speedup_feed": min(x["feed_ms"] for x in arms["loop"]) / min(x["feed_ms"] for x in arms["list"]),
                    "per_video_sha256_equal": bool(same)}
                print(json.dumps({f"{src}/{wl}": res["runs"][f"{src}/{wl}"]}), file=sys.stderr, flush=True)
        del head, features_of, pool
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
