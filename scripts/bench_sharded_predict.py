"""Config 5 inference (BASELINE.json: a 100k-frame 512x512 video, batched soft-argmax) on every GPU of a box: each rank
predicts a contiguous shard of the video with ``BatchedPredictor(..., shard=(rank, world))`` and one ``gather()`` puts
the (N, 3K) table on every rank.

    torchrun --nproc-per-node G scripts/bench_sharded_predict.py [--frames N] [--sources head,e2e]

Two sources, 17 keypoints, chunks of 96 frames, graph replay:
  head  streamed bf16 (., 2048, 16, 16) features: the trained-like response of ``bench.make_problem`` at the 512x512
        geometry (the ``cfg5_batched_inference_*`` entries of scripts/bench_configs.py), a resident pool of 4 chunks
        per rank cycled through;
  e2e   device-synthesised uint8 512x512 frames (a resident pool of 2 chunks) through ``frames_normalize`` and a
        torchvision ResNet-50 (random init, bf16, channels-last) as ``features_of``.
Global frame f is pool frame f mod P (P frames in the pool) at every G: each rank starts the pool at its first frame,
so the table does not depend on G.  Per source: rank 0 first predicts the whole video alone (shard (0, 1)) while the other ranks wait, which gives the
G = 1 time and table of the same session; then every rank predicts its shard.  A rank's time runs from a common start
(barrier + synchronise) to the end of its ``gather()``, on CUDA events; frames/s = N / the slowest rank's time.  The
table's SHA-256 makes runs at different G comparable bit for bit.  One JSON object goes to stdout on rank 0 (and to
--out if given).  Needs one GPU per rank; changes no device setting.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402
from lightning_pose_b200.utils.predictions import BatchedPredictor, frame_range_for_rank  # noqa: E402

K, T, IMG = 17, 96, 512


def card(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if out else {"nvidia_smi": "unavailable"}


def head_source(dev):
    """(head, features_of, pool): the trained-like config-5 head and 4 resident chunks of bf16 features."""
    bench.FEAT_HW, bench.HM, bench.IMG = 16, 128, IMG
    prob = bench.make_problem(8, seed=7, device=dev, regime="trained")  # 8 clips x 48 = 384 frames = 4 chunks
    bench.FEAT_HW, bench.HM, bench.IMG = 12, 96, 384
    head = HeatmapHead("resnet50", 2048, K)
    d1, d2 = list(head.upsampling_layers)[1:]
    with torch.no_grad():
        w1, b1, w2, b2 = prob["head_params"]
        d1.weight.copy_(w1), d1.bias.copy_(b1), d2.weight.copy_(w2), d2.bias.copy_(b2)
    feats = prob["feats"].bfloat16().to(dev)
    return head.to(dev).eval(), None, [feats[i * T : (i + 1) * T].contiguous() for i in range(4)]


def e2e_source(dev):
    """(head, features_of, pool): ResNet-50 on normalised uint8 frames, 2 resident chunks of synthetic frames."""
    import torchvision

    torch.manual_seed(0)
    net = torchvision.models.resnet50()
    trunk = torch.nn.Sequential(*list(net.children())[:-2]).to(dev, torch.bfloat16).to(memory_format=torch.channels_last).eval()
    head = HeatmapHead("resnet50", 2048, K).to(dev).eval()

    def features_of(u8):
        return trunk(ops.frames_normalize(u8, size=(IMG, IMG), channels_last=True, dtype=torch.bfloat16).permute(0, 3, 1, 2))

    gen = torch.Generator(device=dev).manual_seed(1)
    return head, features_of, [torch.randint(0, 256, (T, IMG, IMG, 3), dtype=torch.uint8, device=dev, generator=gen) for _ in range(2)]


def predict(head, features_of, pool, n, shard, dev):
    """Warm (capture, one gather), then the timed run: (ms to the end of gather, gather ms, table)."""
    bp = BatchedPredictor(head, K, n, T, (IMG, IMG), features_of=features_of, shard=shard)
    lo, hi = bp.feed_range
    frames = torch.cat(pool)  # the rank's j-th chunk holds global frames lo + j T ...: pool frames from lo mod P on
    pool = list(torch.roll(frames, -(lo % frames.shape[0]), 0).split(T))
    del frames
    if lo < hi:
        bp.feed(pool[0])
        bp.cursor.fill_(lo)
    bp.gather()
    torch.cuda.synchronize(dev)
    if shard[1] > 1:
        dist.barrier()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    for j in range(-(-(hi - lo) // T)):
        bp.feed(pool[j % len(pool)])
    e1.record()
    table = bp.gather()
    e2.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e2), e1.elapsed_time(e2), table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100_000)
    ap.add_argument("--sources", default="head,e2e")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rank, world, local = (int(os.environ.get(v, d)) for v, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    if not torch.cuda.is_available() or torch.cuda.device_count() <= local:
        raise SystemExit(f"rank {rank}: needs one CUDA device per rank (local rank {local}, {torch.cuda.device_count()} devices)")
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        n = args.frames
        res = {"G": world, "frames": n, "chunk": T, "keypoints": K, "image": IMG, "sources": {}}
        for name in args.sources.split(","):
            head, features_of, pool = {"head": head_source, "e2e": e2e_source}[name](dev)
            one = None
            if rank == 0 and world > 1:
                ms, _, table = predict(head, features_of, pool, n, (0, 1), dev)
                one = {"ms": ms, "frames_per_s": n / ms * 1e3, "sha256": hashlib.sha256(table.cpu().numpy().tobytes()).hexdigest()}
            dist.barrier()
            ms, gather_ms, table = predict(head, features_of, pool, n, (rank, world), dev)
            mine = {"rank": rank, "rows": list(frame_range_for_rank(n, rank, world)), "ms": ms, "gather_ms": gather_ms,
                    "sha256": hashlib.sha256(table.cpu().numpy().tobytes()).hexdigest(), "card": card(local)}
            if world == 1:  # the run is its own G = 1 reference
                one = {"ms": ms, "frames_per_s": n / ms * 1e3, "sha256": mine["sha256"]}
            ranks = [None] * world
            dist.all_gather_object(ranks, mine)
            slowest = max(r["ms"] for r in ranks)
            if rank == 0:
                fps = n / slowest * 1e3
                res["sources"][name] = {
                    "G1_same_session": one, "ranks": ranks, "ms_slowest": slowest, "frames_per_s": fps,
                    "gather_ms_max": max(r["gather_ms"] for r in ranks),
                    "scaling_efficiency_vs_G1": fps / (world * one["frames_per_s"]),
                    "sha256_all_ranks_equal": len({r["sha256"] for r in ranks}) == 1,
                    "sha256_equals_G1": all(r["sha256"] == one["sha256"] for r in ranks)}
            del head, features_of, pool, table
            torch.cuda.empty_cache()
        if rank == 0:
            line = json.dumps(res)
            print(line, flush=True)
            if args.out:
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "w") as f:
                    f.write(line + "\n")
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
