#!/usr/bin/env python
"""What channels-last features cost the heatmap head, against NCHW features and against copying them to NCHW first.

Per shape and operation, three variants alternate inside one process: NCHW features (nchw), channels-last features read
in place (nhwc), and channels-last features copied to NCHW before the head and, in training, their gradient copied back
(copy: what a channels-last producer paid before the head read them in place).  L2 is flushed before each repetition;
median and min-max of the repetitions in microseconds, from CUDA events.  A second pass profiles the channels-last
shuffle and data-gradient kernels alone against their bytes models (share of the H100 SXM data sheet's 3.35 TB/s; both
are bandwidth-bound: they move every feature byte once and compute nothing or little).  Needs a GPU; prints one JSON
line per measurement."""
import argparse
import ctypes
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402

SHAPES = {  # name: (frames, C, H, W, backbone, dtype)
    "config2 resnet50 768x(2048,12,12)": (768, 2048, 12, 12, "resnet50", torch.bfloat16),
    "config3 vit-s 768x(384,16,16)": (768, 384, 16, 16, "vits_dino", torch.bfloat16),
    "config3 vit-s fp32": (768, 384, 16, 16, "vits_dino", torch.float32),
    "config4 chunk 384x(384,24,24)": (384, 384, 24, 24, "vits_dino", torch.bfloat16),
    "config5 chunk 256x(2048,12,12)": (256, 2048, 12, 12, "resnet50", torch.bfloat16),
    "mirror-fish 96x(2048,8,12)": (96, 2048, 8, 12, "resnet50", torch.bfloat16),
}
HBM = 3.35e12


def timed(fn, reps, flush):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps):
        flush.zero_()
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        out.append(start.elapsed_time(stop) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every batch size")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_channels_last: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    for name, (b, c, h, w, arch, dtype) in SHAPES.items():
        b = max(1, int(b * args.scale))
        torch.manual_seed(0)
        head = HeatmapHead(arch, c, 17).cuda()
        x = (torch.randn(b, c, h, w, device="cuda") * 0.5).to(dtype)
        xc = x.contiguous(memory_format=torch.channels_last)
        gout = torch.randn_like(head(x[:1])).expand(b, -1, -1, -1).contiguous()

        def train(feat, copy):
            leaf = feat.detach().requires_grad_(True)
            (head(leaf.contiguous() if copy else leaf) * gout).sum().backward()  # the copy's backward returns the gradient to nhwc
            return leaf.grad

        ops_ = {
            "forward": lambda f, copy: head(f.contiguous() if copy else f),
            "forward+decode": lambda f, copy: head.forward_with_keypoints(f.contiguous() if copy else f),
            "train fwd+bwd": train,
        }
        variants = {"nchw": (x, False), "nhwc": (xc, False), "copy": (xc, True)}
        for op, fn in ops_.items():
            grad = op.startswith("train")
            times = {v: [] for v in variants}
            with torch.set_grad_enabled(grad):
                for f, copy in variants.values():  # warm up every variant of the shape
                    fn(f, copy)
                for _ in range(args.reps):  # alternate
                    for v, (f, copy) in variants.items():
                        times[v] += timed(lambda: fn(f, copy), 1, flush)
            print(json.dumps({"shape": name, "op": op, **{v: {"median_us": round(statistics.median(t), 1), "min_us": round(min(t), 1),
                                                                "max_us": round(max(t), 1)} for v, t in times.items()}}), flush=True)
        if dtype == torch.bfloat16:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    flush.zero_()
                    train(xc, False)
                torch.cuda.synchronize()
            nbytes = ctypes.c_size_t(0)
            ops.check(ops.lib.lpb_head_bf16_saved_bytes(b, c, h, w, ctypes.byref(nbytes)))
            feat_bytes = b * c * h * w * 2
            g1_bytes = nbytes.value // (c // 32) * 10  # the gradient operand: 10 K-chunks per frame in the same row layout
            models = {"rows_shuffle_nhwc_kernel": feat_bytes + nbytes.value, "b3a_dgrad_kernel": g1_bytes + feat_bytes}
            for kname, model in models.items():
                ts = [e.device_time_total / max(1, e.count) for e in prof.key_averages() if kname in e.key]
                if ts:
                    us = sum(ts) / len(ts)
                    print(json.dumps({"shape": name, "kernel": kname, "mean_us": round(us, 1), "model_bytes": model,
                                      "share_of_3.35TB/s": round(model / (us * 1e-6) / HBM, 3), "bound": "HBM bandwidth"}), flush=True)


if __name__ == "__main__":
    main()
