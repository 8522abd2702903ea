"""Per-layer times of the fp32 head's transposed convolutions (ops.convt_forward_f32 / convt_backward_f32) at the
head shapes of the benchmark configs, 768 frames each:
  config2   ResNet-50 (2048, 12, 12) features, deconvs 512 -> 17 -> 17
  config5   ResNet-50 (2048, 16, 16) features, deconvs 512 -> 17 -> 17
  config3   ViT-S (384, 16, 16) features, one deconv 96 -> 17
  mirror    ResNet-50 (2048, 8, 12) features, deconvs 512 -> 51 -> 51 (mirror-fish, 51 keypoints)
Each layer: forward, wgrad (convt_backward_f32 without the data gradient: the weight and bias gradients and their
zeroing) and bwd (with the data gradient); dgrad = bwd - wgrad.  CUDA events around each call, the L2 flushed before
it (a 256 MB write), median of REPS calls after two warm-up calls.  Useful FLOPs = 2 B Hi Wi Cin Cout 9 per pass
(taps that land outside the map included); "share_3xtf32" = 3 x useful FLOPs / 495 TFLOP/s (dense TF32, H100 SXM data
sheet, not a reached figure) over the time.  A shape the library refuses records the error.  The card's name, power
limit and SM clocks are read in the same call.  Usage:
    python scripts/bench_f32_convt.py [--tree DIR] [out.json]
--tree imports the package from another checkout (to time two builds in one session).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

B = 768
REPS = 12
TF32_DENSE = 495e12
# name: (shuffle, Cin, Hi, Wi, Cout) of each layer, Hi / Wi the conv-input (shuffled) size
LAYERS = {
    "config2_l1": (True, 512, 24, 24, 17),
    "config2_l2": (False, 17, 48, 48, 17),
    "config5_l1": (True, 512, 32, 32, 17),
    "config5_l2": (False, 17, 64, 64, 17),
    "config3_l1": (True, 96, 32, 32, 17),
    "mirror_l1": (True, 512, 16, 24, 51),
    "mirror_l2": (False, 51, 32, 48, 51),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"query": q, "value": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("out", nargs="?", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch

    from lightning_pose_b200 import ops

    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        ms = []
        for i in range(REPS + 2):
            flush.fill_(i & 0xFF)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 2:
                ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    res = {"card": card(), "tree": os.path.abspath(args.tree), "frames": B, "layers": {}}
    for name, (sh, cin, hi, wi, cout) in LAYERS.items():
        x = torch.randn((B, 4 * cin, hi // 2, wi // 2) if sh else (B, cin, hi, wi), device=dev, generator=gen)
        w = torch.randn(cin, cout, 3, 3, device=dev, generator=gen) / (cin * 2.25) ** 0.5
        bias = torch.randn(cout, device=dev, generator=gen)
        g = torch.randn(B, cout, 2 * hi, 2 * wi, device=dev, generator=gen)
        flop = 2.0 * B * hi * wi * cin * cout * 9
        entry = {"shape": [B, cin, hi, wi, cout, int(sh)], "useful_gflop_per_pass": flop / 1e9}
        runs = {"forward": lambda: ops.convt_forward_f32(x, w, bias, sh),
                "wgrad": lambda: ops.convt_backward_f32(x, g, w, sh, need_dx=False),
                "bwd": lambda: ops.convt_backward_f32(x, g, w, sh, need_dx=True)}
        for key, fn in runs.items():
            try:
                entry[f"{key}_ms"] = timed(fn)
            except Exception as e:  # noqa: BLE001 (a refused shape is a result)
                entry[f"{key}_error"] = str(e).splitlines()[0][:200]
        if "bwd_ms" in entry and "wgrad_ms" in entry:
            entry["dgrad_ms"] = entry["bwd_ms"] - entry["wgrad_ms"]
        for key in ("forward", "wgrad", "dgrad"):
            t = entry.get(f"{key}_ms")
            if t:
                entry[f"{key}_useful_tflops"] = flop / (t * 1e-3) / 1e12
                entry[f"{key}_share_3xtf32"] = 3 * flop / TF32_DENSE / (t * 1e-3)
        res["layers"][name] = entry
        print(json.dumps({name: entry}), flush=True)
        del x, g
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
