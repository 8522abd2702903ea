"""Three-deconv heads (downsample_factor 1 on a ResNet-50) on the 16-bit tensor-core route against the fp32 route they took
before it (``ops.head_forward_f32`` / ``convt_backward_f32`` on the features up-cast to fp32), and config 2's two-deconv
head as a control.

Shapes: (256, 2048, 12, 12) features -> 17 x 192 x 192 heatmaps (384 x 384 images) and (96, 2048, 16, 16) -> 17 x 256 x 256
(512 x 512 images); the control is (256, 2048, 12, 12) -> 17 x 96 x 96 with two deconvs.  bf16 features throughout.
Operations, each timed per call with CUDA events, the L2 flushed before each call (a 256 MB write), median and range of
REPS calls after two warm-up calls, the routes alternated call by call in one process:
  forward          HeatmapHead.forward without autograd
  forward_decode   forward_with_keypoints without autograd (head + soft-argmax decode)
  train_dense      forward with autograd, then the backward of a dense heatmap gradient (made before the timed window)
  train_targets    forward with autograd, the keypoint-target heatmap MSE, backward
  train_decode     forward_with_keypoints with autograd, the keypoint-target heatmap MSE plus a keypoint loss (the decode
                   windows), backward
An operation a route cannot run (the decode's shared-memory tile, the fp32 plane softmax's plane size) records the
library's error instead of a time.
The fp32 route is selected by making ``ops.head3_supported`` refuse every head, which is the route every three-deconv
head took before the 16-bit kernels served it.  The card's name, power limit and SM clocks are read in the same call.
Usage:
    python scripts/bench_three_deconv.py [out.json]
"""
from __future__ import annotations

import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402

REPS = 15
K = 17
SHAPES = {"3d_256x2048x12x12": (256, 2048, 12, 12, 1), "3d_96x2048x16x16": (96, 2048, 16, 16, 1), "control_2d_256x2048x12x12": (256, 2048, 12, 12, 2)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"nvidia_smi": {"query": q, "value": out}, "torch_name": torch.cuda.get_device_name(0)}


HEAD3_SUPPORTED = ops.head3_supported


def select_route(fp32: bool):
    """fp32: three-deconv heads take the fp32 kernels (the route before the 16-bit kernels covered them)."""
    ops.head3_supported = (lambda *a, **k: False) if fp32 else HEAD3_SUPPORTED


def main():
    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    results = {"card": card(), "reps": REPS, "rows": {}}

    for name, (b, c, h, w, ds) in SHAPES.items():
        torch.manual_seed(0)
        head = HeatmapHead("resnet50", c, K, downsample_factor=ds).to(dev)
        for layer in list(head.upsampling_layers)[1:]:
            torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
        gen = torch.Generator(device=dev).manual_seed(1)
        feats = (torch.randn(b, c, h, w, device=dev, generator=gen) * 0.5).bfloat16()
        up = 2 ** (5 - ds)  # heatmap size / feature size
        img = float(2 ** ds * up * h)
        g_hm = torch.randn(b, K, up * h, up * w, device=dev, generator=gen) * 1e-3
        g_kp = torch.randn(b, 2 * K, device=dev, generator=gen)
        kp = torch.rand(b, K, 2, device=dev, generator=gen) * img
        vis = torch.full((b, K), 2, dtype=torch.int32, device=dev)

        def forward():
            with torch.no_grad():
                head(feats)

        def forward_decode():
            with torch.no_grad():
                head.forward_with_keypoints(feats)

        def train_dense():
            f = feats.detach().requires_grad_(True)
            head(f).backward(g_hm)

        def train_targets():
            f = feats.detach().requires_grad_(True)
            ops.heatmap_mse_from_keypoints(kp, head(f), img, img, visibility=vis).backward()

        def train_decode():
            f = feats.detach().requires_grad_(True)
            hm, kpp, _ = head.forward_with_keypoints(f)
            loss = ops.heatmap_mse_from_keypoints(kp, hm, img, img, visibility=vis) + (kpp * g_kp).sum()
            loss.backward()

        ops_ = {"forward": forward, "forward_decode": forward_decode, "train_dense": train_dense, "train_targets": train_targets,
                "train_decode": train_decode}
        routes = {"16bit": False} if ds == 2 else {"16bit": False, "fp32": True}
        times = {(o, r): [] for o in ops_ for r in routes}
        errors = {}
        for i in range(REPS + 2):
            for oname, fn in ops_.items():
                for rname, fp32 in routes.items():
                    if (oname, rname) in errors:
                        continue
                    flush.fill_(i & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    select_route(fp32)
                    try:
                        e0.record()
                        fn()
                        e1.record()
                        torch.cuda.synchronize()
                    except Exception as e:  # a route that fails records its error instead of a time
                        errors[(oname, rname)] = repr(e)[:300]
                        continue
                    finally:
                        select_route(False)
                    if i >= 2:
                        times[(oname, rname)].append(e0.elapsed_time(e1))
                    head.zero_grad(set_to_none=True)
        row = {}
        for (oname, rname), ms in times.items():
            key = f"{oname}/{rname}"
            if (oname, rname) in errors:
                row[key] = {"error": errors[(oname, rname)]}
            else:
                row[key] = {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "n": len(ms)}
        results["rows"][name] = row
        print(name, json.dumps(row), flush=True)
        del feats, g_hm
        torch.cuda.empty_cache()
    results["card_after"] = card()
    text = json.dumps(results, indent=1)
    print(text)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
