"""Curriculum patch masking on the device: kernel times, the reference's loop on the same card, and the multi-view
transformer's labeled step with masking off and on.

Workloads (fp32 and bf16 images, 3 channels):
  config4   8 examples x 4 views x 384 x 384 (576 patches per view), BASELINE config 4
  v6_256    8 examples x 6 views x 256 x 256 (256 patches per view)
Masking at the curriculum's final ratio 0.5 (step past final_step): half the patches of every view.

Rows:
  select          lpb_patch_mask_select alone (one CTA per (example, view))
  apply           lpb_patch_mask_apply alone, with its share of HBM bandwidth on its bytes model (every image byte read
                  once and written once; the mask's B * V * P * 4 bytes are left out)
  select_apply    PatchMasker.apply_patch_masking with a device step: both launches and the output allocations
  reference_loop  a restatement of PatchMasker.apply_patch_masking (lightning_pose/callbacks.py:318-401) on the same card:
                  per (example, view) a torch.Generator on the device, its manual_seed, randperm, the mask scatter and one
                  slice assignment per masked patch, whose bounds are 0-d device tensors (host reads through __index__)
  step_*          HeatmapTrackerMultiviewTransformer.training_step + the gradients of the head and view embeddings
                  (no optimizer), config 4, the stand-in transformer of scripts/bench_configs.py, K = 17, heatmap MSE:
                  masking off, on (eager), on (CUDA-graph replay of the whole step)

CUDA events around each call with the L2 flushed before it (a 256 MB write); median and min-max of REPS calls after two
warm-up calls (the reference loop: 3 calls after one).  The card's name, power limit and SM clock are read in the same
call.  Usage: python scripts/bench_patch_mask.py [out.json] (one JSON line is printed; also written to out.json when
given).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REPS = 20
HBM_GBS = 3350.0  # H100 SXM data sheet
WORKLOADS = {"config4": (8, 4, 384, 384), "v6_256": (8, 6, 256, 256)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"query": q, "value": out}


def main():
    import torch

    from lightning_pose_b200 import ops
    from lightning_pose_b200.callbacks import PatchMasker
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn, reps=REPS, warmup=2):
        for _ in range(warmup):
            fn()
        ts = []
        for _ in range(reps):
            flush.random_(generator=gen)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return {"median_ms": round(float(np.median(ts)), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}

    cfg = {"init_step": 700, "final_step": 5000, "init_ratio": 0.1, "final_ratio": 0.5}
    masker = PatchMasker(cfg, patch_seed=0)
    step_value = 6000  # past final_step: ratio 0.5

    def reference_loop(images, training_step):
        """PatchMasker.apply_patch_masking of callbacks.py:318-401, restated (same operations, same order)."""
        batch_size, num_views, _, height, width = images.shape
        patch_size = 16
        num_patches_h, num_patches_w = height // patch_size, width // patch_size
        progress = min((training_step - cfg["init_step"]) / (cfg["final_step"] - cfg["init_step"]), 1.0)
        mask_ratio = cfg["init_ratio"] + progress * (cfg["final_ratio"] - cfg["init_ratio"])
        total = num_patches_h * num_patches_w
        m = int(mask_ratio * total)
        patch_mask = torch.ones(batch_size, num_views, total, device=images.device)
        masked = images.clone()
        for b in range(batch_size):
            for v in range(num_views):
                g = torch.Generator(device=images.device)
                g.manual_seed(0 + training_step + b * 1000 + v * 100)
                idx = torch.randperm(total, device=images.device, generator=g)[:m]
                patch_mask[b, v, idx] = 0
                for p in idx:
                    ph = (p // num_patches_w) * patch_size
                    pw = (p % num_patches_w) * patch_size
                    masked[b, v, :, ph:ph + patch_size, pw:pw + patch_size] = 0
        return masked, patch_mask

    res = {"card_before": card(), "reps": REPS, "hbm_gbs_datasheet": HBM_GBS, "curriculum": cfg, "step": step_value, "kernels": {}}
    step = torch.full((1,), step_value, dtype=torch.int64, device=dev)
    for name, (b, v, h, w) in WORKLOADS.items():
        row = {}
        for dt_name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            x = torch.randn(b, v, 3, h, w, device=dev, generator=gen).to(dt)
            mask = ops.patch_mask_select(x, step, 0, **{k: cfg[k] for k in ("init_step", "final_step", "init_ratio", "final_ratio")})
            nbytes = 2 * x.numel() * x.element_size()
            t_apply = timed(lambda: ops.patch_mask_apply(x, mask))
            r = {
                "patches_per_view": mask.shape[-1], "masked_per_view": int((mask[0, 0] == 0).sum()),
                "select": timed(lambda: ops.patch_mask_select(x, step, 0, cfg["init_step"], cfg["final_step"], cfg["init_ratio"], cfg["final_ratio"])),
                "apply": {**t_apply, "bytes_model": nbytes, "gbs": round(nbytes / t_apply["median_ms"] / 1e6, 1),
                          "frac_hbm": round(nbytes / t_apply["median_ms"] / 1e6 / HBM_GBS, 3)},
                "select_apply": timed(lambda: masker.apply_patch_masking(x, training_step=step)),
            }
            if dt == torch.float32 or name == "config4":
                r["reference_loop"] = timed(lambda: reference_loop(x, step_value), reps=3, warmup=1)
            row[dt_name] = r
        res["kernels"][name] = row

    # ---- the labeled step at config 4 ------------------------------------------------------------------------------------
    class Patch(torch.nn.Module):  # stand-in ViT patch embedding (scripts/bench_configs.py)
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Conv2d(3, 384, 16, stride=16)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class Mix(torch.nn.Module):  # stand-in encoder: one token-mixing linear layer
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(384, 384)

        def forward(self, t):
            return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()

    b, v, h, w = WORKLOADS["config4"]
    k = 17
    torch.manual_seed(4)
    kp = torch.rand(b, v * k * 2, device=dev, generator=gen) * h
    images = torch.randn(b, v, 3, h, w, device=dev, generator=gen)
    batch = {"images": images, "keypoints": kp.clone(), "heatmaps": ops.generate_heatmaps(kp.reshape(b, v * k, 2), h, w, (96, 96)),
             "bbox": torch.tensor([[0.0, 0.0, float(h), float(w)] * v], device=dev).repeat(b, 1), "is_multiview": True}
    steps = {}
    for mode in ("off", "on_eager", "on_graph"):
        tr = HeatmapTrackerMultiviewTransformer(k, v, Patch(), Mix(), 384, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
                                                patch_masker=None if mode == "off" else masker).to(dev)
        tr.global_step.fill_(step_value)
        params = list(tr.head.parameters()) + [tr.view_embeddings]

        def labeled_step():
            batch["images"] = images
            batch["keypoints"].copy_(kp)
            return torch.autograd.grad(tr.training_step(batch, 0)["loss"], params)

        if mode != "on_graph":
            steps[mode] = timed(labeled_step)
            continue
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                labeled_step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            labeled_step()
        steps[mode] = timed(graph.replay)
    res["labeled_step_config4"] = {**steps, "note": "stand-in transformer, heatmap MSE only, gradients of head + view embeddings, no optimizer; "
                                                    "masking at ratio 0.5"}
    res["card_after"] = card()
    if len(sys.argv) > 1:
        out = sys.argv[1]
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
