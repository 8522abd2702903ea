"""Device time of training from keypoint targets made on the device against dense target planes.

  (a) HeatmapKLLoss and HeatmapJSLoss, forward + backward, at config 2's labeled batch (256 x 17 planes of 96 x 96 from
      384 x 384 images): fused (lpb_heatmap_loss_from_keypoints_*, no target plane written) against
      GaussianTargets.materialize() + the dense loss (targets written, then read by the forward and the backward)
  (b) the config-3 context (MHCRNN) labeled step, evaluate_labeled + backward: 16 examples x 5 frames of 256 x 256, a
      stride-16 stand-in backbone (one strided convolution to 384 bf16 channels), heatmap MSE
  (c) the config-4 multi-view transformer labeled step, evaluate_labeled + backward: 8 examples x 4 views of 384 x 384,
      a stand-in transformer (patch convolution + one token-mixing linear layer, 384 channels), heatmap MSE
For (b) and (c) the dense-target batch carries the planes already on the device, as a DataLoader would ship them; the
keypoint-only batch carries (keypoints, visibility).  Each form is timed with CUDA events after an L2 flush, the forms
alternated, medians over --reps calls.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_keypoint_targets.py [--reps 20] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from profile_head_gemms import gpu_info  # noqa: E402


def timed(forms: dict, reps: int, flush, warmup: int = 3) -> dict:
    ms = {k: [] for k in forms}
    for i in range(reps + warmup):
        for name, fn in (forms.items() if i % 2 == 0 else reversed(forms.items())):
            flush()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= warmup:
                ms[name].append(e0.elapsed_time(e1))
    return {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in ms.items()}


def labels(b, planes, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    kp = torch.rand(b, planes, 2, device=dev, generator=g) * torch.tensor([w, h], device=dev, dtype=torch.float32)
    vis = torch.full((b, planes), 2, dtype=torch.int32, device=dev)
    vis[:, ::7] = 0  # some unlabeled keypoints
    return kp, vis


def losses_at_config2(dev, flush, reps):
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.heatmaps import GaussianTargets

    b, k, img, hm = 256, 17, 384, 96
    kp, vis = labels(b, k, img, img, dev, 1)
    preds = torch.softmax(torch.randn(b, k, hm * hm, device=dev), -1).reshape(b, k, hm, hm).requires_grad_(True)
    out = {}
    for kind in ("kl", "js"):
        def fused():
            targ = GaussianTargets(kp, img, img, (hm, hm), visibility=vis)
            loss = ops.heatmap_loss_from_keypoints(kind, targ.keypoints, preds, img, img, visibility=vis)
            return torch.autograd.grad(loss, preds)

        def materialized():
            targ = GaussianTargets(kp, img, img, (hm, hm), visibility=vis)
            loss = ops.heatmap_loss(targ.materialize(), preds, kind)
            return torch.autograd.grad(loss, preds)

        (ga,), (gb,) = fused(), materialized()
        rel = float((ga - gb).abs().max()) / float(gb.abs().max())
        out[kind] = {"ms": timed({"fused": fused, "materialized": materialized}, reps, flush), "grad_max_rel_diff": rel}
    plane = b * k * hm * hm * 4
    out["bytes_model"] = {"fused": 3 * plane, "materialized": 6 * plane, "target_plane_bytes": plane}
    out["shape"] = [b, k, hm, hm]
    return out


class _Conv(torch.nn.Module):
    def __init__(self, c, stride):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, c, stride, stride=stride)

    def forward(self, x):
        return self.conv(x).bfloat16()


class _Patch(torch.nn.Module):
    def __init__(self, d):
        super().__init__()
        self.proj = torch.nn.Conv2d(3, d, 16, stride=16)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class _Mix(torch.nn.Module):
    def __init__(self, d):
        super().__init__()
        self.lin = torch.nn.Linear(d, d)

    def forward(self, t):
        return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()


def step_forms(tr, dense_batch, kp_batch, kp0):
    def run(batch):
        def f():
            batch["keypoints"].copy_(kp0)  # the dense route's model_to_frame_batch rewrites the keypoints in place
            tr.zero_grad(set_to_none=True)
            tr.evaluate_labeled(batch, "train", 1.0).backward()
        return f

    return {"keypoint_only": run(kp_batch), "dense_targets": run(dense_batch)}


def context_step(dev, flush, reps):
    from lightning_pose_b200 import ops
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import HeatmapTrackerMHCRNN

    b, k, img, hm = 16, 17, 256, 64
    torch.manual_seed(0)
    tr = HeatmapTrackerMHCRNN(k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None), backbone=_Conv(384, 16),
                              backbone_arch="vits_dino", num_fc_input_features=384).to(dev)
    kp, vis = labels(b, k, img, img, dev, 2)
    images = torch.randn(b, 5, 3, img, img, device=dev)
    bbox = torch.tensor([[0.0, 0.0, float(img), float(img)]], device=dev).repeat(b, 1)
    kp0 = kp.reshape(b, -1).clone()
    dense = {"images": images, "bbox": bbox, "keypoints": kp0.clone(), "heatmaps": ops.generate_heatmaps(kp, img, img, (hm, hm), visibility=vis)}
    only = {"images": images, "bbox": bbox, "keypoints": kp0.clone(), "visibility": vis}
    return {"ms": timed(step_forms(tr, dense, only, kp0), reps, flush), "dense_target_bytes_per_step": b * k * hm * hm * 4,
            "keypoint_bytes_per_step": b * k * (2 * 4 + 4), "shape": [b, 5, 3, img, img]}


def multiview_step(dev, flush, reps):
    from lightning_pose_b200 import ops
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    b, v, k, img, hm, d = 8, 4, 17, 384, 96, 384
    torch.manual_seed(0)
    tr = HeatmapTrackerMultiviewTransformer(k, v, _Patch(d), _Mix(d), d, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)).to(dev)
    kp, vis = labels(b, v * k, img, img, dev, 3)
    images = torch.randn(b, v, 3, img, img, device=dev)
    bbox = torch.tensor([[0.0, 0.0, float(img), float(img)] * v], device=dev).repeat(b, 1)
    kp0 = kp.reshape(b, -1).clone()
    common = {"images": images, "bbox": bbox, "is_multiview": True}
    dense = {**common, "keypoints": kp0.clone(), "heatmaps": ops.generate_heatmaps(kp, img, img, (hm, hm), visibility=vis)}
    only = {**common, "keypoints": kp0.clone(), "visibility": vis}
    return {"ms": timed(step_forms(tr, dense, only, kp0), reps, flush), "dense_target_bytes_per_step": b * v * k * hm * hm * 4,
            "keypoint_bytes_per_step": b * v * k * (2 * 4 + 4), "shape": [b, v, 3, img, img]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert args.reps >= 15, "medians over at least 15 calls"
    assert torch.cuda.is_available(), "bench_keypoint_targets.py measures on the GPU"
    dev = torch.device("cuda:0")
    flush = bench.L2Flusher(dev)
    res = {"gpu_before": gpu_info(), "reps": args.reps,
           "a_losses_config2": losses_at_config2(dev, flush, args.reps),
           "b_context_step_config3": context_step(dev, flush, args.reps),
           "c_multiview_step_config4": multiview_step(dev, flush, args.reps),
           "gpu_after": gpu_info()}
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
