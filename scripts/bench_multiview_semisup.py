"""The multi-view transformer's semi-supervised training step (SemiSupervisedHeatmapTrackerMultiviewTransformer) at
BASELINE config 4, replayed from one CUDA graph and eager, and each of its two branches.

Setup: 8 labeled examples x 4 views and T = 32 unlabeled frames x 4 views, 384 x 384 model frames, K = 17, the
stand-in transformer of scripts/bench_configs.py (patch convolution + one token-mixing layer, bf16 tokens (·, 384, 24, 24)
into the head).  Labeled losses: heatmap MSE; unsupervised: temporal + pca_multiview (one fused launch) + temporal
heatmap MSE, annealed by the device-held weight.  The unlabeled views are uint8 surfaces (1024 x 1280 x 2,
720 x 1280 x 2) augmented on the device (training.imgaug "dlc") inside the step.  Every step is forward + the
gradients of the head and view embeddings (no optimizer).

Rows:
  step_graph / step_eager         the whole semi-supervised training_step + gradients
  labeled_graph / labeled_eager   the labeled branch alone: HeatmapTrackerMultiviewTransformer.training_step + gradients
  unlabeled_graph / unlabeled_eager  the unlabeled branch alone: augmented ingest, forward, the unsupervised losses
                                  (LossFactory.total_on_device) + gradients
  kernel launches                 kernel nodes of each captured graph

CUDA events around each call, median and min-max of REPS calls after three warm-up calls.  The card's name, power limit
and SM clocks are read in the same call.  Usage: python scripts/bench_multiview_semisup.py [out.json] (one JSON line is
printed; also written to out.json when given).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REPS = 30
B, V, T, K, SIZE, D = 8, 4, 32, 17, (384, 384), 384
SOURCES = [(1024, 1280), (1024, 1280), (720, 1280), (720, 1280)]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"query": q, "value": out}


def main():
    import torch

    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.video import frames_to_unlabeled_batch
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import SemiSupervisedHeatmapTrackerMultiviewTransformer
    from lightning_pose_b200.utils.predictions import _graph_kernel_count

    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)

    class Patch(torch.nn.Module):  # stand-in ViT patch embedding (scripts/bench_configs.py)
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Conv2d(3, D, 16, stride=16)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class Mix(torch.nn.Module):  # stand-in encoder: one token-mixing linear layer
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(D, D)

        def forward(self, t):
            return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()

    h, w = SIZE
    fit = torch.rand(256, 2 * V * K, generator=torch.Generator().manual_seed(1)) * 400  # PCA fit rows (frame pixels)
    unsup = {"temporal": {"log_weight": 0.5, "epsilon": 1.0, "prob_threshold": 0.05},
             "pca_multiview": {"loss_name": "pca_multiview", "log_weight": 1.0, "epsilon": 2.0, "components_to_keep": 3, "mirrored_column_matches": [[v * K + j for j in range(K)] for v in range(V)]},
             "temporal_heatmap_mse": {"loss_name": "temporal_heatmap_mse", "log_weight": 0.0, "epsilon": 0.0, "prob_threshold": 0.05}}
    torch.manual_seed(4)
    tr = SemiSupervisedHeatmapTrackerMultiviewTransformer(
        K, V, Patch(), Mix(), D, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
        loss_factory_unsupervised=LossFactory(unsup, fit)).to(dev)
    tr.total_unsupervised_importance.fill_(0.5)
    params = list(tr.head.parameters()) + [tr.view_embeddings]
    kp = torch.rand(B, V * K * 2, device=dev, generator=gen) * h
    images = torch.randn(B, V, 3, h, w, device=dev, generator=gen)
    labeled = {"images": images, "keypoints": kp.clone(), "heatmaps": ops.generate_heatmaps(kp.reshape(B, V * K, 2), h, w, (h // 4, w // 4)),
               "bbox": torch.tensor([[0.0, 0.0, float(h), float(w)] * V], device=dev).repeat(B, 1), "is_multiview": True}
    views = [torch.randint(0, 256, (T, sh, sw, 3), dtype=torch.uint8, device=dev, generator=gen) for sh, sw in SOURCES]
    draws = torch.Generator(device=dev).manual_seed(2)

    def reset_labeled():
        labeled["images"] = images
        labeled["keypoints"].copy_(kp)  # model_to_frame_batch rewrites the targets in place

    def step():
        reset_labeled()
        unlabeled = frames_to_unlabeled_batch(views, SIZE, imgaug="dlc", generator=draws)
        return torch.autograd.grad(tr.training_step({"labeled": labeled, "unlabeled": unlabeled}, 0)["loss"], params)

    def labeled_branch():
        reset_labeled()
        return torch.autograd.grad(super(SemiSupervisedHeatmapTrackerMultiviewTransformer, tr).training_step(labeled, 0)["loss"], params)

    def unlabeled_branch():
        unlabeled = frames_to_unlabeled_batch(views, SIZE, imgaug="dlc", generator=draws)
        loss, _ = tr.loss_factory_unsup.total_on_device("train", tr.total_unsupervised_importance, **tr.get_loss_inputs_unlabeled(unlabeled))
        return torch.autograd.grad(loss, params)

    def timed(fn, reps=REPS, warmup=3):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3)}

    def captured(fn):
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                fn()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph(keep_graph=True)  # kept so that its kernel nodes can be counted
        graph.register_generator_state(draws)
        with torch.cuda.graph(graph):
            fn()
        launches = _graph_kernel_count(graph)
        graph.instantiate()
        return graph, launches

    res = {"card_before": card(), "reps": REPS, "setup": {"labeled": [B, V, 3, h, w], "unlabeled_frames": T, "views": V,
                                                            "keypoints": K, "sources": SOURCES, "features": "bf16 (., 384, 24, 24)",
                                                            "unsupervised": list(unsup)}}
    for name, fn in (("step", step), ("labeled", labeled_branch), ("unlabeled", unlabeled_branch)):
        res[f"{name}_eager"] = timed(fn)
        graph, launches = captured(fn)
        res[f"{name}_graph"] = {**timed(graph.replay), "kernel_launches": launches}
        del graph
    res["card_after"] = card()
    if len(sys.argv) > 1:
        out = sys.argv[1]
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
