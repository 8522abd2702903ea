"""Time the regression head and training steps on the GPU (CUDA events, L2 flushed before every call, medians).

    python scripts/bench_regression.py [--out results.json] [--calls 30]      (prints one JSON line; --out also writes it)

* head forward / backward at 768 x (2048, 12, 12) bf16 (a ResNet-50 at 384 x 384): the fused entries
  (lpb_regression_head_fwd/_bwd) against torch's adaptive_avg_pool2d + linear and their autograd on the same card.
  Bytes model: the forward reads the features once (+ the small fp32 pooled / out), the backward writes d features
  once; achieved bandwidth is reported as a share of the H100 SXM's 3.35 TB/s.
* labeled and semi-supervised training steps (forward, losses, backward) with a stand-in convolutional backbone, eager
  and as a CUDA-graph replay.
The card's name, power limit and SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lightning_pose_b200.losses.factory import LossFactory  # noqa: E402
from lightning_pose_b200.models.heads.regression import LinearRegressionHead  # noqa: E402
from lightning_pose_b200.models.regression_tracker import RegressionTracker, SemiSupervisedRegressionTracker  # noqa: E402

PEAK_BW = 3.35e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def timed(fn, calls: int, flush: torch.Tensor) -> float:
    """median ms of fn over `calls` calls, each after an L2 flush (a 256 MB write) outside the timed window."""
    for _ in range(3):
        fn()
    times = []
    for _ in range(calls):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


class Stem(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 2048, 32, stride=32)

    def forward(self, x):
        return self.conv(x)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--calls", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_regression.py needs a CUDA device")
    dev = torch.device("cuda:0")
    flush = torch.empty(64 * 2**20, dtype=torch.float32, device=dev)
    res: dict = {"card": card()}

    b, c, h, w, k = 768, 2048, 12, 12, 17
    torch.manual_seed(0)
    head = LinearRegressionHead(c, 2 * k).to(dev)
    x = torch.randn(b, c, h, w, device=dev).bfloat16().requires_grad_(True)
    g = torch.randn(b, 2 * k, device=dev)
    feat_bytes = x.numel() * x.element_size()
    y = head(x)

    def torch_fwd():
        return nn.functional.linear(nn.functional.adaptive_avg_pool2d(x, 1).flatten(1).float(), head.linear_layer.weight,
                                    head.linear_layer.bias)

    yt = torch_fwd()
    res["head_fwd_ms"] = {"fused": timed(lambda: head(x), args.calls, flush), "torch": timed(torch_fwd, args.calls, flush)}
    res["head_bwd_ms"] = {
        "fused": timed(lambda: torch.autograd.grad(y, [x, *head.parameters()], g, retain_graph=True), args.calls, flush),
        "torch": timed(lambda: torch.autograd.grad(yt, [x, *head.parameters()], g, retain_graph=True), args.calls, flush),
    }
    with torch.no_grad():
        res["head_out_max_abs_diff_vs_torch"] = float((head(x) - torch_fwd()).abs().max())
    for kind in ("fwd", "bwd"):
        t = res[f"head_{kind}_ms"]["fused"] / 1e3
        res[f"head_{kind}_fused_bandwidth_share"] = feat_bytes / t / PEAK_BW
    res["bytes_model"] = {"features_read_fwd": feat_bytes, "dfeatures_written_bwd": feat_bytes}

    # training steps with a stand-in backbone: (64, 3, 384, 384) -> (64, 2048, 12, 12)
    for semi in (False, True):
        torch.manual_seed(1)
        sup = LossFactory({"regression": {"log_weight": 0.0}}, None)
        kw = dict(backbone=Stem(), num_fc_input_features=2048, loss_factory=sup)
        if semi:
            unsup = LossFactory({"temporal": {"log_weight": 1.0, "epsilon": 2.0}}, None)
            tr = SemiSupervisedRegressionTracker(k, loss_factory_unsupervised=unsup, **kw).to(dev)
        else:
            tr = RegressionTracker(k, **kw).to(dev)
        params = [p for p in tr.parameters()]
        lab = {"images": torch.randn(64, 3, 384, 384, device=dev), "keypoints": torch.rand(64, 2 * k, device=dev) * 384}
        batch = {"labeled": lab, "unlabeled": {"frames": torch.randn(32, 3, 384, 384, device=dev),
                                               "transforms": torch.tensor([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], device=dev)}} if semi else lab

        def step():
            return torch.autograd.grad(tr.training_step(batch, 0)["loss"], params)

        eager = timed(step, args.calls, flush)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        res[f"{'semisup' if semi else 'labeled'}_step_ms"] = {"eager": eager, "graph": timed(graph.replay, args.calls, flush)}
    res["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
