"""Device time of the labeled chain's backward (bench.py's step, 256 labeled frames): d loss -> head gradients.

Two forms of the same backward, alternated repetition by repetition in one process, each after an L2 flush:
  dense     the keypoint-target MSE's gradient written as a dense fp32 tensor (heatmap_mse_from_kp_bwd_kernel), then the
            head backward reading it (plane_dot_kernel, g2_build with a dense gradient): what the step ran before the
            gradient stayed implicit
  implicit  the head backward rebuilding the gradient from the keypoints (plane_dot_targets_kernel, g2_build's target form)
Both give the same bits (tests/test_mse_grad_fused_gpu.py).  The byte model counts the HBM traffic of the three kernels
that differ, from the shapes.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_labeled_bwd.py [--clips 16] [--reps 30] [--json OUT]
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


def byte_model(frames: int) -> dict:
    """HBM bytes of the kernels that differ between the two forms (one fp32 heatmap tensor = hm; G2 = the bf16 gradient
    operand of layer 2 in its padded row layout, 10 K-chunks of 16 bytes per row)."""
    hm = frames * bench.K_PTS * bench.HM * bench.HM * 4
    hi = wi = bench.HM // 2
    rows = (hi * (wi + 1) + 2 * (wi + 2) + 7) // 8 * 8
    g2 = frames * 10 * rows * 16
    fac = frames * bench.K_PTS * (4 + 2 * bench.HM) * 4
    return {
        "dense": {"mse_bwd": 2 * hm, "plane_dot": 2 * hm, "g2_build": 2 * hm + g2},
        "implicit": {"plane_dot_targets": hm + fac, "g2_build_targets": hm + g2 + fac},
        "heatmap_tensor_bytes": hm,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16, help="clips of bench.py's step: 16 labeled frames each")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_labeled_bwd.py measures on the GPU"
    from lightning_pose_b200 import ops

    dev = torch.device("cuda:0")
    prob = bench.make_problem(args.clips, seed=1234, device=dev)
    hp = bench.HotPath(prob, dev, fwd_only=True)
    nl = args.clips * bench.B_LABELED
    f = prob["feats"][:nl].to(torch.bfloat16).to(dev).requires_grad_(True)
    params = list(hp.head.parameters())
    hm, _, _ = hp.head.forward_with_keypoints(f)
    loss = 0.5 * ops.heatmap_mse_from_keypoints(hp.kp_lab, hm, bench.IMG, bench.IMG, visibility=hp.vis)

    def dense():
        (g,) = torch.autograd.grad(loss, hm, retain_graph=True)
        return torch.autograd.grad(hm, [f] + params, g.materialize(), retain_graph=True)

    def implicit():
        return torch.autograd.grad(loss, [f] + params, retain_graph=True)

    a, b = dense(), implicit()
    same = all(torch.equal(x, y) for x, y in zip(a, b))
    flush = bench.L2Flusher(dev)
    forms = {"dense": dense, "implicit": implicit}
    ms = {k: [] for k in forms}
    for i in range(args.reps + 3):
        for name, fn in (forms.items() if i % 2 == 0 else reversed(forms.items())):
            flush()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                ms[name].append(e0.elapsed_time(e1))
    model = byte_model(nl)
    res = {
        "what": "labeled chain backward (loss -> d features + head weight gradients), L2 flushed, forms alternated",
        "frames": nl, "reps": args.reps, "gpu": gpu_info(), "bitwise_equal": same,
        "ms": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in ms.items()},
        "bytes_model": model,
    }
    res["saved_ms_median"] = res["ms"]["dense"]["median"] - res["ms"]["implicit"]["median"]
    res["saved_bytes_model"] = sum(model["dense"].values()) - sum(model["implicit"].values())
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
