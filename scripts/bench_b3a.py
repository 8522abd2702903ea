"""Device time of the layer-1 data gradient (b3a_dgrad_kernel) on its own, at BASELINE config 2's head.

The head's backward with feature gradients runs b3a; the same backward on frozen features (features that do not require
a gradient) runs everything else and skips it.  b3a's time is the difference of the two medians, each backward timed with CUDA
events after an L2 flush.  The kernel's own device time in the same backwards (torch.profiler, mean per call) is printed
beside it.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_b3a.py [--frames 256 512] [--reps 25] [--json OUT]
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


def time_backward(out, inputs, gout, reps, flush):
    ms = []
    for i in range(reps + 3):
        flush()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.autograd.grad(out, inputs, gout, retain_graph=True)
        e1.record()
        torch.cuda.synchronize()
        if i >= 3:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def kernel_us(out, inputs, gout, reps, flush, name="b3a_dgrad_kernel"):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            flush()
            torch.autograd.grad(out, inputs, gout, retain_graph=True)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if name in e.key]
    return round(sum(e.device_time_total for e in ev) / max(1, sum(e.count for e in ev)), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_b3a.py measures on the GPU"
    dev = torch.device("cuda:0")
    import lightning_pose_b200  # noqa: F401
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(0)
    head = HeatmapHead("resnet50", bench.FEAT_C, bench.K_PTS).to(dev)
    params = list(head.parameters())
    flush = bench.L2Flusher(dev)
    with bench.ClockSampler(0) as clk:
        rows = []
        for n in args.frames:
            g = torch.Generator(device=dev).manual_seed(n)
            feats = (torch.randn(n, bench.FEAT_C, bench.FEAT_HW, bench.FEAT_HW, device=dev, generator=g) * 0.5).bfloat16()
            f = feats.clone().requires_grad_(True)
            out = head(f)
            gout = torch.randn(out.shape, device=dev, generator=g)
            full = time_backward(out, [f] + params, gout, args.reps, flush)
            kern = kernel_us(out, [f] + params, gout, args.reps, flush)
            del out, f
            out = head(feats)  # frozen features: the backward is not asked for d features
            frozen = time_backward(out, params, gout, args.reps, flush)
            del out
            rows.append({"frames": n, "backward_ms": full, "frozen_ms": frozen, "b3a_us": round(1e3 * (full[0] - frozen[0]), 1),
                         "b3a_kernel_us": kern})
    res = {"gpu": gpu_info(), "clocks": clk.summary(), "reps": args.reps, "rows": rows}
    print(f"{res['gpu'].get('name')}  power limit {res['gpu'].get('power.limit')}  SM clock {res['clocks'].get('sm_mhz')} MHz")
    for r in rows:
        print(f"{r['frames']:5d} frames: backward {r['backward_ms'][0]:.3f} ms, frozen features {r['frozen_ms'][0]:.3f} ms "
              f"(median of {args.reps}) -> b3a {r['b3a_us']:.1f} us; b3a kernel {r['b3a_kernel_us']:.1f} us")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
