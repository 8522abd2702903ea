"""Inference on fp32 / bf16 / fp16 features: head-forward times and keypoint error against the fp32 oracle.

Timing (no gradients, final softmax on): the head forward, and the head forward + soft-argmax decode
(``HeatmapHead.forward_with_keypoints``), for fp32, bf16 and fp16 features at
  config2   768 x (2048, 12, 12) features, deconvs 512 -> 17 -> 17      (whole-frame kernels)
  config5   96 x (2048, 16, 16), one BatchedPredictor chunk -> 128^2 heatmaps (banded kernels)
  config3   768 x (384, 16, 16), one deconv 96 -> 17                      (banded kernels)
  mirror    768 x (2048, 8, 12), deconvs 512 -> 51 -> 51                 (keypoint groups)
and one BatchedPredictor config-5 chunk (96 frames of streamed features, CUDA-graph replay) at bf16 and fp16.  CUDA
events around each call with the L2 flushed before it (a 256 MB write); median and min-max of REPS calls after two
warm-up calls.

Accuracy: bench.make_problem(regime="trained") features and weights at config 2 (the inputs of kp_error_hist.py),
rounded to bf16 and to fp16; keypoints of each route against the float64 head + decode on the fp32 features and
weights.  Median, p99 and max px over confident keypoints (oracle confidence > 0.5), and the fraction within
1e-4 x image size (384 px).

The card's name, power limit and SM clocks are read in the same call.  Usage: python scripts/bench_f16_predict.py [out.json]
(the result is printed as one JSON line, and also written to out.json when given)
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

REPS = 15
SHAPES = {  # name: (frames, C, H, W, (c1[, c2]))
    "config2": (768, 2048, 12, 12, (17, 17)),
    "config5_chunk": (96, 2048, 16, 16, (17, 17)),
    "config3": (768, 384, 16, 16, (17,)),
    "mirror_fish": (768, 2048, 8, 12, (51, 51)),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"query": q, "value": out}


def main():
    import torch

    import bench
    import scale_oracle as S
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(2):
            fn()
        ts = []
        for _ in range(REPS):
            flush.random_(generator=gen)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return {"median_ms": round(float(np.median(ts)), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}

    def make_head(c, ch):
        torch.manual_seed(3)
        head = HeatmapHead("resnet50", c, ch[1], deconv_out_channels=ch[0]) if len(ch) == 2 else HeatmapHead("vits_dino", c, ch[0])
        for layer in list(head.upsampling_layers)[1:]:
            torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
        return head.to(dev).eval().requires_grad_(False)

    res = {"card_before": card(), "reps": REPS, "timing": {}}
    with torch.no_grad():
        for name, (b, c, h, w, ch) in SHAPES.items():
            head = make_head(c, ch)
            f32 = torch.randn(b, c, h, w, device=dev, generator=gen) * 0.5
            row = {}
            for dt_name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16), ("fp16", torch.float16)):
                f = f32.to(dt)
                row[dt_name] = {"head": timed(lambda: head(f)), "head_decode": timed(lambda: head.forward_with_keypoints(f))}
            res["timing"][name] = row
        # one BatchedPredictor config-5 chunk of streamed features, graph replay
        b, c, h, w, ch = SHAPES["config5_chunk"]
        head = make_head(c, ch)
        chunk_rows = {}
        for dt_name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
            feats = (torch.randn(b, c, h, w, device=dev, generator=gen) * 0.5).to(dt)
            bp = BatchedPredictor(head, ch[-1], (REPS + 3) * b, b, (512, 512))  # room for every timed chunk
            bp.feed(feats)  # capture
            chunk_rows[dt_name] = {**timed(lambda: bp.feed(feats)), "launches_per_chunk": bp.launches_per_chunk}
        res["timing"]["batched_predictor_config5_chunk"] = chunk_rows

    # ---- accuracy at config 2, trained-like regime -----------------------------------------------------------------
    prob = bench.make_problem(2, seed=99, device=dev, regime="trained")
    w1, b1, w2, b2 = prob["head_params"]
    head = HeatmapHead("resnet50", bench.FEAT_C, bench.K_PTS)
    d1, d2 = list(head.upsampling_layers)[1:]
    with torch.no_grad():
        d1.weight.copy_(w1), d1.bias.copy_(b1), d2.weight.copy_(w2), d2.bias.copy_(b2)
    head = head.to(dev).eval().requires_grad_(False)
    feats = prob["feats"].to(dev)
    ref = S.head_ref_chunked(feats, [w1.to(dev), w2.to(dev)], [b1.to(dev), b2.to(dev)], softmax=True, operands=None)
    kp_ref, cf_ref, _, _ = S.decode_ref(ref, 2)
    conf = (cf_ref > 0.5).flatten().cpu().numpy()
    acc = {"workload": f"config 2: {feats.shape[0]} frames of make_problem(regime='trained'), K = {bench.K_PTS}, image {bench.IMG} px",
           "bar_px": 1e-4 * bench.IMG, "frac_confident": float(conf.mean())}
    for dt_name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16), ("fp32", torch.float32)):
        with torch.no_grad():
            _, kp, _ = head.forward_with_keypoints(feats.to(dt))
        d = (kp.double() - kp_ref).abs().reshape(-1, bench.K_PTS, 2).amax(-1).flatten().cpu().numpy()[conf]
        acc[dt_name] = {"n": int(d.size), "median_px": float(np.median(d)), "p99_px": float(np.percentile(d, 99)), "max_px": float(d.max()),
                        "frac_within_bar": float((d <= 1e-4 * bench.IMG).mean())}
    res["accuracy_vs_fp32_oracle"] = acc
    res["card_after"] = card()
    if len(sys.argv) > 1:  # the JSON goes where the caller asks; without a path it is only printed
        out = sys.argv[1]
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
