"""The mirror-fish head (51 keypoints: three mirrored views x 17) on the bf16 tensor-core route and on fp32 features.

768 frames of (2048, 8, 12) ResNet-50 features (256 x 384 images), deconvs 512 -> 51 -> 51, heatmaps (768, 51, 64, 96).
Timed per call with CUDA events, the L2 flushed before each call (a 256 MB write), after a warm-up of every shape:
  forward          HeatmapHead.forward without autograd
  forward_decode   forward_with_keypoints without autograd (head + soft-argmax decode)
  train_backward   the training form's backward alone (forward_with_keypoints with autograd is set up untimed):
                   a dense heatmap-MSE-shaped gradient plus the decode's keypoint gradient (sparse windows on the bf16
                   route; the dense decode backward on fp32 features).  An entry that fails records the error
                   instead of a time.
The card's name, power limit and SM clocks are read in the same call.  Usage:
    python scripts/bench_wide_head.py [out.json]
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402

B, C, H, W, K = 768, 2048, 8, 12, 51
REPS = 10


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"nvidia_smi": {"query": q, "value": out}, "torch_name": torch.cuda.get_device_name(0)}


def main():
    assert torch.cuda.is_available(), "this benchmark measures the H100; it needs cuda:0"
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    head = HeatmapHead("resnet50", C, K, deconv_out_channels=K).to(dev)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    gen = torch.Generator(device=dev).manual_seed(1)
    f32 = torch.randn(B, C, H, W, device=dev, generator=gen) * 0.5
    feats = {"bf16": f32.bfloat16(), "fp32": f32}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    g_hm = torch.randn(B, K, 8 * H, 8 * W, device=dev, generator=gen) * 1e-3
    g_kp = torch.randn(B, 2 * K, device=dev, generator=gen)

    def timed(fn, setup=None):
        ms = []
        for i in range(REPS + 2):  # two warm-up calls
            state = setup() if setup else None
            flush.fill_(i & 0xFF)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(state) if setup else fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 2:
                ms.append(e0.elapsed_time(e1))
        ms.sort()
        return {"median_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1], "reps": REPS}

    res = {"shape": {"B": B, "C": C, "H": H, "W": W, "K": K, "heatmaps": [B, K, 8 * H, 8 * W]}, "card_before": card()}
    for name, x in feats.items():
        routed = ops.head_bf16_supported(tuple(x.shape), [K, K], train=False) and x.dtype == torch.bfloat16
        entry = {"tensor_core_forward": routed}
        with torch.no_grad():
            entry["forward"] = timed(lambda: head(x))
            entry["forward_decode"] = timed(lambda: head.forward_with_keypoints(x))

        def setup(x=x):
            hm, kp, _ = head.forward_with_keypoints(x.detach().requires_grad_(True))
            return hm, kp

        try:
            entry["tensor_core_backward"] = ops.head_bf16_supported(tuple(x.shape), [K, K], train=True) and x.dtype == torch.bfloat16
            entry["train_backward"] = timed(lambda st: torch.autograd.backward(list(st), [g_hm, g_kp]), setup)
        except Exception as exc:  # noqa: BLE001  (recorded, not hidden)
            entry["train_backward"] = {"error": str(exc)[:200]}
        head.zero_grad(set_to_none=True)
        res[name] = entry
    with torch.no_grad():
        a, b = head(feats["bf16"]), head(feats["fp32"])
        res["bf16_vs_fp32_heatmaps_max_abs_diff"] = float((a - b).abs().max())
        res["heatmap_max"] = float(b.max())
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
