"""Distribution of |d(x, y)| between the bf16 tensor-core head (+ decode) and the fp32 CPU oracle on identical inputs
(BASELINE configs[1] shapes, bench.py's "trained-like" regime and a random-weights regime).  GPU box.
Writes gpurun_out/r02_bf16_keypoint_error.json (copied to profiles/ afterwards)."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402
from oracle import lp_oracle as O  # noqa: E402


def run(regime: str, clips: int = 2):
    dev = torch.device("cuda:0")
    prob = bench.make_problem(clips, seed=99, device=dev, regime="trained")
    w1, b1, w2, b2 = prob["head_params"]
    if regime == "random":
        torch.manual_seed(5)
        w1 = torch.nn.init.xavier_uniform_(torch.empty_like(w1), gain=3.0)
        w2 = torch.nn.init.xavier_uniform_(torch.empty_like(w2), gain=3.0)
        prob["feats"] = torch.randn_like(prob["feats"]) * 0.5
    feats = prob["feats"].bfloat16()
    head = HeatmapHead("resnet50", bench.FEAT_C, bench.K_PTS)
    d1, d2 = list(head.upsampling_layers)[1:]
    with torch.no_grad():
        d1.weight.copy_(w1), d1.bias.copy_(b1), d2.weight.copy_(w2), d2.bias.copy_(b2)
    head = head.to(dev)
    with torch.no_grad():
        hm, kp, cf = head.forward_with_keypoints(feats.to(dev))
    # fp32 oracle on the same (bf16-valued) features, fp32 weights, fp32 everywhere
    hm_ref = O.head_forward(feats.float(), [w1, w2], [b1, b2])
    kp_ref, cf_ref = O.decode_softargmax(hm_ref, 2, 1000.0)
    # and with the kernel's operand roundings (weights, inter-layer activations in bf16): isolates accumulation order
    import torch.nn.functional as F
    r = lambda t: t.bfloat16().float()
    mid = F.conv_transpose2d(F.pixel_shuffle(feats.float(), 2), r(w1), b1, stride=2, padding=1, output_padding=1)
    hm_r = O.spatial_softmax2d(F.conv_transpose2d(r(mid), r(w2), b2, stride=2, padding=1, output_padding=1), 1.0)
    kp_r, _ = O.decode_softargmax(hm_r, 2, 1000.0)
    out = {}
    for name, ref in (("vs_fp32_reference", kp_ref), ("vs_same_roundings", kp_r)):
        d = (kp.cpu() - ref).reshape(-1, bench.K_PTS, 2).abs().amax(-1).flatten().numpy()
        conf_ok = (cf_ref.flatten().numpy() > 0.5)
        sel = d[conf_ok] if conf_ok.any() else d
        out[name] = {"n": int(sel.size), "frac_confident": float(conf_ok.mean()), "median_px": float(np.median(sel)), "p90_px": float(np.percentile(sel, 90)),
                     "p99_px": float(np.percentile(sel, 99)), "max_px": float(sel.max()), "rel_p99": float(np.percentile(sel, 99) / bench.IMG),
                     "frac_within_1e-4_rel": float((sel <= 1e-4 * bench.IMG).mean())}
    rel = ((hm.cpu() - hm_ref).abs() / (hm_ref.abs() + 1e-7)).flatten().numpy()
    out["heatmap_rel_err_vs_fp32"] = {"median": float(np.median(rel)), "p99": float(np.percentile(rel, 99)), "max": float(rel.max())}
    out["confidence_abs_err_vs_fp32"] = {"p99": float(np.percentile((cf.cpu() - cf_ref).abs().flatten().numpy(), 99))}
    return out


if __name__ == "__main__":
    res = {"workload": "cfg 2: (96 frames, 2048, 12, 12) bf16 features -> 96x96 heatmaps -> 384x384 field, K = 17", "north_star_bar_px": 1e-4 * bench.IMG,
           "trained_like": run("trained"), "random_weights": run("random")}
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "r02_bf16_keypoint_error.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))
