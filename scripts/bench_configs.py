"""Informal timings of the other BASELINE configs' hot paths (configs 3, 4, 5) on one GPU: not bench lines (bench.py
measures configs[1]), but the numbers DESIGN.md quotes for them.  Writes gpurun_out/r02_configs.json."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lightning_pose_b200.models.heads.heatmap import HeatmapHead  # noqa: E402
from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead  # noqa: E402
from lightning_pose_b200.utils.predictions import BatchedPredictor  # noqa: E402

dev = torch.device("cuda:0")
pk, _ = bench.peaks()
flush = bench.L2Flusher(dev)
K = 17
res = {}


def head_for(arch, cin, gain=3.0):
    torch.manual_seed(1)
    head = HeatmapHead(arch, cin, K)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=gain)
    return head.to(dev)


def fwd_bwd(name, arch, shape, hm):
    b, c, fh, fw = shape
    head = head_for(arch, c)
    feats = (torch.randn(shape, device=dev) * 0.5).bfloat16()
    fb, hb = c * fh * fw * 2, K * hm * hm * 4
    with torch.no_grad():
        ms, med = bench.time_stage(lambda: head(feats), flush)
    res[f"{name}_head_fwd"] = {"frames": b, "ms": ms, "us_per_frame": 1e3 * ms / b, "algorithmic_bytes": b * (fb + hb), "frac_hbm": b * (fb + hb) / ms / 1e6 / pk["hbm_gbs"]}
    with torch.no_grad():
        ms, med = bench.time_stage(lambda: head.forward_with_keypoints(feats), flush)
    res[f"{name}_head+decode_fwd"] = {"frames": b, "ms": ms, "us_per_frame": 1e3 * ms / b, "algorithmic_bytes": b * (fb + hb + 204),
                                      "frac_hbm": b * (fb + hb + 204) / ms / 1e6 / pk["hbm_gbs"]}
    f = feats.clone().requires_grad_(True)
    out = head(f)
    g = torch.randn_like(out)
    params = list(head.parameters())
    ms, med = bench.time_stage(lambda: torch.autograd.grad(out, [f] + params, g, retain_graph=True), flush)
    res[f"{name}_head_bwd_dense"] = {"frames": b, "ms": ms, "us_per_frame": 1e3 * ms / b, "algorithmic_bytes": b * (2 * hb + 2 * fb),
                                     "frac_hbm": b * (2 * hb + 2 * fb) / ms / 1e6 / pk["hbm_gbs"]}


# config 3: ViT-S 256x256 (one deconv, 64x64 heatmaps); labeled context batch 16 x 5 frames + clip of 16
fwd_bwd("cfg3_vits_256", "vits_dino", (96, 384, 16, 16), 64)
# config 4: 4 views x 384x384 through the same head: (8 x 4, 384, 24, 24) -> 96x96
fwd_bwd("cfg4_multiview_384", "vits_dino", (32, 384, 24, 24), 96)
# config 5 shape, training form, for reference: ResNet-50 512x512 -> (., 2048, 16, 16) -> 128x128
fwd_bwd("cfg5_resnet50_512", "resnet50", (96, 2048, 16, 16), 128)

# config 3, context head on a clip: T = 64 frames -> 60 valid outputs (sf + mf heatmaps)
torch.manual_seed(2)
mh = HeatmapMHCRNNHead("vits_dino", 384, K, upsampling_factor=1).to(dev)
seq = (torch.randn(64, 384, 16, 16, device=dev) * 0.5).bfloat16()
with torch.no_grad():
    ms, _ = bench.time_stage(lambda: mh.forward_sequence(seq), flush)
res["cfg3_mhcrnn_forward_sequence"] = {"frames": 64, "ms": ms, "us_per_frame": 1e3 * ms / 64}
s2 = seq.clone().requires_grad_(True)
sf, mf = mh.forward_sequence(s2)
g1, g2 = torch.randn_like(sf), torch.randn_like(mf)
ms, _ = bench.time_stage(lambda: torch.autograd.grad([sf, mf], [s2] + list(mh.parameters()), [g1, g2], retain_graph=True, allow_unused=True), flush)
res["cfg3_mhcrnn_backward"] = {"frames": 64, "ms": ms, "us_per_frame": 1e3 * ms / 64}

# decode alone on trained-like (peaked) planes of each config's heatmap size: the head timings above use random weights, whose
# multi-modal heatmaps take the dense decode path (worst case); a trained network's planes are unimodal
def peaked(n, s_):
    yy, xx = torch.meshgrid(torch.arange(s_, device=dev), torch.arange(s_, device=dev), indexing="ij")
    c = torch.rand(n, K, 2, device=dev) * (s_ - 20) + 10
    hm = torch.exp(-((yy[None, None] - c[..., 1, None, None]) ** 2 + (xx[None, None] - c[..., 0, None, None]) ** 2) / (2 * 1.3**2)) + 1e-6
    return hm / hm.sum((2, 3), keepdim=True)


from lightning_pose_b200 import ops  # noqa: E402

for name, n, s_ in (("cfg3_64", 96, 64), ("cfg4_96", 32, 96), ("cfg5_128", 96, 128)):
    hm = peaked(n, s_)
    ms, _ = bench.time_stage(lambda: ops.decode_softargmax(hm, 2, 1000.0), flush)
    nb = n * (K * s_ * s_ * 4 + 204)
    res[f"{name}_decode_fwd_peaked"] = {"frames": n, "ms": ms, "us_per_frame": 1e3 * ms / n, "algorithmic_bytes": nb, "frac_hbm": nb / ms / 1e6 / pk["hbm_gbs"]}

# config 5: batched inference driver on a trained-like response: bench.make_problem at the 512x512 geometry
# (features (., 2048, 16, 16), heatmaps 128x128), 100 chunks of 96 frames (4 resident chunks cycled: 403 MB > L2)
bench.FEAT_HW, bench.HM, bench.IMG = 16, 128, 512
prob = bench.make_problem(8, seed=7, device=dev, regime="trained")  # 8 clips x 48 = 384 frames = 4 chunks
bench.FEAT_HW, bench.HM, bench.IMG = 12, 96, 384
head = HeatmapHead("resnet50", 2048, K)
d1, d2 = list(head.upsampling_layers)[1:]
with torch.no_grad():
    w1, b1, w2, b2 = prob["head_params"]
    d1.weight.copy_(w1), d1.bias.copy_(b1), d2.weight.copy_(w2), d2.bias.copy_(b2)
head = head.to(dev).eval()
chunk, nchunks = 96, 100
feats_all = prob["feats"].bfloat16().to(dev)
pool = [feats_all[i * chunk : (i + 1) * chunk].contiguous() for i in range(4)]
for use_graph, sub in ((True, None), (False, None), (True, 48)):
    bp = BatchedPredictor(head, K, chunk * nchunks, chunk, (512, 512), use_graph=use_graph, sub_chunk=sub)
    bp.feed(pool[0])  # capture / warm
    bp.cursor.zero_()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(nchunks):
        bp.feed(pool[i % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    nb = chunk * nchunks * (2048 * 256 * 2 + 204)
    kp, cf = bp.results()
    res[f"cfg5_batched_inference_{'graph' if use_graph else 'eager'}_sub{sub or chunk}"] = {
        "frames": chunk * nchunks, "ms": ms, "frames_per_s": chunk * nchunks / ms * 1e3, "algorithmic_bytes": nb, "frac_hbm": nb / ms / 1e6 / pk["hbm_gbs"],
        "mean_confidence": float(cf.mean()),
        "note": "trained-like planted response (unimodal heatmaps); features resident on the device (includes the D2D copy of each chunk into the graph's static input); K1+K2 algorithmic bytes = features + 204 B/frame"}

# config 4 with a camera calibration (B = 8 per rank, 4 views, 17 keypoints, 384x384): the 3-D stage alone (pairwise
# triangulation -> pair-mean reprojection into model coordinates -> pairwise-projection loss), forward and backward, and
# the labeled multiview step (forward + backward, heatmap MSE) with the two 3-D losses on and off.  The transformer is a
# stand-in (patch conv + one token-mixing linear layer), so the step time is the head + decode + loss path.
import math  # noqa: E402
import subprocess  # noqa: E402

from lightning_pose_b200.losses.factory import LossFactory  # noqa: E402
from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer  # noqa: E402

cb, cv, img = 8, 4, 384
gen = torch.Generator().manual_seed(41)
Kc, Ec = torch.zeros(cb, cv, 3, 3), torch.zeros(cb, cv, 3, 4)
for j in range(cv):
    a = j / cv * math.pi  # cameras on a half circle, none facing another
    Kc[:, j] = torch.tensor([[800.0, 0.0, img / 2], [0.0, 800.0, img / 2], [0.0, 0.0, 1.0]])
    Ec[:, j] = torch.tensor([[math.cos(a), 0.0, -math.sin(a), 0.0], [0.0, 1.0, 0.0, 0.0], [math.sin(a), 0.0, math.cos(a), 2.0]])
Dc = torch.randn(cb, cv, 5, generator=gen) * 0.05
cams = [t.to(dev) for t in (Kc, Ec, Dc)]
kp_frame = (img / 2 - 2 + torch.rand(cb, cv, K, 2, generator=gen) * 4).to(dev).requires_grad_(True)
kp3 = (torch.randn(cb, K, 3, generator=gen) * 0.3).to(dev)
bbox_c = torch.tensor([[img / 2 - 2, img / 2 - 2, 4.0, 4.0] * cv], device=dev).repeat(cb, 1)  # rays near the optical axes


def stage3d():
    p3d = ops.triangulate_pairs(kp_frame, *cams)
    rep = ops.project_points(p3d, *cams, mean_over_pairs=True, bbox=bbox_c, model_size=(img, img))
    return ops.pairwise_projections_loss(kp3, p3d) + rep.sum() * 1e-6


with torch.no_grad():
    ms, _ = bench.time_stage(stage3d, flush)
res["cfg4_calibrated_3d_stage_fwd"] = {"frames": cb * cv, "ms": ms, "launches": 3}
ms, _ = bench.time_stage(lambda: torch.autograd.grad(stage3d(), kp_frame), flush)
res["cfg4_calibrated_3d_stage_fwd+bwd"] = {"frames": cb * cv, "ms": ms, "launches": 6, "note": "includes torch autograd bookkeeping and the small elementwise ops it adds"}


class Patch(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = torch.nn.Conv2d(3, 384, 16, stride=16)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class Mix(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(384, 384)

    def forward(self, t):
        return (self.lin(t) + t.mean(1, keepdim=True)).bfloat16()


kp_model = (torch.rand(cb, cv * K * 2, generator=gen) * img).to(dev)
batch = {"images": torch.randn(cb, cv, 3, img, img, generator=gen).to(dev), "keypoints": kp_model.clone(),
         "heatmaps": ops.generate_heatmaps(kp_model.reshape(cb, cv * K, 2), img, img, (96, 96)), "bbox": bbox_c, "is_multiview": True,
         "keypoints_3d": kp3, "intrinsic_matrix": cams[0], "extrinsic_matrix": cams[1], "distortions": cams[2]}
losses_on = {"heatmap_mse": {"log_weight": 0.0}, "supervised_pairwise_projections": {"log_weight": 0.0},
             "supervised_reprojection_heatmap_mse": {"log_weight": 0.0, "original_image_height": img, "original_image_width": img,
                                                     "downsampled_image_height": 96, "downsampled_image_width": 96}}
for tag, losses in (("3d_losses_off", {"heatmap_mse": {"log_weight": 0.0}}), ("3d_losses_on", losses_on)):
    torch.manual_seed(3)
    tr = HeatmapTrackerMultiviewTransformer(K, cv, Patch(), Mix(), 384, loss_factory=LossFactory(losses, None)).to(dev)
    params = list(tr.head.parameters()) + [tr.view_embeddings]

    def labeled_step():
        batch["keypoints"].copy_(kp_model)
        return torch.autograd.grad(tr.evaluate_labeled(batch, "train", 1.0), params)

    ms, _ = bench.time_stage(labeled_step, flush)
    res[f"cfg4_calibrated_labeled_step_{tag}"] = {"frames": cb * cv, "ms": ms, "note": "eager; stand-in transformer; includes the RMSE diagnostic"}
card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
res["cfg4_calibrated_card"] = {"nvidia_smi": card, "torch_name": torch.cuda.get_device_name(0)}

os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", "r02_configs.json"), "w"), indent=1)
print(json.dumps(res, indent=1))
