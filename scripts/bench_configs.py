"""Informal timings of the other BASELINE configs' hot paths (configs 3, 4, 5) on one GPU: not bench lines (bench.py
measures configs[1]), but the numbers DESIGN.md quotes for them.  Writes gpurun_out/r02_configs.json."""
import json
import os
import subprocess
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


class Patch(torch.nn.Module):  # stand-in ViT patch embedding of the config-4 transformer
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


def cfg2_unlabeled_aug():
    """One reference unlabeled training step's augmented ingest (training.imgaug "dlc"): T = 32 uint8 frames
    (dali.base.train.sequence_length) of a 1024 x 1024 and a 406 x 396 source, resized to 384 x 384.  The augmented
    kernel (FCHW fp32 and FHWC bf16, shot noise on and off) against its bytes model (each source byte read once, each
    output written once), the plain lpb_frames_normalize on the same frames, and the eager torch composition
    (interpolate -> affine_grid / grid_sample -> brightness / contrast -> torch.poisson -> normalise)."""
    import torch.nn.functional as F

    from lightning_pose_b200 import ops

    t, side = 32, 384
    mean_t = torch.tensor(ops.IMAGENET_MEAN, device=dev)[:, None, None]
    std_t = torch.tensor(ops.IMAGENET_STD, device=dev)[:, None, None]
    seed = torch.tensor([12345], dtype=torch.int64, device=dev)
    for sh, sw in ((1024, 1024), (406, 396)):
        tag = f"{sh}x{sw}"
        u8 = torch.randint(0, 256, (t, sh, sw, 3), dtype=torch.uint8, device=dev)
        src_bytes = t * sh * sw * 3
        for noise in ("on", "off"):
            params = torch.tensor([6.0, 1.1, 0.9, 1.05, 0.95, 5.0 if noise == "on" else 0.0], device=dev)
            for dtype, cl, form in ((torch.float32, False, "fchw_f32"), (torch.bfloat16, True, "fhwc_bf16")):
                fn = lambda: ops.frames_augment_normalize(u8, (side, side), params, seed, channels_last=cl, dtype=dtype)
                ms, med = bench.time_stage(fn, flush)
                nbytes = src_bytes + t * 3 * side * side * (4 if dtype == torch.float32 else 2)
                res[f"cfg2_unlabeled_aug_{tag}_{form}_noise_{noise}"] = {
                    "frames": t, "ms": ms, "ms_median": med, "bytes_model": nbytes, "gbs": nbytes / ms / 1e6,
                    "frac_hbm": nbytes / ms / 1e6 / pk["hbm_gbs"]}
        for dtype, cl, form in ((torch.float32, False, "fchw_f32"), (torch.bfloat16, True, "fhwc_bf16")):
            ms, med = bench.time_stage(lambda: ops.frames_normalize(u8, size=(side, side), channels_last=cl, dtype=dtype), flush)
            nbytes = src_bytes + t * 3 * side * side * (4 if dtype == torch.float32 else 2)
            res[f"cfg2_unlabeled_aug_{tag}_{form}_plain_ingest"] = {"frames": t, "ms": ms, "ms_median": med, "bytes_model": nbytes,
                                                                   "gbs": nbytes / ms / 1e6, "frac_hbm": nbytes / ms / 1e6 / pk["hbm_gbs"]}

        def eager():
            p, _ = ops.draw_dlc_params(1, dev)
            ang, sx, sy, br, ct, fac = p[0].unbind()
            x = F.interpolate(u8.permute(0, 3, 1, 2).float(), size=(side, side), mode="bilinear", align_corners=False)
            th = torch.deg2rad(ang)
            a = torch.stack([torch.stack([sx * torch.cos(th), -sx * torch.sin(th)]), torch.stack([sy * torch.sin(th), sy * torch.cos(th)])])
            ai = torch.linalg.inv(a)  # destination -> source, about c in pixel units, then in grid_sample's [-1, 1] units
            c = torch.tensor([side / 2.0, side / 2.0], device=dev)
            theta = torch.cat([ai, (c - ai @ c)[:, None]], dim=1)
            to_norm = torch.tensor([[2.0 / side, 0, -1], [0, 2.0 / side, -1], [0, 0, 1]], device=dev)
            full = torch.cat([theta, torch.tensor([[0.0, 0.0, 1.0]], device=dev)])
            theta_n = (to_norm @ full @ torch.linalg.inv(to_norm))[:2]
            grid = F.affine_grid(theta_n[None].expand(t, 2, 3), [t, 3, side, side], align_corners=False)
            x = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
            x = br * (0.5 + ct * (x - 0.5))
            x = torch.poisson(torch.clamp(x / fac, min=0)) * fac
            return (x / 255.0 - mean_t) / std_t

        with torch.no_grad():
            ms, med = bench.time_stage(eager, flush, reps=10, warmup=2)
        res[f"cfg2_unlabeled_aug_{tag}_eager_torch"] = {"frames": t, "ms": ms, "ms_median": med,
                                                        "note": "FCHW fp32, noise on; interpolate -> affine_grid/grid_sample -> elementwise -> torch.poisson -> normalise"}
        del u8
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res["cfg2_unlabeled_aug_card"] = {"nvidia_smi": card, "torch_name": torch.cuda.get_device_name(0), "hbm_gbs_used": pk["hbm_gbs"]}


if sys.argv[1:] == ["cfg2_unlabeled_aug"]:  # these entries alone, as JSON on stdout: python scripts/bench_configs.py cfg2_unlabeled_aug
    cfg2_unlabeled_aug()
    print(json.dumps(res, indent=1))
    sys.exit(0)


def cfg3_context():
    """Video prediction with the config-3 context model: 92 new frames per chunk (sequence_length 96) of (., 384, 16, 16)
    bf16 features -> 64 x 64 heatmaps, K = 17, 40 chunks.  Three paths: the context predictor (graph replay / eager), the
    reference's form (predict_step per overlapping window of 96 frames, i.e. forward_sequence + two decodes + selection +
    remap, then host stacking and fix_context_preds_confs), and the same predictor in single-frame mode (sf head only)."""
    import subprocess

    from lightning_pose_b200 import ops
    from lightning_pose_b200.utils.predictions import PredictionHandler

    t, s, nch, k = 92, 96, 40, K
    n = t * nch
    torch.manual_seed(3)
    mh = HeatmapMHCRNNHead("vits_dino", 384, k, upsampling_factor=1).to(dev).eval()
    pool = [(torch.randn(t, 384, 16, 16, device=dev) * 0.5).bfloat16() for _ in range(2)]
    box = torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=dev).repeat(t, 1)

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(reps):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    for mode in ("graph", "eager"):
        bp = BatchedPredictor(mh, k, n, t, (256, 256), use_graph=mode == "graph")
        ms = timed(lambda i=0: bp.feed(pool[i % 2], box), nch - 1)
        res[f"cfg3_context_predictor_{mode}"] = {"new_frames_per_chunk": t, "ms_per_chunk": ms, "frames_per_s": 1e3 * t / ms,
                                                 "launches_per_chunk": bp.launches_per_chunk}
    sf_only = BatchedPredictor(mh.head_sf, k, n, t, (256, 256))
    ms = timed(lambda i=0: sf_only.feed(pool[i % 2], box), nch - 1)
    res["cfg3_context_single_frame_predictor_graph"] = {"frames_per_chunk": t, "ms_per_chunk": ms, "frames_per_s": 1e3 * t / ms,
                                                        "launches_per_chunk": sf_only.launches_per_chunk}
    # reference form: windows of 96 frames (4 of them re-run from the previous window), host stack + fix-up at the end
    win = torch.cat([pool[0], pool[1][:4]])
    wbox = box[:1].repeat(s, 1)
    ph = PredictionHandler([f"bp{i}" for i in range(k)], n, model_type="heatmap_mhcrnn")

    def reference_form(i=0):
        preds = []
        for _ in range(4):
            with torch.no_grad():
                sf, mf = mh.forward_sequence(win)
                kp_sf, cf_sf = mh.run_subpixelmaxima(sf)
                kp_mf, cf_mf = mh.run_subpixelmaxima(mf)
            pick = torch.gt(cf_mf, cf_sf)
            kp = torch.where(pick[..., None], kp_mf.reshape(-1, k, 2), kp_sf.reshape(-1, k, 2)).reshape(-1, 2 * k)
            preds.append((ops.remap_keypoints(kp, None, wbox, 256, 256), torch.where(pick, cf_mf, cf_sf)))
        kp_all = torch.vstack([p[0] for p in preds]).cpu()
        ph.fix_context_preds_confs(kp_all)

    ms = timed(reference_form, 5) / 4
    res["cfg3_context_reference_form"] = {"new_frames_per_window": t, "ms_per_window": ms, "frames_per_s": 1e3 * t / ms,
                                          "note": "eager; forward_sequence on 96 frames per window + host stack/fix-up, amortised over 4 windows"}
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res["cfg3_context_card"] = {"nvidia_smi": card, "torch_name": torch.cuda.get_device_name(0)}


def cfg4_predict():
    """Multi-view video prediction with the config-4 transformer: 4 views of uint8 frames at mixed sizes (1024 x 1280 x 2,
    720 x 1280 x 2) -> 384 x 384, the stand-in transformer at embedding 384 -> (T 4, 384, 24, 24) -> 96 x 96 heatmaps,
    K = 17, T = 32 and 96 frames per chunk.  The ingest kernel against its bytes model (the source rows its bilinear taps
    touch, read whole, plus the output) and against V x lpb_frames_normalize + torch.stack; the predictor's chunk (graph
    replay and eager); the reference's form (per-view normalise + stack + predict_step + a host copy per batch + the host
    per-view split)."""
    import subprocess

    import pandas  # noqa: F401  (imported here so that the handler's first call does not time the import)

    from lightning_pose_b200 import ops
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer
    from lightning_pose_b200.utils.predictions import PredictionHandler

    shapes, side, k, v = ((1024, 1280), (1024, 1280), (720, 1280), (720, 1280)), 384, K, 4
    torch.manual_seed(4)
    model = HeatmapTrackerMultiviewTransformer(k, v, Patch(), Mix(), 384).to(dev).eval()

    def touched_rows(h):  # distinct source rows read by the taps of the side output rows (y0 and y1 of resized_pixel)
        sy = np.maximum((np.arange(side) + 0.5) * np.float32(h / side) - 0.5, 0)
        y0 = np.minimum(sy.astype(np.int64), h - 1)
        return len(set(y0) | set(np.minimum(y0 + 1, h - 1)))

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(reps):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    for t in (32, 96):
        gen = torch.Generator(device=dev).manual_seed(t)
        pool = [[torch.randint(0, 256, (t, h, w, 3), dtype=torch.uint8, device=dev, generator=gen) for h, w in shapes] for _ in range(2)]
        views = pool[0]
        src = sum(t * touched_rows(h) * w * 3 for h, w in shapes)
        for dtype, cl, form in ((torch.float32, False, "fchw_f32"), (torch.bfloat16, True, "fhwc_bf16")):
            out_bytes = t * v * 3 * side * side * (4 if dtype == torch.float32 else 2)
            ms, med = bench.time_stage(lambda: ops.frames_normalize_views(views, (side, side), channels_last=cl, dtype=dtype), flush)
            ms_s, med_s = bench.time_stage(lambda: torch.stack([ops.frames_normalize(x, size=(side, side), channels_last=cl, dtype=dtype) for x in views], 1), flush)
            res[f"cfg4_predict_T{t}_ingest_{form}"] = {
                "frames": t, "views": v, "ms": ms, "ms_median": med, "bytes_model": src + out_bytes, "gbs": (src + out_bytes) / ms / 1e6,
                "frac_hbm": (src + out_bytes) / ms / 1e6 / pk["hbm_gbs"], "per_view_normalize_plus_stack_ms": ms_s,
                "per_view_normalize_plus_stack_ms_median": med_s}
        n = t * 12
        for mode in ("graph", "eager"):
            bp = BatchedPredictor(model.head, k, n, t, (side, side), features_of=model.forward_vit, use_graph=mode == "graph", num_views=v)
            ms = timed(lambda i=0: bp.feed(pool[i % 2]), 11)
            res[f"cfg4_predict_T{t}_predictor_{mode}"] = {"video_frames_per_chunk": t, "ms_per_chunk": ms, "video_frames_per_s": 1e3 * t / ms,
                                                         "launches_per_chunk": bp.launches_per_chunk}
        ph = PredictionHandler([f"bp{i}" for i in range(k)], n, model_type="heatmap_multiview_transformer", view_names=["a", "b", "c", "d"])

        def reference_form(i=0):  # one batch of the reference's loop, the handler's host split amortised over 4 batches
            batch = {"frames": torch.stack([ops.frames_normalize(x, size=(side, side)) for x in pool[i % 2]], 1),
                     "bbox": torch.tensor([[0.0, 0.0, float(h), float(w)] for h, w in shapes], device=dev).reshape(1, -1).repeat(t, 1),
                     "is_multiview": True}
            kp, cf = model.predict_step(batch, i)
            preds.append((kp.cpu(), cf.cpu()))
            if len(preds) == 4:
                ph.frame_count = 4 * t
                ph(preds, is_multiview_video=True)
                preds.clear()

        preds = []
        ms = timed(reference_form, 8)
        res[f"cfg4_predict_T{t}_reference_form"] = {"video_frames_per_batch": t, "ms_per_batch": ms, "video_frames_per_s": 1e3 * t / ms,
                                                    "note": "eager; per-view normalise + stack + predict_step + host copy per batch + host per-view split"}
        del pool, views
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res["cfg4_predict_card"] = {"nvidia_smi": card, "torch_name": torch.cuda.get_device_name(0), "hbm_gbs_used": pk["hbm_gbs"]}


if sys.argv[1:2] == ["cfg4_predict"]:  # only the multi-view prediction entries; an optional second argument names a JSON file
    cfg4_predict()
    if len(sys.argv) > 2:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[2])), exist_ok=True)
        json.dump(res, open(sys.argv[2], "w"), indent=1)
    print(json.dumps(res, indent=1))
    sys.exit(0)


if sys.argv[1:2] == ["cfg3_context"]:  # only the context-prediction entries; an optional second argument names a JSON file
    cfg3_context()
    if len(sys.argv) > 2:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[2])), exist_ok=True)
        json.dump(res, open(sys.argv[2], "w"), indent=1)
    print(json.dumps(res, indent=1))
    sys.exit(0)

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

# config 5 with a crop-zoom pose model: 96-frame chunks of 1024x1024 uint8 frames, each cropped to a random in-frame box
# (sides 256-896 px) and resized to the 384x384 model input.  Bytes model of the crop kernel: output bytes plus the input
# bytes its bilinear taps touch, at most min(crop side, 2 x output side) rows and columns of the crop per frame.  The
# reference's path is its own crop_and_resize_frames (the staged oracle/_ref copy) on full-resolution normalised fp32
# frames (what its DALI pipeline hands over), with that normalisation (torch, eager) timed as well.
import pandas as pd  # noqa: E402

from oracle import ref_loader  # noqa: E402

cf_, cs_, cside_ = 96, 1024, 384
gen = torch.Generator(device=dev).manual_seed(51)
u8_pool = [torch.randint(0, 256, (cf_, cs_, cs_, 3), dtype=torch.uint8, device=dev, generator=gen) for _ in range(2)]
n_crop = cf_ * 20
side = torch.randint(256, 897, (n_crop, 2), device=dev, generator=gen).float()
origin = torch.rand(n_crop, 2, device=dev, generator=gen) * (cs_ - side)
boxes_c = torch.stack([origin[:, 0].floor(), origin[:, 1].floor(), side[:, 0], side[:, 1]], 1).contiguous()  # x, y, h, w
bx = boxes_c[:cf_]
touched = (torch.clamp(bx[:, 2], max=2 * cside_) * torch.clamp(bx[:, 3], max=2 * cside_)).sum().item() * 3
for tag, dt, cl in (("fchw_f32", torch.float32, False), ("fchw_bf16", torch.bfloat16, False), ("fhwc_bf16", torch.bfloat16, True)):
    out_bytes = cf_ * 3 * cside_ * cside_ * (4 if dt == torch.float32 else 2)
    ms, med = bench.time_stage(lambda: ops.frames_crop_normalize(u8_pool[0], bx, (cside_, cside_), channels_last=cl, dtype=dt), flush)
    res[f"cfg5_crop_kernel_{tag}"] = {"frames": cf_, "ms": ms, "ms_median": med, "bytes_model": out_bytes + touched,
                                     "gbs": (out_bytes + touched) / ms / 1e6, "frac_hbm": (out_bytes + touched) / ms / 1e6 / pk["hbm_gbs"]}
ref_bboxes = ref_loader.load("lightning_pose.data.bboxes")
rows_df = pd.DataFrame(bx.cpu().numpy().astype(np.float64), columns=["x", "y", "h", "w"])
mean_t, std_t = torch.tensor(ops.IMAGENET_MEAN, device=dev)[:, None, None], torch.tensor(ops.IMAGENET_STD, device=dev)[:, None, None]
full_f32 = (u8_pool[0].permute(0, 3, 1, 2).float() / 255.0 - mean_t) / std_t
with torch.no_grad():
    ms_n, _ = bench.time_stage(lambda: (u8_pool[0].permute(0, 3, 1, 2).float() / 255.0 - mean_t) / std_t, flush, reps=5, warmup=1)
    ms_c, _ = bench.time_stage(lambda: ref_bboxes.crop_and_resize_frames(full_f32, rows_df, [cside_, cside_]), flush, reps=5, warmup=1)
    ref_out, ref_boxes = ref_bboxes.crop_and_resize_frames(full_f32, rows_df, [cside_, cside_])
    mine, mine_boxes = ops.frames_crop_normalize(u8_pool[0], bx, (cside_, cside_))
del full_f32
res["cfg5_crop_reference"] = {"frames": cf_, "normalise_ms": ms_n, "crop_and_resize_frames_ms": ms_c, "total_ms": ms_n + ms_c,
                              "max_abs_diff_vs_kernel": float((ref_out - mine).abs().max()), "boxes_equal": bool(torch.equal(ref_boxes, mine_boxes)),
                              "note": "reference crop_and_resize_frames (staged oracle/_ref) on fp32 full-resolution frames; normalisation in eager torch"}
del ref_out
head_c = head_for("resnet50", 2048)
head_c.eval()
sel, scl = torch.arange(2048, device=dev) % 3, torch.randn(2048, device=dev)[None, :, None, None]


def backbone(fr):  # stand-in backbone (elementwise): (T, 3, 384, 384) -> (T, 2048, 12, 12) bf16
    return (torch.nn.functional.avg_pool2d(fr.float(), 32)[:, sel] * scl).bfloat16()


for mode in ("on", "off"):
    kw = {"bboxes": boxes_c, "frame_hw": (cs_, cs_)} if mode == "on" else {}
    fo = backbone if mode == "on" else (lambda u8: backbone(ops.frames_normalize(u8, size=(cside_, cside_))))
    bp = BatchedPredictor(head_c, K, n_crop, cf_, (cside_, cside_), features_of=fo, **kw)
    bp.feed(u8_pool[0])  # capture / warm
    bp.cursor.zero_()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n_crop // cf_):
        bp.feed(u8_pool[i % 2])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (n_crop // cf_)
    res[f"cfg5_crop_predictor_chunk_crop_{mode}"] = {
        "frames_per_chunk": cf_, "ms_per_chunk": ms, "launches_per_chunk": bp.launches_per_chunk,
        "note": "graph replay per chunk incl. the D2D copy of the uint8 chunk into the graph's input; crop off = the same uint8 chunk "
                "resized whole (lpb_frames_normalize); stand-in elementwise backbone, random head weights"}
card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
res["cfg5_crop_card"] = {"nvidia_smi": card, "torch_name": torch.cuda.get_device_name(0)}
cfg3_context()
cfg4_predict()
cfg2_unlabeled_aug()

os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", "r02_configs.json"), "w"), indent=1)
print(json.dumps(res, indent=1))
