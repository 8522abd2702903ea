"""Per-call latency of FramePredictor.predict_frame, from a host numpy frame to the returned dict, against the
reference's own form restated (cv2.resize and numpy on the host, one host -> device copy, the eager model, .cpu()).

    python scripts/bench_predict_frame.py [--calls 1000] [--warmup 50] [--out result.json]

Cases (the backbone of bench_sharded_predict.py's end-to-end row: torchvision ResNet-50, random init, bf16,
channels-last; K = 17):
  cfg2        a 384 x 384 model on 1024 x 1280 camera frames, without a box
  cfg2_box    the same with a (x, y, w, h) = (300, 200, 600, 500) box
  cfg3_ctx    a context (MHCRNN) model on 5 frames of 1024 x 1280 resized to 256 x 256
Each call ends in a device synchronise, so a host clock around it is the call's latency: median and p99 of ``--calls``
calls after ``--warmup``.  The ingest kernel alone is timed with CUDA events over graph replays of 100 launches.  The
card's name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lightning_pose_b200 import ops  # noqa: E402
from lightning_pose_b200.utils.predictions import FramePredictor  # noqa: E402

K = 17
FRAME_HW = (1024, 1280)


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if out else {"nvidia_smi": "unavailable"}


def trunk(dev):
    import torchvision

    torch.manual_seed(0)
    net = torchvision.models.resnet50()
    return torch.nn.Sequential(*list(net.children())[:-2]).to(dev, torch.bfloat16).to(memory_format=torch.channels_last).eval()


def tracker(context: bool, dev):
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import HeatmapTrackerMHCRNN

    bb = trunk(dev)
    if context:
        return HeatmapTrackerMHCRNN(K, backbone=bb, backbone_arch="resnet50", num_fc_input_features=2048).to(dev).eval()
    return HeatmapTracker(K, backbone=bb, num_fc_input_features=2048).to(dev).eval()


def latency(fn, calls: int, warmup: int) -> dict:
    for _ in range(warmup):
        fn()
    ts = np.empty(calls)
    for i in range(calls):
        t0 = time.perf_counter()
        fn()
        ts[i] = time.perf_counter() - t0
    return {"median_ms": float(np.median(ts) * 1e3), "p99_ms": float(np.percentile(ts, 99) * 1e3), "calls": calls}


def reference_form(tr, image_hw, context: bool, dev):
    """Model.predict_frame restated (api/model.py:388-509): numpy crop, cv2.resize + numpy normalisation, one H2D copy,
    the eager model on bf16 channels-last images, .cpu()."""
    import cv2

    mean, std = np.array(ops.IMAGENET_MEAN, np.float32), np.array(ops.IMAGENET_STD, np.float32)
    h, w = image_hw

    def pre(img):
        t = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR).astype(np.float32) / 255.0
        return np.transpose((t - mean) / std, (2, 0, 1))

    def run(frame, box):
        if box is not None:
            bx, by, bw, bh = box
            crop = frame[..., by : by + bh, bx : bx + bw, :]
            bbox = [bx, by, crop.shape[-3], crop.shape[-2]]
        else:
            crop, bbox = frame, [0, 0, frame.shape[-3], frame.shape[-2]]
        x = np.stack([pre(c) for c in crop]) if context else pre(crop)[None]
        images = torch.from_numpy(x).to(dev).to(torch.bfloat16)
        images = images.contiguous(memory_format=torch.channels_last) if not context else images
        images = images[None] if context else images
        batch = {"images": images, "keypoints": torch.zeros(1, 2 * K, device=dev), "heatmaps": torch.zeros(1, K, 1, 1, device=dev),
                 "bbox": torch.tensor([bbox], dtype=torch.float32, device=dev)}
        with torch.inference_mode():
            res = tr.get_loss_inputs_labeled(batch)
        kp, cf = res["keypoints_pred"], res["confidences"]
        if context:
            pick = cf[1:] > cf[:1]
            kp = torch.where(pick[..., None], kp[1:].reshape(1, K, 2), kp[:1].reshape(1, K, 2))
            cf = torch.where(pick, cf[1:], cf[:1])
        return kp[0].cpu().numpy().reshape(-1, 2), cf[0].cpu().numpy()

    return run


def ingest_kernel_us(frames_np, box, image_hw, channels_last, dev, reps=100, rounds=20) -> float:
    """The ingest alone: CUDA events around graph replays of ``reps`` back-to-back launches."""
    x = torch.from_numpy(frames_np).to(dev)
    b = torch.tensor(box, dtype=torch.int32, device=dev)
    shape = (x.shape[0], *image_hw, 3) if channels_last else (x.shape[0], 3, *image_hw)
    out = torch.empty(shape, dtype=torch.bfloat16, device=dev)
    bbox = torch.empty((1, 4), dtype=torch.float32, device=dev)
    call = lambda: ops.frames_crop_resize_cv2(x, image_hw, b, channels_last=channels_last, dtype=torch.bfloat16, out=out, bbox_out=bbox)  # noqa: E731
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            call()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(rounds):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * rounds)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict_frame: no CUDA device")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    res = {"card": card(), "torch_name": torch.cuda.get_device_name(0)}
    cases = {"cfg2": (False, (384, 384), None), "cfg2_box": (False, (384, 384), (300, 200, 600, 500)),
             "cfg3_ctx": (True, (256, 256), None)}
    for name, (context, image_hw, box) in cases.items():
        tr = tracker(context, dev)
        frame = rng.integers(0, 256, ((5,) if context else ()) + (*FRAME_HW, 3), dtype=np.uint8)
        fp = FramePredictor(tr.head, K, image_hw, features_of=tr.backbone, dtype=torch.bfloat16, channels_last=True)
        row = {"predict_frame": latency(lambda: fp.predict_frame(frame, bbox=box), args.calls, args.warmup),
               "launches_per_call": fp.launches_per_call}
        whole = (0, 0, FRAME_HW[1], FRAME_HW[0])
        row["ingest_kernel_us"] = ingest_kernel_us(frame if context else frame[None], box or whole, image_hw, True, dev)
        try:
            ref = reference_form(tr, image_hw, context, dev)
        except ImportError:
            row["reference_form"] = "not measured (no cv2)"
        else:
            row["reference_form"] = latency(lambda: ref(frame, box), args.calls, args.warmup)
            got = fp.predict_frame(frame, bbox=box)
            kp_ref, _ = ref(frame, box)
            # the reference form runs bf16 images converted from fp32 numpy on the host, the predictor the same
            # normalised values rounded on the device: the keypoints agree to the head's bf16 accuracy
            row["max_abs_keypoint_diff_px_vs_reference_form"] = float(np.nanmax(np.abs(got["keypoints"] - kp_ref)))
        res[name] = row
        print(name, json.dumps(row), flush=True)
        del tr, fp
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
