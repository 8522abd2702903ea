"""Per-call latency of FramePredictor.push_frame (one new frame per call, a context model's last frames kept on the
device) against predict_frame on the five-frame stack, from a host numpy frame to the returned dict.

    python scripts/bench_predict_stream.py [--calls 1000] [--warmup 50] [--out result.json]

The setup of bench_predict_frame.py's context case: torchvision ResNet-50 (random init, bf16, channels-last), K = 17,
1024 x 1280 camera frames, a config-3 context (MHCRNN) model at 256 x 256, without a box and with the (x, y, w, h) =
(300, 200, 600, 500) box.  Each call ends in a device synchronise, so a host clock around it is the call's latency:
median and p99 of ``--calls`` calls after ``--warmup``.  The pushes cycle through 16 distinct frames, and predict_frame
gets the matching five-frame windows.  Kernels per call are the captured graphs' kernel nodes.  After the timed calls
the last push is compared with predict_frame on its five frames.  The card's name, power limit and SM clocks are read
in the same run.
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

from bench_predict_frame import FRAME_HW, K, card, latency, tracker  # noqa: E402
from lightning_pose_b200.utils.predictions import FramePredictor  # noqa: E402

IMAGE_HW = (256, 256)
POOL = 16


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict_stream: no CUDA device")
    dev = torch.device("cuda:0")
    pool = np.random.default_rng(0).integers(0, 256, (POOL, *FRAME_HW, 3), dtype=np.uint8)
    windows = [pool[np.arange(i - 4, i + 1) % POOL] for i in range(POOL)]  # frames i - 4 .. i, contiguous copies
    res = {"card": card(), "torch_name": torch.cuda.get_device_name(0)}
    for name, box in (("cfg3_ctx", None), ("cfg3_ctx_box", (300, 200, 600, 500))):
        tr = tracker(True, dev)
        kw = dict(features_of=tr.backbone, dtype=torch.bfloat16, channels_last=True)
        stream, single = FramePredictor(tr.head, K, IMAGE_HW, **kw), FramePredictor(tr.head, K, IMAGE_HW, **kw)
        n = {"push": 0, "stack": 0}

        def push():
            stream.push_frame(pool[n["push"] % POOL], bbox=box)
            n["push"] += 1

        def stack():
            single.predict_frame(windows[n["stack"] % POOL], bbox=box)
            n["stack"] += 1

        row = {"push_frame": latency(push, args.calls, args.warmup), "launches_per_push": stream.launches_per_push,
               "predict_frame_5": latency(stack, args.calls, args.warmup), "launches_per_call": single.launches_per_call}
        i = n["push"]
        got = stream.push_frame(pool[i % POOL], bbox=box)
        want = single.predict_frame(windows[i % POOL], bbox=box)  # stream frames i - 4 .. i
        assert got["frame"] == i - 2
        row["bit_identical_to_predict_frame"] = bool(np.array_equal(got["keypoints"], want["keypoints"])
                                                     and np.array_equal(got["confidence"], want["confidence"]))
        row["max_abs_keypoint_diff_px_vs_predict_frame"] = float(np.nanmax(np.abs(got["keypoints"] - want["keypoints"])))
        row["max_confidence"] = float(np.nanmax(want["confidence"]))
        # predict_frame runs the backbone on five frames at once, a push on one: the same bits only if a frame's
        # features do not depend on the batch
        x = torch.from_numpy(windows[0]).to(dev).permute(0, 3, 1, 2).float().div(255).to(torch.bfloat16)
        x = x.contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            row["backbone_batch_independent"] = bool(torch.equal(tr.backbone(x), torch.cat([tr.backbone(x[j : j + 1]) for j in range(5)])))
        res[name] = row
        print(name, json.dumps(row), flush=True)
        del tr, stream, single
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
