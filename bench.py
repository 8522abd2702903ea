#!/usr/bin/env python
"""Benchmark of the lightning-pose hot path on H100.

Workload = BASELINE.json configs[1]: ResNet-50 semi-supervised (temporal + PCA losses), synthetic
384x384 video, 17 keypoints.  One *step* = one pass of the hot path over one batch of synthetic
backbone features: per clip 16 labeled frames + 32 unlabeled frames ->
  head (PixelShuffle + 2 deconvs + softmax) on all frames
  -> labeled: fused Gaussian-target generation + heatmap MSE; soft-argmax decode
  -> unlabeled: soft-argmax decode -> affine undo + model->frame remap -> temporal + PCA losses
  -> backward of all of the above into the features and the head parameters (unless --fwd-only).
`value` is frames/s with the features resident in HBM; `e2e` repeats the same step from pinned host
buffers through the public API (H2D of the features and D2H of the loss scalars inside the timed region).

`--impl reference` times the CPU oracle (the restated reference path, all host threads) on a bounded
sample of the same workload.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

K_PTS, IMG, FEAT_C, FEAT_HW, HM = 17, 384, 2048, 12, 96
B_LABELED, T_UNLABELED = 16, 32  # config_default.yaml: train_batch_size 16, dali.base.train.sequence_length 32
METRIC = "train frames/sec at 384x384x17kpt (hot path: head+targets+decode+losses)"


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))), "measured"
    except Exception:
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "fallback"  # H100 SXM data sheet (dense)


class ClockSampler:
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index: int):
        self.rows, self.proc, self.index = [], None, index

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.index), "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None
        return self

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def __exit__(self, *a):
        if self.proc:
            time.sleep(0.15)
            self.proc.terminate()

    def summary(self):
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx.append(float(r[1]))
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unsampled"]}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


def _inverse_pixel_shuffle(xs: torch.Tensor) -> torch.Tensor:
    """(N, C, 2H, 2W) -> (N, 4C, H, W) with out[4c + 2di + dj, i, j] = xs[c, 2i+di, 2j+dj]."""
    return torch.nn.functional.pixel_unshuffle(xs, 2)


def make_problem(n_clips: int, seed: int, device, regime: str = "trained"):
    """Seeded synthetic inputs of BASELINE configs[1] (no datasets / checkpoints are reachable).  Plain tensors only:
    both arms (ours, the reference on the CPU) build their own head from ``head_params``.

    regime "trained": what the semi-supervised phase of training sees - unimodal, Gaussian-like heatmaps
      (peak ~0.1, sigma ~1.25 heatmap px, cf. SURVEY 8(d) "peaked").  Built by construction, since the head is
      linear: the two deconvs carry 2x-bilinear kernels routed per keypoint (+1e-3 noise) and the features carry a
      planted non-negative response bump per keypoint (+ N(0, 0.1) noise); unlabeled clips follow a random walk.
    regime "fresh": the reference's own initialiser (xavier-uniform gain 0.01, zero bias) on randn*0.5 features
      -> flat heatmaps, for which the soft-argmax has to evaluate the whole 384x384 field.
    """
    g = torch.Generator().manual_seed(seed)
    n_lab, n_unl = n_clips * B_LABELED, n_clips * T_UNLABELED
    n_frames = n_lab + n_unl
    torch.manual_seed(seed)
    c4, hs = FEAT_C // 4, 2 * FEAT_HW
    # reference initialiser (models/heads/heatmap.py:74-83): xavier-uniform gain 0.01, zero bias
    w1 = torch.nn.init.xavier_uniform_(torch.empty(c4, K_PTS, 3, 3), gain=0.01)
    w2 = torch.nn.init.xavier_uniform_(torch.empty(K_PTS, K_PTS, 3, 3), gain=0.01)
    b1, b2 = torch.zeros(K_PTS), torch.zeros(K_PTS)
    # keypoints in heatmap pixels: labeled uniform, unlabeled = per-clip random walk
    kp_hm = torch.empty(n_frames, K_PTS, 2)
    kp_hm[:n_lab] = torch.rand(n_lab, K_PTS, 2, generator=g) * 80 + 8
    walk = torch.cumsum(torch.randn(n_clips, T_UNLABELED, K_PTS, 2, generator=g) * 0.6, dim=1)
    kp_hm[n_lab:] = (torch.rand(n_clips, 1, K_PTS, 2, generator=g) * 60 + 18 + walk).clamp(6, 90).reshape(n_unl, K_PTS, 2)
    feats = torch.empty((n_frames, FEAT_C, FEAT_HW, FEAT_HW), dtype=torch.float32)
    if regime == "trained":
        tri = torch.tensor([[0.25, 0.5, 0.25], [0.5, 1.0, 0.5], [0.25, 0.5, 0.25]])
        group = torch.arange(c4) % K_PTS
        w1 = torch.randn(w1.shape, generator=g) * 1e-3
        w1[torch.arange(c4), group] += tri / (c4 // K_PTS)
        w2 = torch.randn(w2.shape, generator=g) * 1e-3
        w2[torch.arange(K_PTS), torch.arange(K_PTS)] += tri
        centre = torch.arange(hs, dtype=torch.float32) * 4 + 1.5  # heatmap position of a shuffled pixel
        for i in range(0, n_frames, 64):  # bounded temp memory
            kp = kp_hm[i : i + 64]
            dy = (centre[None, None, :, None] - kp[:, :, 1, None, None]) ** 2
            dx = (centre[None, None, None, :] - kp[:, :, 0, None, None]) ** 2
            q = torch.exp(-(dy + dx) / (2 * 4.3**2))  # (n, K, 24, 24) planted response: logit bump, sigma_eff ~1.25 px
            q = q * (13.0 / q.amax(dim=(2, 3), keepdim=True))  # peak logit 13 -> heatmap peak ~0.1-0.25 like a trained net
            xs = q[:, group] + torch.randn((kp.shape[0], c4, hs, hs), generator=g) * 0.1
            feats[i : i + 64] = _inverse_pixel_shuffle(xs)
    else:
        for i in range(0, n_frames, 64):
            feats[i : i + 64] = torch.randn((min(64, n_frames - i), FEAT_C, FEAT_HW, FEAT_HW), generator=g) * 0.5
    kp_lab = kp_hm[:n_lab] * (IMG / HM) + torch.randn(n_lab, K_PTS, 2, generator=g) * 2.0  # labels in image pixels
    kp_lab[torch.rand(n_lab, K_PTS, generator=g) < 0.1] = float("nan")
    vis = torch.randint(0, 3, (n_lab, K_PTS), generator=g)
    ang = np.deg2rad(float(torch.rand(1, generator=g)) * 20 - 10)
    sc = 0.8 + 0.4 * float(torch.rand(1, generator=g))
    tf = torch.tensor([[sc * np.cos(ang), -sc * np.sin(ang), 4.0], [sc * np.sin(ang), sc * np.cos(ang), -3.0]], dtype=torch.float32)
    bbox = torch.tensor([[0.0, 0.0, 406.0, 396.0]]).repeat(n_unl, 1)
    # PCA parameters: rank-6 latent pose + noise (SURVEY 8(d)), all 17 keypoints
    lat = torch.randn(500, 6, generator=g) @ torch.randn(6, 2 * K_PTS, generator=g) * 20 + 200 + torch.randn(500, 2 * K_PTS, generator=g) * 2
    mean = lat.mean(0)
    _, _, vt = torch.linalg.svd(lat - mean, full_matrices=False)
    pca = {"mean": mean, "kept": vt[:6].contiguous(), "eps": 5.0}
    return {"head_params": (w1, b1, w2, b2), "feats": feats, "kp_lab": kp_lab, "vis": vis, "tf": tf, "bbox": bbox, "pca": pca, "n_clips": n_clips}


# ------------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------------
BACKBONE_PARAMS = 23_508_032  # ResNet-50 trunk (SURVEY 8(e): 94.4 MB of fp32 gradients per step with the head's 80,971)


class HotPath:
    # our own kernel launches per step, counted from the launch sites of the step's code path; library kernels of torch
    # (a dozen scalar element-wise ops, NCCL) are not counted
    # per head call: preparation (packs + pads) + k1a + banded layer 2 (one two-pass softmax kernel from 132 frames up) +
    # decode (warp kernel + queued CTA kernel) = 5;  labeled: + fused targets/MSE + its final reduction (2);
    # unlabeled: + remap + unsupervised losses (2)
    LAUNCHES_FWD = 2 * 5 + 2 + 2
    # unlabeled: unsup bwd, remap bwd, decode windows + dense fallback (4), then per head backward: preparation, plane dots,
    # G2 front end, wgrad2, dgrad2, wgrad1, dgrad1 = 7, + the fixed-order sums of dW2, db2, db1, dW1 (4), + the window patch
    # pass (1);  labeled: targets/MSE bwd + the same 7 + 4
    LAUNCHES_BWD = (4 + 7 + 4 + 1) + (1 + 7 + 4) + 1  # + the Adam step

    def __init__(self, prob, device, fwd_only: bool, world: int = 1, ddp_payload_floats: int = 0, two_streams: bool = True):
        from lightning_pose_b200 import ops
        from lightning_pose_b200.ddp import FlatGradAllReducer
        from lightning_pose_b200.models.heads.heatmap import HeatmapHead

        self.ops, self.dev, self.fwd_only = ops, device, fwd_only
        self.n_clips = prob["n_clips"]
        self.head = HeatmapHead("resnet50", FEAT_C, K_PTS)
        d1, d2 = list(self.head.upsampling_layers)[1:]
        with torch.no_grad():
            w1, b1, w2, b2 = prob["head_params"]
            d1.weight.copy_(w1), d1.bias.copy_(b1), d2.weight.copy_(w2), d2.bias.copy_(b2)
        self.head = self.head.to(device)
        self.kp_lab = prob["kp_lab"].to(device)
        self.vis = prob["vis"].to(device)
        self.tf = prob["tf"].to(device)
        self.bbox = prob["bbox"].to(device)
        self.sv = ops.PcaParams(np.arange(K_PTS, dtype=np.int32), K_PTS, 0, None, prob["pca"]["mean"], prob["pca"]["kept"], prob["pca"]["eps"], device)
        self.teps = torch.full((K_PTS,), 20.0, device=device)
        self.w_unsup = 1.0 / (2.0 * np.exp(5.0))
        self.reducer = None
        self.two_streams = two_streams
        self.side = torch.cuda.Stream(device=device) if two_streams else None
        if two_streams and hasattr(torch.autograd.graph, "set_warn_on_accumulate_grad_stream_mismatch"):
            # the head's parameters receive gradients from two streams on purpose (the engine orders them with events)
            torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)
        if not fwd_only:
            from lightning_pose_b200.optim import FusedAdam
            self.opt = FusedAdam(self.head.parameters(), lr=1e-5)  # torch.optim.Adam semantics, one native launch
            if world > 1:
                self.reducer = FlatGradAllReducer(self.head.parameters(), n_scalars=4, extra_floats=ddp_payload_floats)

    def forward_backward(self, feats: torch.Tensor):
        ops, n = self.ops, self.n_clips
        nl = n * B_LABELED
        # the reference runs the labeled and the unlabeled batch through the model separately
        # (heatmap_tracker.py:163-179, :299-340): two feature tensors, two head calls
        f_lab, f_unl = feats[:nl].detach(), feats[nl:].detach()
        if not self.fwd_only:
            f_lab.requires_grad_(True)  # d loss / d features feeds the backbone's backward
            f_unl.requires_grad_(True)
        cur = torch.cuda.current_stream(self.dev)
        with torch.set_grad_enabled(not self.fwd_only):
            if self.two_streams:
                # the labeled and the unlabeled chain share nothing until the loss sum: fork the labeled one onto a second
                # stream (autograd replays each node's backward on its forward stream, so the two backward chains overlap too)
                self.side.wait_stream(cur)
                with torch.cuda.stream(self.side):
                    hm_lab, _kp_lab, _cf_lab = self.head.forward_with_keypoints(f_lab)
                    l_sup = ops.heatmap_mse_from_keypoints(self.kp_lab, hm_lab, IMG, IMG, visibility=self.vis)
            else:
                hm_lab, _kp_lab, _cf_lab = self.head.forward_with_keypoints(f_lab)  # (n*16, 17, 96, 96); keypoints -> rmse metric
                l_sup = ops.heatmap_mse_from_keypoints(self.kp_lab, hm_lab, IMG, IMG, visibility=self.vis)
            _hm_unl, kp, cf = self.head.forward_with_keypoints(f_unl)  # (n*32, ...)
            kp_unl = ops.remap_keypoints(kp, self.tf, self.bbox, IMG, IMG)
            per_clip = ops.unsup_losses(kp_unl.reshape(n, T_UNLABELED, 2 * K_PTS), cf.reshape(n, T_UNLABELED, K_PTS),
                                        temporal_eps=self.teps, prob_threshold=0.05, pca_singleview=self.sv)
            if self.two_streams:
                cur.wait_stream(self.side)
                for t in (hm_lab, l_sup, f_lab):
                    t.record_stream(cur)
            total = 0.5 * l_sup + self.w_unsup * per_clip[:, :2].sum()
        scalars = [total.detach(), l_sup.detach(), per_clip[:, 0].mean().detach(), per_clip[:, 1].mean().detach()]
        if not self.fwd_only:
            total.backward()
        return scalars

    def step(self, feats: torch.Tensor):
        if not self.fwd_only:
            if self.reducer is not None:
                self.reducer.begin_step()  # gradients accumulate straight into the flat buffer; backbone bucket starts
            else:
                self.opt.zero_grad(set_to_none=True)
        scalars = self.forward_backward(feats)
        if not self.fwd_only:
            if self.reducer is not None:
                out = self.reducer.finish_step(scalars)  # head bucket (+ logged scalars) after the backward
                self.opt.step()
                self.last_out = out
                return out
            self.opt.step()
        self.last_out = torch.stack(scalars)
        return self.last_out

    def dump_outputs(self, out_dir: str, scalars: torch.Tensor) -> None:
        """What the timed step hands its caller after the last timed step, as float32 .npy files: the four logged loss
        scalars (total, supervised, temporal, PCA) and the head's parameters (updated by the Adam step) and gradients."""
        os.makedirs(out_dir, exist_ok=True)
        arrays = {"losses": scalars}
        for name, p in self.head.named_parameters():
            arrays[f"param.{name}"] = p
            if p.grad is not None:
                arrays[f"grad.{name}"] = p.grad
        for name, t in arrays.items():
            np.save(os.path.join(out_dir, f"{name}.npy"), t.detach().float().cpu().numpy())


class GraphedStep:
    """The whole training step (forward, backward, all-reduce, Adam) captured once into a CUDA graph and replayed:
    the step is ~60 short launches, so launch latency is a visible share of it.  The input tensor is static (the
    resident feature buffer); the returned scalars live in the graph's pool."""

    def __init__(self, hp: "HotPath", feats: torch.Tensor):
        self.feats = feats
        side = torch.cuda.Stream(device=feats.device)
        side.wait_stream(torch.cuda.current_stream(feats.device))
        with torch.cuda.stream(side):
            for _ in range(3):
                hp.step(feats)
        torch.cuda.current_stream(feats.device).wait_stream(side)
        torch.cuda.synchronize(feats.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = hp.step(feats)

    def __call__(self):
        self.graph.replay()
        return self.out


def _teardown(dist, rank: int, world: int) -> None:
    """End of a multi-rank run.  The step lives in a captured CUDA graph that holds NCCL kernels; tearing the
    process group down underneath it can block, and nothing is left to do anyway: the ranks meet on the rendezvous
    store (no collective), and every process leaves with exit code 0 without running the NCCL destructors."""
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    sys.stdout.flush()
    sys.stderr.flush()
    try:
        store = dist.distributed_c10d._get_default_store()
        store.add("lpb_bench_done", 1)
        if rank == 0:  # the store lives in rank 0: leave last
            deadline = time.time() + 120.0
            while int(store.add("lpb_bench_done", 0)) < world and time.time() < deadline:
                time.sleep(0.05)
    except Exception:
        pass
    os._exit(0)


def _wait_for_rank0(dist, timeout_s: float = 900.0) -> None:
    """Ranks != 0 idle (no GPU work, no collective) until rank 0 has finished its single-GPU breakdown, so that nothing
    tears down or competes for the NVSwitch / host while rank 0 is still timing kernels."""
    try:
        store = dist.distributed_c10d._get_default_store()
        deadline = time.time() + timeout_s
        while int(store.add("lpb_rank0_done", 0)) < 1 and time.time() < deadline:
            time.sleep(0.05)
    except Exception:
        pass


def time_steps(fn, steps, warmup, barrier=None):
    for _ in range(warmup):
        fn()
    if barrier:
        barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    if barrier:
        barrier()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


class L2Flusher:
    """Writes a buffer larger than the L2 (50 MB on an H100) between timed repetitions of a single stage."""

    def __init__(self, dev, mib: int = 256):
        self.buf = torch.empty(mib * 2**20 // 4, dtype=torch.float32, device=dev)
        self.k = 0

    def __call__(self):
        self.k += 1
        self.buf.fill_(float(self.k & 7))


def time_stage(fn, flush, reps=20, warmup=3):
    """Mean device time of ``fn`` (CUDA events on the launching stream), L2 flushed before every repetition; the
    flush itself is outside the event pair."""
    for _ in range(warmup):
        fn()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    torch.cuda.synchronize()
    for e0, e1 in evs:
        flush()
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    ts = sorted(e0.elapsed_time(e1) for e0, e1 in evs)
    return float(np.mean(ts)), float(ts[len(ts) // 2])


# algorithmic HBM bytes per frame (SURVEY 8(d), K = 17, 384^2, ds = 2; DESIGN.md section 4 restates them)
HM_BYTES = K_PTS * HM * HM * 4          # one frame of fp32 heatmaps: 626,688
KP_BYTES = K_PTS * 12                   # x, y, confidence


def kernel_breakdown(hp: "HotPath", feats, reps=20):
    """Per-stage device time for the roofline line: every forward AND backward stage of the step, each timed alone
    with the L2 flushed before every repetition.  Returns {stage: {ms, ms_median, algorithmic_bytes, gbs}}."""
    ops, n = hp.ops, hp.n_clips
    nf, nl = feats.shape[0], hp.n_clips * B_LABELED
    nu = nf - nl
    fb = FEAT_C * FEAT_HW * FEAT_HW * feats.element_size()  # feature bytes per frame
    flush = L2Flusher(feats.device)
    out = {}

    def add(name, fn, nbytes, what):
        ms, med = time_stage(fn, flush, reps)  # rates use the MEDIAN of the repetitions (robust to a stray slow repetition)
        out[name] = {"ms": med, "ms_mean": ms, "algorithmic_bytes": nbytes, "gbs": nbytes / med / 1e6, "what": what}

    with torch.no_grad():
        # the two halves of HeatmapHead.forward_with_keypoints as the step runs them: on the bf16 path the head's softmax pass
        # also writes the per-plane decode hints (16 B per plane) and the decode consumes them
        hints = None
        if feats.dtype == torch.bfloat16:
            d1, d2 = list(hp.head.upsampling_layers)[1:]
            wts, bss = [d1.weight, d2.weight], [d1.bias, d2.bias]
            head_fn = lambda: ops._head_forward_bf16(feats, wts, bss, True, want_hints=True)
            hm, hints = head_fn()
        else:
            head_fn = lambda: hp.head(feats)
            hm = head_fn()
        kp, cf, _ = ops.decode_forward_hinted(hm, 2, 1000.0, hints)
        kp = kp.reshape(nf, -1)
        add("head_fwd", head_fn, nf * (fb + HM_BYTES), "K1: features -> normalised heatmaps (+ decode hints), inference form (k1a + banded layer 2)")
        add("decode_fwd", lambda: ops.decode_forward_hinted(hm, 2, 1000.0, hints), nf * (HM_BYTES + KP_BYTES),
            "K2: heatmaps (+ hints) -> (x, y, confidence)")
        add("target_mse_fwd", lambda: ops.heatmap_mse_from_keypoints(hp.kp_lab, hm[:nl], IMG, IMG, visibility=hp.vis),
            nl * (HM_BYTES + KP_BYTES), "K3: fused Gaussian targets + heatmap MSE (labeled frames)")
        add("unsup_losses_fwd", lambda: ops.unsup_losses(kp[nl:].reshape(n, T_UNLABELED, -1), cf[nl:].reshape(n, T_UNLABELED, -1),
                                                       temporal_eps=hp.teps, prob_threshold=0.05, pca_singleview=hp.sv),
            nu * KP_BYTES, "K4: remapped keypoints -> temporal + PCA losses")
    if not hp.fwd_only:
        params = list(hp.head.parameters())
        # labeled branch: dense heatmap-loss gradient -> G2 front end -> wgrad/dgrad of both deconvs
        f_lab = feats[:nl].detach().requires_grad_(True)
        hm_lab, _, _ = hp.head.forward_with_keypoints(f_lab)
        l_sup = ops.heatmap_mse_from_keypoints(hp.kp_lab, hm_lab, IMG, IMG, visibility=hp.vis)
        g_hm = torch.autograd.grad(l_sup, hm_lab, retain_graph=True)[0]
        add("target_mse_bwd", lambda: torch.autograd.grad(l_sup, hm_lab, retain_graph=True), nl * 2 * HM_BYTES,
            "K3 backward: heatmaps -> d heatmaps (dense)")
        add("head_bwd_labeled", lambda: torch.autograd.grad(hm_lab, [f_lab] + params, g_hm, retain_graph=True),
            nl * (2 * HM_BYTES + 2 * fb), "K1 backward, dense form: (heatmaps, d heatmaps, features) -> d features + weight gradients")
        # unlabeled branch: keypoint gradient -> sparse decode windows -> G2 front end -> wgrad/dgrad
        f_unl = feats[nl:].detach().requires_grad_(True)
        _hm_u, kp_u, cf_u = hp.head.forward_with_keypoints(f_unl)
        kp_r = ops.remap_keypoints(kp_u, hp.tf, hp.bbox, IMG, IMG)
        per_clip = ops.unsup_losses(kp_r.reshape(n, T_UNLABELED, 2 * K_PTS), cf_u.reshape(n, T_UNLABELED, K_PTS),
                                    temporal_eps=hp.teps, prob_threshold=0.05, pca_singleview=hp.sv)
        l_uns = per_clip[:, :2].sum()
        g_kp = torch.autograd.grad(l_uns, kp_u, retain_graph=True)[0]
        add("unsup_losses_bwd", lambda: torch.autograd.grad(l_uns, kp_u, retain_graph=True), nu * 2 * KP_BYTES, "K4 backward (+ remap)")
        add("head_bwd_unlabeled", lambda: torch.autograd.grad(kp_u, [f_unl] + params, g_kp, retain_graph=True),
            nu * (HM_BYTES + 2 * fb), "K2 + K1 backward, sparse form: decode windows + (heatmaps, features) -> d features + weight gradients")
    return out


def run_ours(args):
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    dist = None
    if world > 1:
        import torch.distributed as dist_

        dist = dist_
        dist.init_process_group("nccl", device_id=dev)
    import lightning_pose_b200  # noqa: F401  (fails loudly without the CUDA library)

    prob = make_problem(args.clips, seed=1234 + rank, device=dev, regime=args.regime)
    payload = int(args.ddp_payload_mb * 1e6 / 4) if (world > 1 and not args.fwd_only) else 0
    hp = HotPath(prob, dev, args.fwd_only, world, ddp_payload_floats=payload, two_streams=not args.serial_chains)
    tdt = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    feats_host = prob["feats"].to(tdt).pin_memory()
    feats = feats_host.to(dev, non_blocking=True)
    esz = feats.element_size()
    n_frames = feats.shape[0]
    barrier = (lambda: dist.barrier()) if dist else None

    step_fn = lambda: hp.step(feats)
    graphed = False
    if args.profile_step:
        # for a run under ncu: W + K eager steps and nothing else (no stage breakdown, no e2e leg) -- not a bench line
        for _ in range(args.warmup):
            step_fn()
        torch.cuda.synchronize()
        kin = None
        if args.kineto:
            # in-situ kernel durations (CUPTI activity records: no replay, no cache flush, no serialisation beyond the
            # stream order) -- the complement of the ncu launch list, whose per-launch times are cold-cache
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    step_fn()
                torch.cuda.synchronize()
            kin = [{"kernel": e.key[:70], "calls": e.count, "us_per_step": round(e.device_time_total / args.steps, 2),
                    "us_per_call": round(e.device_time_total / max(e.count, 1), 2)}
                   for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total) if e.device_time_total > 0]
            try:  # the last step's launches in time order (name, us)
                from torch.autograd import DeviceType
                evs = sorted([e for e in prof.events() if e.device_type == DeviceType.CUDA], key=lambda e: e.time_range.start)
                per = len(evs) // args.steps
                kin = {"by_kernel": kin, "last_step": [[e.name[:60], round(e.time_range.elapsed_us(), 2)] for e in evs[len(evs) - per:]]}
            except Exception as exc:  # noqa: BLE001
                kin = {"by_kernel": kin, "last_step_error": repr(exc)}
        else:
            for _ in range(args.steps):
                step_fn()
            torch.cuda.synchronize()
        if rank == 0:
            print(json.dumps({"profile_step": True, "steps": args.steps, "warmup": args.warmup, "kineto": kin}))
        if dist:
            _teardown(dist, rank, world)
        return
    if not args.no_graph:
        try:
            step_fn = GraphedStep(hp, feats)
            graphed = True
        except Exception as exc:  # a failed capture leaves the process in an undefined state: start over without it
            sys.stderr.write(f"bench: CUDA-graph capture failed ({type(exc).__name__}: {exc}); re-running with --no-graph\n")
            sys.stderr.flush()
            os.execv(sys.executable, [sys.executable] + sys.argv + ["--no-graph"])
    with ClockSampler(local) as clk:
        ms = time_steps(step_fn, args.steps, args.warmup, barrier)
    if args.dump_outputs and rank == 0:
        hp.dump_outputs(args.dump_outputs, step_fn.out if graphed else hp.last_out)
    t = torch.tensor([ms], device=dev)
    if dist:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total = float(t)
    value = world * n_frames * args.steps / (ms_total / 1e3)

    # ---- e2e: pinned host features -> device inside the timed region, loss scalars read back -----
    dbuf = torch.empty_like(feats)
    losses_host = torch.empty(4, dtype=torch.float32).pin_memory()

    # The loader side of a training loop: batch i+1 is copied (pinned host -> device, own stream) while batch i
    # trains; all K copies and all K result read-backs happen inside the timed region.
    dbufs = [dbuf, torch.empty_like(feats)]
    copy_stream = torch.cuda.Stream(device=dev)
    copied = [torch.cuda.Event() for _ in range(2)]
    consumed = [torch.cuda.Event() for _ in range(2)]

    def e2e_run(n):
        main = torch.cuda.current_stream(dev)
        for i in range(n + 1):
            if i < n:  # stage batch i
                j = i % 2
                with torch.cuda.stream(copy_stream):
                    if i >= 2:
                        copy_stream.wait_event(consumed[j])
                    dbufs[j].copy_(feats_host, non_blocking=True)
                    copied[j].record(copy_stream)
            if i >= 1:  # train on batch i-1
                j = (i - 1) % 2
                main.wait_event(copied[j])
                out = hp.step(dbufs[j])
                consumed[j].record(main)
                losses_host.copy_(out, non_blocking=True)

    e2e_steps = max(2, min(args.steps, 6))
    e2e_run(2)  # warm-up
    if barrier:
        barrier()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    e2e_run(e2e_steps)
    ev1.record()
    if barrier:
        barrier()
    torch.cuda.synchronize()
    ms_e2e = ev0.elapsed_time(ev1)
    t = torch.tensor([ms_e2e], device=dev)
    if dist:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_value = world * n_frames * e2e_steps / (float(t) / 1e3)

    if rank != 0:
        if dist:
            _wait_for_rank0(dist)  # stay quiet while rank 0 times its single-GPU stages
            _teardown(dist, rank, world)
        return
    pk, pk_src = peaks()
    # single-GPU stage timings: a fresh single-rank HotPath (no collective inside), peers idle
    hp_b = HotPath(prob, dev, args.fwd_only, two_streams=not args.serial_chains) if world > 1 else hp
    br = kernel_breakdown(hp_b, feats)
    fwd_only_value = None
    if not args.fwd_only:
        hp_fwd = HotPath(prob, dev, True, two_streams=not args.serial_chains)
        fwd_fn = GraphedStep(hp_fwd, feats) if graphed else (lambda: hp_fwd.step(feats))
        ms_f = time_steps(fwd_fn, args.steps, 3)
        fwd_alg = n_frames * (FEAT_C * FEAT_HW * FEAT_HW * esz + HM_BYTES + KP_BYTES)  # SURVEY 8(d) "fused path total, training fwd"
        fwd_only_value = {"value": n_frames * args.steps / (ms_f / 1e3), "unit": "frames/s", "ms_per_step": ms_f / args.steps,
                          "algorithmic_bytes_per_step": fwd_alg, "frac_hbm": fwd_alg * args.steps / ms_f / 1e6 / pk["hbm_gbs"]}
    flat = None
    if not args.no_flat:
        # secondary regime: the reference's own initialiser (xavier gain 0.01) on randn features -> flat heatmaps ->
        # the decode cannot prune and evaluates the whole 384x384 field (SURVEY 7 "hard parts" 1)
        prob_f = make_problem(args.clips, seed=4321 + rank, device=dev, regime="fresh")
        hp_f = HotPath(prob_f, dev, args.fwd_only, two_streams=not args.serial_chains)
        feats_f = prob_f["feats"].to(tdt).to(dev)
        nst = max(2, args.steps // 2)
        flat_fn = GraphedStep(hp_f, feats_f) if graphed else (lambda: hp_f.step(feats_f))
        ms_flat = time_steps(flat_fn, nst, 3)
        flat = {"value": n_frames * nst / (ms_flat / 1e3), "unit": "frames/s", "ms_per_step": ms_flat / nst,
                "regime": "fresh init: reference initialiser (xavier gain 0.01) on randn*0.5 features; flat heatmaps, dense decode",
                "stages": {k: round(v["ms"], 4) for k, v in kernel_breakdown(hp_f, feats_f, reps=5).items()}}
        del flat_fn, hp_f, feats_f, prob_f
    # roofline: the stage with the largest measured share of the step
    dom = max(br, key=lambda k: br[k]["ms"])
    line = {
        "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_total / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": args.dtype, "data": "synthetic",
        "config": {
            "workload": f"BASELINE configs[1] hot path on ResNet-50 features (B,2048,12,12): {args.clips} clips/step/GPU x (16 labeled + 32 unlabeled) frames, "
                        f"K=17, heatmaps 96x96, decode field 384x384; pass = {'forward' if args.fwd_only else 'forward + backward + Adam step on the head (+ gradient all-reduce when N>1)'}",
            "backward": "all native: loss stack, remap, sparse soft-argmax windows, target+mse, fused softmax-backward/G2 front end, tensor-core dgrad+wgrad of both transposed convolutions; Adam step on the head parameters: one native launch (lpb_adam_step)",
            "frames_per_step_per_gpu": n_frames, "regime": ("trained-like synthetic response (unimodal Gaussian-like heatmaps; planted features + bilinear per-keypoint deconvs, see bench.make_problem); fresh_init_regime = reference initialiser"
                                                                                  if args.regime == "trained" else "fresh init (reference initialiser, flat heatmaps)"),
            "launch": ("whole step replayed from one CUDA graph" if graphed else "eager launches")
                      + ("; labeled and unlabeled chains forked onto two streams" if not args.serial_chains else "; one stream"),
            "l2_policy": f"step: inputs larger than L2 ({feats.numel() * esz / 2**20:.0f} MiB of features per step); stages: L2 flushed (256 MiB write) before each of 20 timed repetitions",
            "parallelism": f"dp{world}",
            "ddp": (f"2 NCCL all-reduces per step: a {payload * 4 / 1e6:.1f} MB synthetic backbone-gradient bucket (stands in for ResNet-50's {BACKBONE_PARAMS:,} parameters, which this "
                    "head-only step does not produce) on a side stream overlapped with the head's backward, then the head bucket (80,971 gradients written in place by autograd + 4 logged scalars)"
                    if hp.reducer is not None else "none (N=1)"),
        },
        "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": feats.numel() * esz, "d2h_bytes_per_step": 16},
        "gpu_launches": (HotPath.LAUNCHES_FWD + (0 if args.fwd_only else HotPath.LAUNCHES_BWD)) * args.steps,
        "clocks": clk.summary(),
        "roofline": {"bound": "hbm", "kernel": f"{dom}: {br[dom]['what']}", "achieved": br[dom]["gbs"], "peak": pk["hbm_gbs"], "unit": "GB/s",
                     "frac": br[dom]["gbs"] / pk["hbm_gbs"], "peak_source": pk_src,
                     "algorithmic_bytes_per_launch": br[dom]["algorithmic_bytes"], "launch_ms": br[dom]["ms"],
                     "selection": "arg-max of the per-stage device times below (each stage timed alone, median of 20 repetitions, L2 flushed before each)"},
        "stages": {k: {"ms": round(v["ms"], 4), "ms_mean": round(v["ms_mean"], 4), "GBps": round(v["gbs"], 1), "frac_hbm": round(v["gbs"] / pk["hbm_gbs"], 4)} for k, v in br.items()},
    }
    if fwd_only_value is not None:
        line["forward_only"] = fwd_only_value
    if flat is not None:
        line["fresh_init_regime"] = flat
    if world == 1 and not args.no_cpu_baseline:
        line["cpu_baseline"] = cpu_reference(seed=1234, clips=1, reps=1, train=not args.fwd_only)
    print(json.dumps(line))
    sys.stdout.flush()
    if dist:
        try:
            dist.distributed_c10d._get_default_store().add("lpb_rank0_done", 1)
        except Exception:
            pass
        _teardown(dist, rank, world)


# ------------------------------------------------------------------------------------------------
# reference arm: the reference's own CPU code (oracle/ref_arm.py -> oracle/ref_loader.py) on the host cores.
# Nothing on this path imports lightning_pose_b200.
# ------------------------------------------------------------------------------------------------
def cpu_threads() -> int:
    """torch CPU ops on these small tensors stop scaling (and regress) beyond ~32 threads; override with LPB_CPU_THREADS."""
    return int(os.environ.get("LPB_CPU_THREADS", min(os.cpu_count() or 1, 32)))


def _cpu_model() -> str:
    try:
        return [l.split(":")[1].strip() for l in open("/proc/cpuinfo") if l.startswith("model name")][0]
    except Exception:
        return "?"


def cpu_reference(seed, clips, reps, train=True):
    from oracle.ref_arm import ReferenceStep

    torch.set_num_threads(cpu_threads())
    prob = make_problem(clips, seed=seed, device="cpu", regime="trained")
    step = ReferenceStep(prob, IMG, HM, B_LABELED, T_UNLABELED)
    step(train)  # warm-up
    t0 = time.perf_counter()
    for _ in range(reps):
        step(train)
    dt = (time.perf_counter() - t0) / reps
    frames = clips * (B_LABELED + T_UNLABELED)
    code = "the reference's own files (oracle/_ref via oracle/ref_loader.py; kornia restated)" if step.kind == "reference" else "torch CPU restatement (oracle/lp_oracle.py)"
    return {"value": frames / dt, "unit": "frames/s", "cores": torch.get_num_threads(), "kind": step.kind,
            "sample": f"{clips} clip(s) = {frames} frames of the same workload, {'forward+backward' if train else 'forward'} pass, fp32, {code}, {_cpu_model()}",
            "seconds_per_sample": dt}


def run_reference(args):
    if int(os.environ.get("RANK", 0)) != 0:
        return
    from oracle.ref_arm import ReferenceStep

    torch.set_num_threads(cpu_threads())
    clips = 1
    prob = make_problem(clips, seed=1234, device="cpu", regime=args.regime)
    step = ReferenceStep(prob, IMG, HM, B_LABELED, T_UNLABELED)
    train = not args.fwd_only
    for _ in range(min(args.warmup, 1)):
        step(train)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step(train)
    dt = time.perf_counter() - t0
    frames = clips * (B_LABELED + T_UNLABELED)
    value = frames * args.steps / dt
    code = "the reference's own files executed unmodified (oracle/_ref, oracle/ref_loader.py; kornia restated)" if step.kind == "reference" else "torch CPU restatement of the reference path (oracle/lp_oracle.py)"
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"BASELINE configs[1] hot path, bounded sample: {clips} clip/step x (16 labeled + 32 unlabeled) frames, {'forward+backward' if train else 'forward'} pass, CPU"},
        "cpu_baseline": {"value": value, "unit": "frames/s", "cores": torch.get_num_threads(), "kind": step.kind,
                         "sample": f"{frames} frames/step, {code}, {_cpu_model()}"},
        "e2e": {"value": value, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one returned (loss scalars, updated head parameters and "
                         "their gradients) as DIR/<name>.npy (float32); the seeded inputs make runs with the same arguments comparable")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--clips", type=int, default=16, help="clips per step per GPU (48 frames each)")
    ap.add_argument("--regime", default="trained", choices=["trained", "fresh"], help="synthetic input regime (see make_problem)")
    ap.add_argument("--dtype", default="bf16", choices=["f32", "bf16"], help="feature dtype (bf16 = tensor-core head)")
    ap.add_argument("--no-flat", action="store_true", help="skip the secondary fresh-init (flat heatmap) regime")
    ap.add_argument("--fwd-only", action="store_true", help="time the forward pass only (default: full training step)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--profile-step", action="store_true", help="profiling aid: run W + K eager steps and exit (use under ncu; prints no bench line)")
    ap.add_argument("--kineto", action="store_true", help="with --profile-step: per-kernel device times of the timed steps from torch.profiler (CUPTI), in situ")
    ap.add_argument("--serial-chains", action="store_true", help="run the labeled and the unlabeled chain on one stream (default: two streams, forked and joined inside the step)")
    ap.add_argument("--no-graph", action="store_true", help="launch the step eagerly instead of replaying a captured CUDA graph")
    ap.add_argument("--ddp-payload-mb", type=float, default=BACKBONE_PARAMS * 4 / 1e6,
                    help="N>1: size of the synthetic backbone-gradient bucket all-reduced every step (0 = head gradients only)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
