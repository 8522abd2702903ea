"""torch-facing wrappers of the lpb200 C-ABI: custom ops (``torch.library``) + autograd.

PyTorch is plumbing here (device memory, the current CUDA stream, autograd bookkeeping); every
numerical operation below runs in ``liblpb200.so``.  All wrappers refuse non-CUDA tensors: there is
no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np
import torch

import torch.utils._pytree

from ._lib import Head3Sizes, MseTargets, PcaDesc, check, lib

__all__ = [
    "decode_softargmax",
    "upsample2x",
    "generate_heatmaps",
    "keypoints_mask_oob",
    "evaluate_heatmaps_at_location",
    "head_forward",
    "head_forward_f32",
    "head_bf16_supported",
    "head3_supported",
    "convt_forward_f32",
    "convt_backward_f32",
    "head_backward_bf16",
    "decode_backward_windows",
    "remap_keypoints",
    "heatmap_loss",
    "heatmap_mse_from_keypoints",
    "heatmap_loss_from_keypoints",
    "temporal_heatmap_loss",
    "unsup_losses",
    "PcaParams",
    "triangulate_pairs",
    "project_points",
    "frame_to_model",
    "pairwise_projections_loss",
    "regression_head",
    "regression_losses",
]

_KIND = {"mse": 0, "kl": 1, "js": 2}


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: torch.Tensor | None) -> C.c_void_p:
    if isinstance(t, MseKeypointGrad):
        t = t.materialize()
    return C.c_void_p(0 if t is None else t.data_ptr())


def _cuda_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"lpb200: `{name}` must be a CUDA tensor (this package has no CPU fallback)")
    if isinstance(t, MseKeypointGrad):
        t = t.materialize()
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# =====================================================================================
# soft-argmax decode
# =====================================================================================
class BandMax(NamedTuple):
    """Per-band maxima of softmax heatmaps, written by the 16-bit head's softmax (``lpb_head_fwd_bf16_band_max``):
    ``bits`` int32 [B, K, nbands, 8], the float bits of the largest value in heatmap rows [2 j rows, 2 (j + 1) rows) of
    band j, one slot per epilogue warp.  ``lpb_decode_fwd_banded`` sweeps only the bands that can matter."""

    bits: torch.Tensor
    rows: int
    nbands: int


def decode_forward(heatmaps: torch.Tensor, ds: int, temperature: float, band_max: BandMax | None = None):
    """soft-argmax decode -> (xy, conf, stats).  No autograd node of its own (``_decode_fwd`` and ``_HeadFunction`` own
    the backward).  ``band_max``: the head's band maxima of exactly these heatmaps (same outputs, fewer bytes read)."""
    b, k, h, w = heatmaps.shape
    xy = torch.empty((b, k, 2), device=heatmaps.device, dtype=torch.float32)
    conf = torch.empty((b, k), device=heatmaps.device, dtype=torch.float32)
    stats = torch.empty((b, k, 8), device=heatmaps.device, dtype=torch.float32)
    nbytes = C.c_size_t(0)
    check(lib.lpb_decode_fwd_workspace_bytes(b * k, C.byref(nbytes)))
    workspace = torch.empty((nbytes.value,), device=heatmaps.device, dtype=torch.uint8)
    with torch.cuda.device(heatmaps.device):
        if band_max is None:
            check(lib.lpb_decode_fwd(_ptr(heatmaps), b * k, h, w, ds, temperature, _ptr(xy), _ptr(conf), _ptr(stats), _ptr(workspace), _stream()))
        else:
            if band_max.bits.shape != (b, k, band_max.nbands, 8) or band_max.bits.dtype != torch.int32 or not band_max.bits.is_contiguous():
                raise ValueError(f"decode_forward: band maxima {tuple(band_max.bits.shape)} {band_max.bits.dtype} do not belong to heatmaps {tuple(heatmaps.shape)}")
            check(lib.lpb_decode_fwd_banded(_ptr(heatmaps), b * k, h, w, ds, temperature, _ptr(band_max.bits), band_max.rows, band_max.nbands,
                                            _ptr(xy), _ptr(conf), _ptr(stats), _ptr(workspace), _stream()))
    return xy, conf, stats


@torch.library.custom_op("lpb200::decode_fwd", mutates_args=())
def _decode_fwd(heatmaps: torch.Tensor, ds: int, temperature: float) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    return decode_forward(heatmaps, ds, temperature)


def decode_forward_hinted(heatmaps: torch.Tensor, ds: int, temperature: float, hints: BandMax | None):
    """``decode_forward`` with the hints ``_head_forward_16(..., want_hints=True)`` returned: the band maxima of a
    softmax head, or None (full sweeps)."""
    return decode_forward(heatmaps, ds, temperature, band_max=hints)


@_decode_fwd.register_fake
def _(heatmaps, ds, temperature):
    b, k, _, _ = heatmaps.shape
    return heatmaps.new_empty((b, k, 2)), heatmaps.new_empty((b, k)), heatmaps.new_empty((b, k, 8))


@torch.library.custom_op("lpb200::decode_bwd", mutates_args=())
def _decode_bwd(heatmaps: torch.Tensor, stats: torch.Tensor, grad_xy: torch.Tensor, ds: int, temperature: float) -> torch.Tensor:
    b, k, h, w = heatmaps.shape
    g = torch.empty_like(heatmaps)
    with torch.cuda.device(heatmaps.device):
        check(lib.lpb_decode_bwd(_ptr(heatmaps), _ptr(stats), _ptr(grad_xy), b * k, h, w, ds, temperature, _ptr(g), _stream()))
    return g


@_decode_bwd.register_fake
def _(heatmaps, stats, grad_xy, ds, temperature):
    return torch.empty_like(heatmaps)


def _decode_setup(ctx, inputs, output):
    heatmaps, ds, temperature = inputs
    ctx.save_for_backward(heatmaps, output[2])
    ctx.ds, ctx.temperature = ds, temperature


def _decode_backward(ctx, g_xy, g_conf, g_stats):
    heatmaps, stats = ctx.saved_tensors
    if g_xy is None:
        return None, None, None
    return _decode_bwd(heatmaps, stats, g_xy.contiguous().float(), ctx.ds, ctx.temperature), None, None


_decode_fwd.register_autograd(_decode_backward, setup_context=_decode_setup)


def decode_softargmax(heatmaps: torch.Tensor, downsample_factor: int, temperature: float = 1000.0):
    """(B,K,h,w) heatmaps -> (preds (B,2K), confidences (B,K)); differentiable wrt heatmaps (via preds)."""
    hm = _cuda_f32(heatmaps, "heatmaps")
    if hm.dim() != 4:
        raise ValueError(f"heatmaps must be (batch, keypoints, h, w); got {tuple(hm.shape)}")
    if downsample_factor not in (1, 2, 3):
        raise ValueError(f"downsample_factor must be 1, 2 or 3; got {downsample_factor}")
    xy, conf, _ = _decode_fwd(hm, int(downsample_factor), float(temperature))
    return xy.reshape(-1, hm.shape[1] * 2), conf


def upsample2x(inputs: torch.Tensor) -> torch.Tensor:
    x = _cuda_f32(inputs, "inputs")
    b, k, h, w = x.shape
    out = torch.empty((b, k, 2 * h, 2 * w), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        check(lib.lpb_upsample2x(_ptr(x), b * k, h, w, _ptr(out), _stream()))
    return out


# =====================================================================================
# Gaussian targets / windowed evaluation
# =====================================================================================
class _GenerateHeatmaps(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, visibility, height, width, oh, ow, sigma):
        kp = keypoints.contiguous().float()
        b, k, _ = kp.shape
        out = torch.empty((b, k, oh, ow), device=kp.device, dtype=torch.float32)
        with torch.cuda.device(kp.device):
            check(lib.lpb_generate_heatmaps(_ptr(kp), _ptr(visibility), b * k, float(height), float(width), oh, ow, float(sigma), _ptr(out), _stream()))
        ctx.save_for_backward(kp, visibility)
        ctx.meta = (float(height), float(width), oh, ow, float(sigma))
        return out

    @staticmethod
    def backward(ctx, g):
        kp, vis = ctx.saved_tensors
        height, width, oh, ow, sigma = ctx.meta
        gk = torch.empty_like(kp)
        with torch.cuda.device(kp.device):
            check(lib.lpb_generate_heatmaps_bwd(_ptr(kp), _ptr(vis), _ptr(g.contiguous().float()), kp.shape[0] * kp.shape[1], height, width, oh, ow, sigma, _ptr(gk), _stream()))
        return gk, None, None, None, None, None, None


def generate_heatmaps(keypoints, height, width, output_shape, sigma=1.25, keep_gradients=False, visibility=None):
    kp = _cuda_f32(keypoints, "keypoints")
    if kp.dim() != 3 or kp.shape[-1] != 2:
        raise ValueError(f"keypoints must be (batch, num_keypoints, 2); got {tuple(kp.shape)}")
    vis = None
    if visibility is not None:
        if not visibility.is_cuda:
            raise RuntimeError("lpb200: `visibility` must be a CUDA tensor")
        vis = visibility.to(torch.int32).contiguous()
    if not keep_gradients:
        kp = kp.detach()
    return _GenerateHeatmaps.apply(kp, vis, height, width, int(output_shape[0]), int(output_shape[1]), sigma)


def keypoints_mask_oob(keypoints, height, width):
    """Keypoints outside [0, width) x [0, height) -> NaN in both coordinates (labeled-data rule, datasets.py:496-508)."""
    kp = _cuda_f32(keypoints, "keypoints")
    out = torch.empty_like(kp)
    with torch.cuda.device(kp.device):
        check(lib.lpb_keypoints_mask_oob(_ptr(kp), kp.numel() // 2, float(height), float(width), _ptr(out), _stream()))
    return out


def evaluate_heatmaps_at_location(heatmaps, locs, radius: int = 2):
    hm = _cuda_f32(heatmaps, "heatmaps")
    lc = _cuda_f32(locs, "locs")
    b, k, h, w = hm.shape
    out = torch.empty((b, k), device=hm.device, dtype=torch.float32)
    with torch.cuda.device(hm.device):
        check(lib.lpb_evaluate_heatmaps_at_location(_ptr(hm), _ptr(lc), b * k, h, w, int(radius), _ptr(out), _stream()))
    return out


# =====================================================================================
# heatmap head
# =====================================================================================
FEATURES_NCHW, FEATURES_NHWC = 0, 1  # LPB_FEATURES_* (lpb200.h)
_SHUFFLE_NHWC = 2                    # LPB_SHUFFLE_NHWC


def feature_layout(features: torch.Tensor) -> int:
    """The memory format the head's kernels can read ``features`` (B, C, H, W) in without a copy: ``FEATURES_NHWC`` for
    a dense channels-last tensor (``torch.channels_last``, or a token tensor seen through
    ``models.backbones.tokens_to_feature_map``), ``FEATURES_NCHW`` otherwise.  A tensor that is both (C = 1, or
    H = W = 1) counts as NCHW, and so does one with any other strides: its caller makes it contiguous."""
    if features.dim() == 4 and not features.is_contiguous() and features.is_contiguous(memory_format=torch.channels_last):
        return FEATURES_NHWC
    return FEATURES_NCHW


def head_bf16_supported(shape, channels, train: bool, layout: int = FEATURES_NCHW) -> bool:
    """Whether the tensor-core kernels cover this head: feature shape (B, C, H, W), deconv output channels (c1[, c2]),
    memory format of the features (``feature_layout``).

    The library owns the shape rules: the forward's in ``lpb_head_bf16_plan_layout``, the backward's (``train``) in
    ``lpb_head_bwd_bf16_workspace_bytes_layout``.  Neither needs a GPU."""
    b, c, h, w = shape
    if len(channels) not in (1, 2):
        return False
    c1, c2 = channels[0], (channels[1] if len(channels) == 2 else 0)
    plan = C.c_int(0)
    if lib.lpb_head_bf16_plan_layout(c, h, w, c1, c2, layout, C.byref(plan)) != 0:
        return False
    nbytes = C.c_size_t(0)
    return not train or lib.lpb_head_bwd_bf16_workspace_bytes_layout(b, c, h, w, c1, c2, layout, C.byref(nbytes)) == 0


def _head3_sizes(shape, channels, train: bool, layout: int) -> tuple[int, Head3Sizes]:
    """``lpb_head3_query``'s return code and sizes for a three-deconv head (c1, c2, c3) on features of ``shape``."""
    b, c, h, w = shape
    sizes = Head3Sizes()
    return lib.lpb_head3_query(b, c, h, w, *channels, layout, int(train), C.byref(sizes)), sizes


def head3_supported(shape, channels, train: bool, layout: int = FEATURES_NCHW) -> bool:
    """``head_bf16_supported`` for three-deconv heads (``downsample_factor=1`` on a stride-32 backbone): whether the
    tensor-core kernels cover feature shape (B, C, H, W) with deconv output channels (c1, c2, c3) in memory format
    ``layout``, to train (``train``) or to predict.  The library owns the rule (``lpb_head3_query``, no GPU needed)."""
    if len(channels) != 3:
        return False
    return _head3_sizes(tuple(shape), [int(x) for x in channels], train, layout)[0] == 0


def head_16_operand(features, channels, train: bool):
    """``(features as the 16-bit head reads them, layout)`` or None when the tensor-core kernels do not cover the head.

    Channels-last features are read in place where the kernels take them.  Where only the NCHW kernels cover the shape
    (training at W = 32), and for every tensor that is neither format, this is the NCHW copy.  Three-deconv heads are
    asked of ``head3_supported``, every other head of ``head_bf16_supported``."""
    supported = head3_supported if len(channels) == 3 else head_bf16_supported
    layout = feature_layout(features)
    if layout == FEATURES_NHWC and supported(tuple(features.shape), channels, train, FEATURES_NHWC):
        return features, FEATURES_NHWC
    if supported(tuple(features.shape), channels, train):
        return features.contiguous(), FEATURES_NCHW
    return None


def _head_forward_16(f, weights, biases, final_softmax, train=False, want_hints=False, layout=FEATURES_NCHW):
    """tensor-core path (one-, two- or three-deconv heads) on 16-bit features: bf16 (``lpb_head_fwd_bf16``) or fp16
    (``lpb_head_fwd_f16``), and ``lpb_head3_fwd`` for three deconvs, the weights rounded to the features' dtype on the
    device; the caller checks ``head_16_operand`` first.  Both dtypes share the plan and the buffer sizes.  ``layout``: the memory format ``f`` is
    dense in (``FEATURES_NCHW``: contiguous; ``FEATURES_NHWC``: channels-last, read in place).

    ``train=True`` (bf16 only: there is no fp16 backward) returns ``(out, saved)`` where ``saved`` carries what
    ``head_backward_bf16`` needs (the row-layout copy of the shuffled features and the forward workspace with the
    inter-layer activations).

    ``want_hints=True`` appends the decode hints: with ``final_softmax`` the heatmaps' band maxima (``BandMax``, written
    by the softmax pass for ``decode_forward``), otherwise None.
    """
    entry = _HEAD_FWD_16.get(f.dtype)
    if entry is None or (train and f.dtype != torch.bfloat16):
        raise ValueError(f"the 16-bit head takes bf16 or (forward only) fp16 features; got {f.dtype}{' for training' if train else ''}")
    b, c, h, w = f.shape
    n = len(weights)
    w1 = _cuda_f32(weights[0], "weight")
    b1 = _cuda_f32(biases[0], "bias")
    w2 = _cuda_f32(weights[1], "weight") if n >= 2 else None
    b2 = _cuda_f32(biases[1], "bias") if n >= 2 else None
    w3 = _cuda_f32(weights[2], "weight") if n == 3 else None
    b3 = _cuda_f32(biases[2], "bias") if n == 3 else None
    c1, c2, c3 = w1.shape[1], (w2.shape[1] if n >= 2 else 0), (w3.shape[1] if n == 3 else 0)
    nbytes = C.c_size_t(0)
    if n == 3:
        rc, sizes = _head3_sizes((b, c, h, w), (c1, c2, c3), train, layout)
        check(rc)
        plan, ws_bytes, xs_bytes = sizes.plan, sizes.fwd_workspace, sizes.saved
    else:
        plan_c = C.c_int(0)
        check(lib.lpb_head_bf16_plan_layout(c, h, w, c1, c2, layout, C.byref(plan_c)))
        check(lib.lpb_head_bf16_workspace_bytes(b, c, h, w, c1, c2, C.byref(nbytes)))
        plan, ws_bytes = plan_c.value, nbytes.value
    ws = torch.empty((ws_bytes,), device=f.device, dtype=torch.uint8)
    up = {1: 4, 2: 8, 3: 16}[n]
    out = torch.empty((b, (c1, c2, c3)[n - 1], up * h, up * w), device=f.device, dtype=torch.float32)
    xs = None
    if train or plan == 0:  # row-layout copy of the shuffled features: the banded path's operand / the wgrad's input
        if n != 3:
            check(lib.lpb_head_bf16_saved_bytes(b, c, h, w, C.byref(nbytes)))
            xs_bytes = nbytes.value
        xs = torch.empty((xs_bytes,), device=f.device, dtype=torch.uint8)
    hints = None
    with torch.cuda.device(f.device):
        if want_hints and final_softmax:
            rows, nbands = C.c_int(0), C.c_int(0)
            check(lib.lpb_head_band_max_dims(out.shape[2], out.shape[3], C.byref(rows), C.byref(nbands)))
            hints = BandMax(torch.empty((b, out.shape[1], nbands.value, 8), device=f.device, dtype=torch.int32), rows.value, nbands.value)
        if n == 3:
            check(lib.lpb_head3_fwd(_ptr(f), _OPERAND_16[f.dtype], layout, b, c, h, w, _ptr(w1), _ptr(b1), c1, _ptr(w2), _ptr(b2), c2, _ptr(w3),
                                    _ptr(b3), c3, int(bool(final_softmax)), _ptr(out), _ptr(hints.bits if hints is not None else None), _ptr(xs),
                                    _ptr(ws), _stream()))
        elif want_hints and final_softmax:
            check(_HEAD_FWD_16_BAND_MAX[f.dtype](_ptr(f), b, c, h, w, _ptr(w1), _ptr(b1), c1, _ptr(w2), _ptr(b2), c2, layout, _ptr(out),
                                                 _ptr(hints.bits), _ptr(xs), _ptr(ws), _stream()))
        else:
            check(entry(_ptr(f), b, c, h, w, _ptr(w1), _ptr(b1), c1, _ptr(w2), _ptr(b2), c2, int(bool(final_softmax)), layout, _ptr(out), _ptr(xs), _ptr(ws), _stream()))
    if want_hints:
        return (out, (xs, ws), hints) if train else (out, hints)
    if train:
        return out, (xs, ws)
    return out


_HEAD_FWD_16 = {torch.bfloat16: lib.lpb_head_fwd_bf16_layout, torch.float16: lib.lpb_head_fwd_f16_layout}
_HEAD_FWD_16_BAND_MAX = {torch.bfloat16: lib.lpb_head_fwd_bf16_band_max, torch.float16: lib.lpb_head_fwd_f16_band_max}
_OPERAND_16 = {torch.bfloat16: 1, torch.float16: 2}  # LPB_OUT_BF16, LPB_OUT_F16 (lpb200.h)
_head_forward_bf16 = _head_forward_16  # the name bench.py and the bf16 tests call


def decode_backward_windows(heatmaps, stats, grad_xy, ds, temperature):
    """Sparse soft-argmax gradient for the fused head backward: (win, meta, overflow) of ``lpb_decode_bwd_windows``."""
    b, k, h, w = heatmaps.shape
    win = torch.empty((b * k, 32, 32), device=heatmaps.device, dtype=torch.float32)
    meta = torch.empty((b * k, 4), device=heatmaps.device, dtype=torch.int32)
    # only planes whose support overflows a window are ever written/read here (none for peaked heatmaps);
    # the caching allocator hands the block back without touching it
    overflow = torch.empty_like(heatmaps)
    queue = torch.empty((b * k + 1,), device=heatmaps.device, dtype=torch.int32)
    with torch.cuda.device(heatmaps.device):
        check(lib.lpb_decode_bwd_windows(_ptr(heatmaps), _ptr(stats), _ptr(grad_xy), b * k, h, w, ds, temperature, _ptr(win), _ptr(meta), _ptr(overflow), _ptr(queue), _stream()))
    return win, meta, overflow


def head_backward_bf16(g_out, saved, feat_shape, w1, w2, need_dfeat=True, probs=None, windows=None, layout=FEATURES_NCHW, mse=None, w3=None):
    """Gradients of the bf16 head: returns (dfeat bf16 | None, dw1, db1, dw2 | None, db2 | None), and for a three-deconv
    head (``w3`` given, ``lpb_head3_bwd``) also dw3, db3.  ``dfeat`` is dense in ``layout``, the memory format the
    forward read the features in.

    ``g_out``: dense gradient w.r.t. the head output or None; ``probs``: the head output when it ends in the
    spatial softmax (its backward is fused in), None for a logits head; ``windows``: result of
    ``decode_backward_windows`` or None; ``w2`` None for a one-deconv head.  ``mse``: instead of ``g_out``, a
    ``MseKeypointGrad`` of the loss on ``probs``, rebuilt inside the kernels (``lpb_head_bwd_bf16_targets``).
    """
    xs, fws = saved
    b, c, h, w = feat_shape
    g = _cuda_f32(g_out, "g_out") if g_out is not None else None
    if g is None and windows is None and mse is None:
        raise ValueError("head_backward_bf16 needs a dense gradient and/or decode windows")
    if mse is not None and (g is not None or probs is None or not mse.implicit_for(probs)):
        raise ValueError("head_backward_bf16: `mse` stands for the dense gradient of a loss on `probs`")
    w1 = _cuda_f32(w1, "w1")
    w2 = _cuda_f32(w2, "w2") if w2 is not None else None
    w3 = _cuda_f32(w3, "w3") if w3 is not None else None
    c1, c2 = w1.shape[1], (w2.shape[1] if w2 is not None else 0)
    dev = w1.device
    nbytes = C.c_size_t(0)
    if w3 is not None:
        rc, sizes = _head3_sizes((b, c, h, w), (c1, c2, w3.shape[1]), True, layout)
        check(rc)
        nbytes.value = sizes.bwd_workspace_targets if mse is not None else sizes.bwd_workspace
    else:
        check(lib.lpb_head_bwd_bf16_workspace_bytes_targets(b, c, h, w, c1, c2, layout, int(mse is not None), C.byref(nbytes)))
    ws = torch.empty((nbytes.value,), device=dev, dtype=torch.uint8)
    fmt = torch.channels_last if layout == FEATURES_NHWC else torch.contiguous_format
    dfeat = torch.empty((b, c, h, w), device=dev, dtype=torch.bfloat16, memory_format=fmt) if need_dfeat else None
    dw1 = torch.empty_like(w1)
    db1 = torch.empty((c1,), device=dev, dtype=torch.float32)
    dw2 = torch.empty_like(w2) if w2 is not None else None
    db2 = torch.empty((c2,), device=dev, dtype=torch.float32) if w2 is not None else None
    win, meta, ov = windows if windows is not None else (None, None, None)
    targets = C.byref(mse.targets()) if mse is not None else None
    if w3 is not None:
        c3 = w3.shape[1]
        dw3 = torch.empty_like(w3)
        db3 = torch.empty((c3,), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib.lpb_head3_bwd(_ptr(g), targets, _ptr(probs), _ptr(win), _ptr(meta), _ptr(ov), _ptr(xs), _ptr(fws), layout, b, c, h, w, _ptr(w1),
                                    c1, _ptr(w2), c2, _ptr(w3), c3, _ptr(dfeat), _ptr(dw1), _ptr(db1), _ptr(dw2), _ptr(db2), _ptr(dw3), _ptr(db3),
                                    _ptr(ws), _stream()))
        return dfeat, dw1, db1, dw2, db2, dw3, db3
    with torch.cuda.device(dev):
        check(lib.lpb_head_bwd_bf16_targets(_ptr(g), targets, _ptr(probs), _ptr(win), _ptr(meta), _ptr(ov), _ptr(xs), _ptr(fws), b, c, h, w, _ptr(w1), c1,
                                            _ptr(w2), c2, layout, _ptr(dfeat), _ptr(dw1), _ptr(db1), _ptr(dw2), _ptr(db2), _ptr(ws), _stream()))
    return dfeat, dw1, db1, dw2, db2


# ---- fp32 precision path: one transposed convolution at a time (any number of layers), native backward ----------
def _f32_conv_input(x, shuffle: bool):
    """``(x as fp32 the kernels can read, the entries' shuffle argument)``: the PixelShuffle-folding layer reads
    channels-last features in place, everything else is made contiguous."""
    if shuffle and isinstance(x, torch.Tensor) and x.is_cuda and feature_layout(x) == FEATURES_NHWC:
        return x.float(), _SHUFFLE_NHWC  # (.float() keeps the strides)
    return _cuda_f32(x, "input"), int(shuffle)


def convt_forward_f32(x, weight, bias, shuffle: bool):
    """[PixelShuffle(2) +] ConvTranspose2d(k3, s2, p1, op1) in fp32 (3xTF32 on the tensor cores); any Cin, Cout, size.
    With ``shuffle``, channels-last ``x`` is read in place (same result bits as from its NCHW copy)."""
    x, mode = _f32_conv_input(x, shuffle)
    wt = _cuda_f32(weight, "weight")
    bs = _cuda_f32(bias, "bias") if bias is not None else None
    b, c, h, w = x.shape
    cin, hi, wi = (c // 4, 2 * h, 2 * w) if shuffle else (c, h, w)
    if wt.shape[0] != cin:
        raise ValueError(f"weight expects {wt.shape[0]} input channels, got {cin}")
    out = torch.empty((b, wt.shape[1], 2 * hi, 2 * wi), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        check(lib.lpb_convt_fwd_f32(_ptr(x), b, cin, hi, wi, mode, _ptr(wt), _ptr(bs), wt.shape[1], _ptr(out), _stream()))
    return out


def convt_backward_f32(x, grad_out, weight, shuffle: bool, need_dx: bool = True, need_db: bool = True):
    """Autograd of ``convt_forward_f32``: (dx | None, dw, db | None); ``dx`` has the memory format of ``x``.  ``dw`` and
    ``db`` are fixed-order sums (the same bits from run to run on one device model)."""
    x, mode = _f32_conv_input(x, shuffle)
    g = _cuda_f32(grad_out, "grad_out")
    wt = _cuda_f32(weight, "weight")
    b, c, h, w = x.shape
    cin, hi, wi = (c // 4, 2 * h, 2 * w) if shuffle else (c, h, w)
    dx = torch.empty_like(x) if need_dx else None
    dw = torch.empty_like(wt)
    db = torch.empty((wt.shape[1],), device=x.device, dtype=torch.float32) if need_db else None
    nbytes = C.c_size_t(0)
    check(lib.lpb_convt_bwd_f32_workspace_bytes(b, cin, hi, wi, wt.shape[1], C.byref(nbytes)))
    ws = torch.empty((nbytes.value,), device=x.device, dtype=torch.uint8)
    with torch.cuda.device(x.device):
        check(lib.lpb_convt_bwd_f32_ws(_ptr(x), _ptr(g), b, cin, hi, wi, mode, _ptr(wt), wt.shape[1], _ptr(dx), _ptr(dw), _ptr(db), _ptr(ws),
                                       nbytes.value, _stream()))
    return dx, dw, db


def plane_softmax_(x: torch.Tensor) -> torch.Tensor:
    """In-place spatial softmax (T = 1) over each (b, k) plane of a contiguous fp32 tensor."""
    b, k, h, w = x.shape
    with torch.cuda.device(x.device):
        check(lib.lpb_plane_softmax_f32(_ptr(x), b * k, h * w, _stream()))
    return x


def head_forward_f32(features, weights, biases, final_softmax=True, keep_activations=False):
    """fp32 head: PixelShuffle(2) + any number of deconvs + spatial softmax.  Returns ``out`` or, with
    ``keep_activations``, ``(out, inputs_of_each_layer)`` for ``convt_backward_f32``."""
    x, _ = _f32_conv_input(features, True)
    acts = []
    for i, (wt, bs) in enumerate(zip(weights, biases)):
        acts.append(x)
        x = convt_forward_f32(x, wt, bs, shuffle=(i == 0))
    if final_softmax:
        plane_softmax_(x)
    return (x, acts) if keep_activations else x


def head_forward(features, weights, biases, final_softmax=True):
    """PixelShuffle(2) + ConvTranspose2d stack + spatial softmax; forward only.

    bf16 and fp16 features take the 16-bit tensor-core kernels (operands in the features' dtype, fp32 accumulate, fp32
    heatmaps) when the head is a one-, two- or three-deconv head the tiling covers; everything else takes the full-precision
    kernels (3xTF32 on the tensor cores, any depth and keypoint count).  Training uses
    ``HeatmapHead`` which adds the backward.
    """
    if not isinstance(features, torch.Tensor) or not features.is_cuda:
        raise RuntimeError("lpb200: `features` must be a CUDA tensor (this package has no CPU fallback)")
    if len(weights) < 1:
        raise ValueError("head needs at least one deconv layer")
    operand = None
    if features.dtype in _HEAD_FWD_16 and all(b is not None for b in biases):
        operand = head_16_operand(features, [w.shape[1] for w in weights], train=False)
    if operand is not None:
        return _head_forward_16(operand[0], weights, biases, final_softmax, layout=operand[1])
    return head_forward_f32(features, weights, biases, final_softmax)


# =====================================================================================
# coordinate remap
# =====================================================================================
class _Remap(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kp, tf, per_frame, num_views, bb, model_height, model_width, out):
        n, k2 = kp.shape
        res = out if out is not None else torch.empty_like(kp)
        with torch.cuda.device(kp.device):
            check(lib.lpb_remap_keypoints(_ptr(kp), n, k2 // 2, _ptr(tf), per_frame, num_views, _ptr(bb), bb.shape[0], model_height, model_width, _ptr(res), _stream()))
        ctx.save_for_backward(tf, bb)
        ctx.meta = (per_frame, num_views, model_height, model_width)
        if out is not None:
            ctx.mark_dirty(out)
        return res

    @staticmethod
    def backward(ctx, g):
        tf, bb = ctx.saved_tensors
        per_frame, num_views, mh, mw = ctx.meta
        g = g.contiguous().float()
        n, k2 = g.shape
        gi = torch.empty_like(g)
        with torch.cuda.device(g.device):
            check(lib.lpb_remap_keypoints_bwd(_ptr(g), n, k2 // 2, _ptr(tf), per_frame, num_views, _ptr(bb), bb.shape[0], mh, mw, _ptr(gi), _stream()))
        return gi, None, None, None, None, None, None, None


def remap_keypoints(keypoints, transforms, bbox, model_height, model_width, is_multiview=False, num_views=1, out=None):
    """undo_affine_transform_batch + model_to_frame_batch in one launch; differentiable in ``keypoints``."""
    kp = _cuda_f32(keypoints, "keypoints")
    n, k2 = kp.shape
    tf = None
    per_frame = 0
    if transforms is not None and transforms.shape[-1] == 3:
        tf = _cuda_f32(transforms, "transforms")
        if not is_multiview and tf.dim() == 3:
            if tf.shape[0] == 1:  # a lone (1, 2, 3) transform is tiled over the frames (data/utils.py:193-200)
                tf = tf[0].contiguous()
            elif tf.shape[0] == n:
                per_frame = 1
            else:
                raise ValueError(f"per-frame transforms {tuple(tf.shape)} vs {n} frames")
    bb = _cuda_f32(bbox, "bbox")
    if out is not None and kp.requires_grad:
        out = None  # writing through a tensor that autograd tracks is not allowed; return a fresh one
    return _Remap.apply(kp, tf, per_frame, int(num_views), bb, float(model_height), float(model_width), out)


# =====================================================================================
# MHCRNN context branch
# =====================================================================================
class _CrnnCombine(torch.autograd.Function):
    """(x_f + x_b) / 2 of the bidirectional conv-RNN, from per-frame deconv maps and a window index table."""

    @staticmethod
    def forward(ctx, wf, wb, idx, cwf, cbf, twf, tbf, cwb, cbb, twb, tbb):
        n, k, h, w = wf.shape
        m = idx.shape[0]
        f = cwf.shape[0] // k
        dev = wf.device
        Lf, hf = torch.empty((k, 16), device=dev), torch.empty((k, 4), device=dev)
        Lb, hb = torch.empty((k, 16), device=dev), torch.empty((k, 4), device=dev)
        out = torch.empty((m, k, h, w), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib.lpb_crnn_prepare(_ptr(cwf), _ptr(cbf), _ptr(twf), _ptr(tbf), k, f, _ptr(Lf), _ptr(hf), _stream()))
            check(lib.lpb_crnn_prepare(_ptr(cwb), _ptr(cbb), _ptr(twb), _ptr(tbb), k, f, _ptr(Lb), _ptr(hb), _stream()))
            check(lib.lpb_crnn_combine_fwd(_ptr(wf), _ptr(wb), _ptr(idx), m, n, k, h, w, _ptr(Lf), _ptr(hf), _ptr(Lb), _ptr(hb), _ptr(out), _stream()))
        ctx.save_for_backward(wf, wb, idx, cwf, cbf, twf, cwb, cbb, twb, Lf, hf, Lb, hb)
        return out

    @staticmethod
    def backward(ctx, g):
        wf, wb, idx, cwf, cbf, twf, cwb, cbb, twb, Lf, hf, Lb, hb = ctx.saved_tensors
        n, k, h, w = wf.shape
        m = idx.shape[0]
        f = cwf.shape[0] // k
        dev = wf.device
        g = g.contiguous().float()
        dwf, dwb = torch.empty_like(wf), torch.empty_like(wb)
        dLf, dhf, dLb, dhb = torch.empty_like(Lf), torch.empty_like(hf), torch.empty_like(Lb), torch.empty_like(hb)
        outs = [torch.empty_like(t) for t in (cwf, cbf, twf)] + [torch.empty((k,), device=dev)] + [torch.empty_like(t) for t in (cwb, cbb, twb)] + [torch.empty((k,), device=dev)]
        nbytes = C.c_size_t(0)
        check(lib.lpb_crnn_combine_bwd_workspace_bytes(m, n, k, h, w, C.byref(nbytes)))
        ws = torch.empty((nbytes.value,), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            check(lib.lpb_crnn_combine_bwd_ws(_ptr(wf), _ptr(wb), _ptr(idx), _ptr(g), m, n, k, h, w, _ptr(Lf), _ptr(hf), _ptr(Lb), _ptr(hb),
                                              _ptr(dwf), _ptr(dwb), _ptr(dLf), _ptr(dhf), _ptr(dLb), _ptr(dhb), _ptr(ws), nbytes.value, _stream()))
            check(lib.lpb_crnn_prepare_bwd(_ptr(cwf), _ptr(cbf), _ptr(twf), _ptr(dLf), _ptr(dhf), k, f, _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]), _ptr(outs[3]), _stream()))
            check(lib.lpb_crnn_prepare_bwd(_ptr(cwb), _ptr(cbb), _ptr(twb), _ptr(dLb), _ptr(dhb), k, f, _ptr(outs[4]), _ptr(outs[5]), _ptr(outs[6]), _ptr(outs[7]), _stream()))
        return (dwf, dwb, None, *outs)


def crnn_combine(wf, wb, idx, h_f_params, h_b_params):
    """Pre-softmax MHCRNN logits (M, K, H, W).  ``wf`` / ``wb``: (N, K, H, W) maps W_f(x_t) / W_b(x_t) of N frames;
    ``idx``: (M, 5) int32 frame indices of the context slots; ``h_*_params`` = (conv.weight, conv.bias, convT.weight,
    convT.bias) of ``H_f`` / ``H_b``.  Differentiable in the maps and in the eight parameter tensors."""
    wf, wb = _cuda_f32(wf, "wf"), _cuda_f32(wb, "wb")
    if wf.shape != wb.shape or wf.dim() != 4 or wf.shape[2] % 2 or wf.shape[3] % 2:
        raise ValueError(f"deconv maps must be (N, K, H, W) with even H, W; got {tuple(wf.shape)} / {tuple(wb.shape)}")
    idx = idx.to(device=wf.device, dtype=torch.int32).contiguous()
    if idx.dim() != 2 or idx.shape[1] != 5:
        raise ValueError(f"idx must be (M, 5); got {tuple(idx.shape)}")
    ps = [_cuda_f32(t, "crnn parameter") for t in (*h_f_params, *h_b_params)]
    k = wf.shape[1]
    if idx.shape[0] * k >= 65536:  # grid.y limit of one launch: split the windows
        parts = [_CrnnCombine.apply(wf, wb, idx[i : i + 65535 // k], *ps) for i in range(0, idx.shape[0], 65535 // k)]
        return torch.cat(parts, dim=0)
    return _CrnnCombine.apply(wf, wb, idx, *ps)


class _PlaneSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits):
        p = logits.contiguous().float().clone()
        plane_softmax_(p)
        ctx.save_for_backward(p)
        return p

    @staticmethod
    def backward(ctx, g):
        (p,) = ctx.saved_tensors
        return plane_softmax_backward(p, g)


def plane_softmax(logits: torch.Tensor) -> torch.Tensor:
    """spatial_softmax2d(x, temperature=1) with its native backward."""
    return _PlaneSoftmax.apply(_cuda_f32(logits, "logits"))


class _ContextGather(torch.autograd.Function):
    """The window tensor and its adjoint: a frame's gradient is the sum of the window slots that read it."""

    @staticmethod
    def forward(ctx, x, context_length):
        n = x.shape[0]
        out = torch.empty((n, context_length, *x.shape[1:]), device=x.device, dtype=x.dtype)
        with torch.cuda.device(x.device):
            check(lib.lpb_context_gather(_ptr(x), n, x[0].numel() * x.element_size(), context_length, _ptr(out), _stream()))
        ctx.shape, ctx.context_length = x.shape, context_length
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        d = torch.empty(ctx.shape, device=g.device, dtype=g.dtype)
        with torch.cuda.device(g.device):
            check(lib.lpb_context_gather_bwd(_ptr(g), ctx.shape[0], d[0].numel(), ctx.context_length, _OUT_FORMATS[g.dtype], _ptr(d), _stream()))
        return d, None


def context_gather(seq: torch.Tensor, context_length: int = 5) -> torch.Tensor:
    """get_context_from_sequence (base.py:159-196): (n, ...) -> (n, ctx, ...) windows with replicated edges;
    differentiable in ``seq`` for fp32, bf16 and fp16 sequences."""
    if not isinstance(seq, torch.Tensor) or not seq.is_cuda:
        raise RuntimeError("lpb200: `img_seq` must be a CUDA tensor (this package has no CPU fallback)")
    x = seq.contiguous()
    item = x[0].numel() * x.element_size()
    if item % 16:
        raise ValueError(f"items of {item} bytes: the gather moves 16-byte vectors")
    if x.requires_grad and torch.is_grad_enabled() and x.dtype not in _OUT_FORMATS:
        raise ValueError(f"the window gradient is summed for float32, bfloat16 and float16 sequences; got {x.dtype}")
    return _ContextGather.apply(x, int(context_length))


IMAGENET_MEAN = (0.485, 0.456, 0.406)  # lightning_pose/data/__init__.py (_IMAGENET_MEAN / _IMAGENET_STD)
IMAGENET_STD = (0.229, 0.224, 0.225)

# output-format codes of the ingest entries (LPB_OUT_F32 / LPB_OUT_BF16 / LPB_OUT_F16, include/lpb200.h)
_OUT_FORMATS = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def _out_format(dtype) -> int:
    if dtype not in _OUT_FORMATS:
        raise ValueError("dtype must be float32, bfloat16 or float16")
    return _OUT_FORMATS[dtype]


def frames_normalize(frames_u8, size=None, mean=IMAGENET_MEAN, std=IMAGENET_STD, channels_last=False, dtype=torch.float32):
    """uint8 (F, H, W, 3) decoded RGB frames -> normalised (F, 3, h, w) [or (F, h, w, 3)] fp32 / bf16 / fp16 in one pass
    (bf16 and fp16 are the fp32 result rounded to nearest even)."""
    if not isinstance(frames_u8, torch.Tensor) or not frames_u8.is_cuda:
        raise RuntimeError("lpb200: `frames` must be a CUDA tensor (this package has no CPU fallback)")
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise ValueError(f"frames must be uint8 (F, H, W, 3); got {tuple(frames_u8.shape)} {frames_u8.dtype}")
    fmt = _out_format(dtype)
    x = frames_u8.contiguous()
    f, h, w, _ = x.shape
    oh, ow = (int(size[0]), int(size[1])) if size is not None else (h, w)
    out = torch.empty((f, oh, ow, 3) if channels_last else (f, 3, oh, ow), device=x.device, dtype=dtype)
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(x.device):
        check(lib.lpb_frames_normalize(_ptr(x), f, h, w, oh, ow, m3, s3, int(bool(channels_last)), fmt, _ptr(out), _stream()))
    return out


def frames_crop_resize_cv2(frames_u8, size, box=None, mean=IMAGENET_MEAN, std=IMAGENET_STD, channels_last=False,
                           dtype=torch.float32, out=None, bbox_out=None):
    """uint8 (F, H, W, 3) frames -> the preprocessing of the reference's ``Model.predict_frame`` in one launch: the
    numpy-slice crop ``frame[y:y+h, x:x+w]``, ``cv2.resize(INTER_LINEAR)`` on uint8 and ``(u8 / 255 - mean) / std`` in
    fp32, bit for bit (``lpb_frames_crop_resize_cv2``).

    ``box``: None (the whole frame) or a 4-element int32 CUDA tensor [x, y, w, h], read by the kernel (the caller has
    refused a negative origin, a non-positive size and an empty crop).  Returns (frames (F, 3, h, w) [or (F, h, w, 3)],
    bbox (1, 4) fp32 [x, y, actual_h, actual_w]), written into ``out`` / ``bbox_out`` when given."""
    if not isinstance(frames_u8, torch.Tensor) or not frames_u8.is_cuda:
        raise RuntimeError("lpb200: `frames` must be a CUDA tensor (this package has no CPU fallback)")
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3 or frames_u8.shape[0] < 1:
        raise ValueError(f"frames must be uint8 (F >= 1, H, W, 3); got {tuple(frames_u8.shape)} {frames_u8.dtype}")
    fmt = _out_format(dtype)
    dev = frames_u8.device
    if box is not None and (not isinstance(box, torch.Tensor) or box.device != dev or box.dtype != torch.int32
                            or box.numel() != 4 or not box.is_contiguous()):
        raise ValueError("box must be a contiguous 4-element int32 tensor [x, y, w, h] on the frames' device")
    x = frames_u8.contiguous()
    f, h, w, _ = x.shape
    oh, ow = int(size[0]), int(size[1])
    shape = (f, oh, ow, 3) if channels_last else (f, 3, oh, ow)
    if out is None:
        out = torch.empty(shape, device=dev, dtype=dtype)
    elif tuple(out.shape) != shape or out.dtype != dtype or out.device != dev or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous {dtype} {shape} tensor on the frames' device")
    if bbox_out is None:
        bbox_out = torch.empty((1, 4), device=dev, dtype=torch.float32)
    elif bbox_out.dtype != torch.float32 or bbox_out.device != dev or bbox_out.numel() != 4 or not bbox_out.is_contiguous():
        raise ValueError("bbox_out must be a contiguous 4-element float32 tensor on the frames' device")
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(dev):
        check(lib.lpb_frames_crop_resize_cv2(_ptr(x), f, h, w, _ptr(box), oh, ow, m3, s3, int(bool(channels_last)), fmt,
                                             _ptr(out), _ptr(bbox_out), _stream()))
    return out, bbox_out.view(1, 4)


INGEST_MAX_VIEWS = 16  # LPB_INGEST_MAX_VIEWS (include/lpb200.h)


def frames_normalize_views(views_u8, size, mean=IMAGENET_MEAN, std=IMAGENET_STD, channels_last=False, dtype=torch.float32):
    """V synchronised views, uint8 (F, H_v, W_v, 3) each (sizes may differ), -> normalised (F, V, 3, h, w) [or
    (F, V, h, w, 3)] fp32 / bf16 / fp16 in one launch; view v of frame f is bit-identical to ``frames_normalize`` of that view.
    ``reshape(F * V, ...)`` is the frame-major, view-minor batch of the multi-view trackers."""
    views = list(views_u8)
    if not 1 <= len(views) <= INGEST_MAX_VIEWS:
        raise ValueError(f"frames_normalize_views takes 1..{INGEST_MAX_VIEWS} views; got {len(views)}")
    for v in views:
        if not isinstance(v, torch.Tensor) or not v.is_cuda:
            raise RuntimeError("lpb200: `views` must be CUDA tensors (this package has no CPU fallback)")
        if v.dtype != torch.uint8 or v.dim() != 4 or v.shape[-1] != 3:
            raise ValueError(f"each view must be uint8 (F, H, W, 3); got {tuple(v.shape)} {v.dtype}")
        if v.device != views[0].device:
            raise ValueError("all views must be on one device")
    f = views[0].shape[0]
    if any(v.shape[0] != f for v in views):
        raise ValueError(f"all views must have the same frame count; got {[v.shape[0] for v in views]}")
    fmt = _out_format(dtype)
    xs = [v.contiguous() for v in views]
    n = len(xs)
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((f, n, oh, ow, 3) if channels_last else (f, n, 3, oh, ow), device=xs[0].device, dtype=dtype)
    ptrs = (C.c_void_p * n)(*[x.data_ptr() for x in xs])
    hs, ws = (C.c_int * n)(*[x.shape[1] for x in xs]), (C.c_int * n)(*[x.shape[2] for x in xs])
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(xs[0].device):
        check(lib.lpb_frames_normalize_views(ptrs, n, f, hs, ws, oh, ow, m3, s3, int(bool(channels_last)), fmt,
                                             _ptr(out), _stream()))
    return out


def ragged_videos(lengths, sizes) -> torch.Tensor:
    """(n, 3) int64 host table (first row, H, W) of videos of ``lengths`` frames and ``sizes`` (H, W), back to back:
    the video table of the ragged ingest entries (copy it to the device for their ``videos``)."""
    lengths, sizes = [int(n) for n in lengths], [(int(h), int(w)) for h, w in sizes]
    if len(lengths) != len(sizes):
        raise ValueError(f"{len(lengths)} videos but {len(sizes)} frame sizes")
    rows, row0 = [], 0
    for n, (h, w) in zip(lengths, sizes):
        rows.append((row0, h, w))
        row0 += n
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 3)


def ragged_slot_bytes(sizes) -> int:
    """Bytes of one arena slot: the largest uint8 (H, W, 3) frame of ``sizes``, rounded up to 16."""
    return -(-max(int(h) * int(w) * 3 for h, w in sizes) // 16) * 16


def _ragged(arena, slot_bytes: int, frames: int, cursor, videos, videos_host) -> torch.Tensor:
    """Checks the arena arguments shared by the ragged ingests; returns the host table, contiguous."""
    if not isinstance(arena, torch.Tensor) or not arena.is_cuda:
        raise RuntimeError("lpb200: `arena` must be a CUDA tensor (this package has no CPU fallback)")
    if arena.dtype != torch.uint8 or not arena.is_contiguous() or arena.numel() < int(frames) * int(slot_bytes):
        raise ValueError(f"arena must be a contiguous uint8 tensor of at least {int(frames)} slots of {int(slot_bytes)} bytes; "
                         f"got {tuple(arena.shape)} {arena.dtype}")
    if not isinstance(cursor, torch.Tensor) or cursor.device != arena.device or cursor.dtype != torch.int64 or cursor.numel() != 1:
        raise ValueError("cursor must be a one-element int64 tensor on the arena's device")
    host = videos_host.contiguous()
    if (not isinstance(videos, torch.Tensor) or videos.device != arena.device or videos.dtype != torch.int64
            or not videos.is_contiguous() or videos.dim() != 2 or videos.shape[1] != 3 or host.is_cuda
            or host.dtype != torch.int64 or host.shape != videos.shape):
        raise ValueError("videos must be an (n, 3) int64 tensor on the arena's device and videos_host its (n, 3) int64 host copy")
    return host


def frames_normalize_ragged(arena, slot_bytes: int, frames: int, cursor, videos, videos_host, size, mean=IMAGENET_MEAN,
                            std=IMAGENET_STD, channels_last=False, dtype=torch.float32):
    """A chunk of ``frames`` uint8 frames from videos of several sizes -> normalised (F, 3, h, w) [or (F, h, w, 3)]
    fp32 / bf16 / fp16 and their (F, 4) boxes [0, 0, H, W], one launch (``lpb_frames_normalize_ragged``).

    Frame f sits at the start of slot f of ``arena`` (uint8, ``slot_bytes`` per slot, ``ragged_slot_bytes``), rows
    packed; its size is that of the video of ``videos`` (the device copy of ``videos_host``, ``ragged_videos``) holding
    global row ``cursor + f``, read on the device, so a captured graph serves every mix of sizes.  Each image is
    bit-identical to ``frames_normalize`` of that frame alone."""
    host = _ragged(arena, slot_bytes, frames, cursor, videos, videos_host)
    fmt, f, dev = _out_format(dtype), int(frames), arena.device
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((f, oh, ow, 3) if channels_last else (f, 3, oh, ow), device=dev, dtype=dtype)
    boxes = torch.empty((f, 4), device=dev, dtype=torch.float32)
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(dev):
        check(lib.lpb_frames_normalize_ragged(_ptr(arena), int(slot_bytes), f, _ptr(cursor), _ptr(videos), _ptr(host),
                                              videos.shape[0], oh, ow, m3, s3, int(bool(channels_last)), fmt, _ptr(out),
                                              _ptr(boxes), _stream()))
    return out, boxes


# training.imgaug "dlc" draw ranges (lightning_pose/data/video/dali.py:160-175) by column of the augment kernel's
# params: angle (degrees), sx and sy, brightness and contrast, shot-noise factor
DLC_PARAM_RANGES = ((slice(0, 1), -10.0, 10.0), (slice(1, 3), 0.8, 1.2), (slice(3, 5), 0.75, 1.25), (slice(5, 6), 0.0, 10.0))


def draw_dlc_params(num_views: int, device, generator: torch.Generator | None = None):
    """One draw of the DALI video augmentation per view, on the device: (params (V, 6) fp32, seeds (V,) int64).

    Uniform in the reference's ranges (``DLC_PARAM_RANGES``); seeds key each view's shot noise.  ``generator`` is a
    torch generator on ``device`` (default: the device's default generator, which a captured CUDA graph replays with
    fresh draws)."""
    params = torch.empty((int(num_views), 6), device=device, dtype=torch.float32)
    for cols, lo, hi in DLC_PARAM_RANGES:
        params[:, cols].uniform_(lo, hi, generator=generator)
    seeds = torch.randint(-(2**63), 2**63 - 1, (int(num_views),), device=device, dtype=torch.int64, generator=generator)
    return params, seeds


def frames_augment_normalize(frames_u8, size, params, seed, mean=IMAGENET_MEAN, std=IMAGENET_STD, channels_last=False,
                             dtype=torch.float32, transform_out=None):
    """uint8 (F, H, W, 3) frames of one view -> resize, rotate-scale warp, brightness/contrast, shot noise and
    normalisation in one pass (the DALI augmentation of training.imgaug "dlc", include/lpb200.h).

    ``params``: (6,) fp32 CUDA tensor [angle (degrees), sx, sy, brightness, contrast, factor]; ``seed``: one-element
    int64 CUDA tensor.  Both are read by the kernel, not the host.  Returns (frames (F, 3, h, w) [or (F, h, w, 3)],
    transform (2, 3) fp32: the source -> destination matrix the warp applied, what ``remap_keypoints`` undoes); the
    transform is written into ``transform_out`` when given (a CUDA fp32 tensor of 6 elements)."""
    if not isinstance(frames_u8, torch.Tensor) or not frames_u8.is_cuda:
        raise RuntimeError("lpb200: `frames` must be a CUDA tensor (this package has no CPU fallback)")
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise ValueError(f"frames must be uint8 (F, H, W, 3); got {tuple(frames_u8.shape)} {frames_u8.dtype}")
    if dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("dtype must be float32 or bfloat16")
    if size is None or len(size) != 2:
        raise ValueError("size (h, w) is required: the augmentation runs on resized frames")
    dev = frames_u8.device
    if not isinstance(params, torch.Tensor) or params.device != dev or params.dtype != torch.float32 or params.numel() != 6:
        raise ValueError("params must be a 6-element float32 tensor on the frames' device")
    if not isinstance(seed, torch.Tensor) or seed.device != dev or seed.dtype != torch.int64 or seed.numel() != 1:
        raise ValueError("seed must be a one-element int64 tensor on the frames' device")
    if transform_out is None:
        transform_out = torch.empty((2, 3), device=dev, dtype=torch.float32)
    elif transform_out.device != dev or transform_out.dtype != torch.float32 or transform_out.numel() != 6 or not transform_out.is_contiguous():
        raise ValueError("transform_out must be a contiguous 6-element float32 tensor on the frames' device")
    x = frames_u8.contiguous()
    p, sd = params.contiguous(), seed.contiguous()
    f, h, w, _ = x.shape
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((f, oh, ow, 3) if channels_last else (f, 3, oh, ow), device=dev, dtype=dtype)
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(dev):
        check(lib.lpb_frames_augment_normalize(_ptr(x), f, h, w, oh, ow, _ptr(p), _ptr(sd), m3, s3, int(bool(channels_last)),
                                               int(dtype == torch.bfloat16), _ptr(out), _ptr(transform_out), _stream()))
    return out, transform_out.view(2, 3)


# curriculum patch masking (lpb_patch_mask_*, include/lpb200.h)
PATCH_SIZE = 16  # LPB_PATCH_SIZE
PATCH_MAX = 4096  # LPB_PATCH_MAX: patches per view


def _patch_images(images) -> tuple[int, int, int, int, int]:
    """Checks the (B, V, C, H, W) batch of the patch-masking entries; returns its shape."""
    if not isinstance(images, torch.Tensor) or not images.is_cuda:
        raise RuntimeError("lpb200: `images` must be a CUDA tensor (this package has no CPU fallback)")
    if images.dim() != 5:
        raise ValueError(f"images must be (batch, views, channels, height, width); got {tuple(images.shape)}")
    if images.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"images must be float32 or bfloat16; got {images.dtype}")
    if not images.is_contiguous():
        raise ValueError("images must be contiguous")
    b, v, c, h, w = images.shape
    if (h // PATCH_SIZE) * (w // PATCH_SIZE) > PATCH_MAX:
        raise ValueError(f"{h} x {w} images have {(h // PATCH_SIZE) * (w // PATCH_SIZE)} patches of {PATCH_SIZE} x {PATCH_SIZE} "
                         f"per view; at most {PATCH_MAX}")
    return b, v, c, h, w


def patch_mask_select(images, step, patch_seed: int, init_step: int, final_step: int, init_ratio: float, final_ratio: float):
    """The patch mask of one training step, drawn on the device: (B, V, P) fp32, 1 = kept, 0 = masked.

    ``images``: (B, V, C, H, W) fp32 / bf16 CUDA batch (only its shape is read); ``step``: one-element int64 tensor on its
    device, read by the kernel (so a captured graph replays with the step it holds).  Each view masks exactly
    int(ratio(step) * P) of its P 16 x 16 patches, a uniformly random subset fixed by (patch_seed, step, example, view)."""
    b, v, _, h, w = _patch_images(images)
    if not isinstance(step, torch.Tensor) or step.device != images.device or step.dtype != torch.int64 or step.numel() != 1:
        raise ValueError("step must be a one-element int64 tensor on the images' device")
    p = (h // PATCH_SIZE) * (w // PATCH_SIZE)
    mask = torch.empty((b, v, p), device=images.device, dtype=torch.float32)
    seed = (int(patch_seed) + 2**63) % 2**64 - 2**63  # any integer, as torch.Generator.manual_seed takes it, to int64
    with torch.cuda.device(images.device):
        check(lib.lpb_patch_mask_select(_ptr(step.contiguous()), b, v, h, w, seed, int(init_step), int(final_step), float(init_ratio),
                                        float(final_ratio), _ptr(mask), _stream()))
    return mask


def patch_mask_apply(images, mask):
    """``images`` with every patch whose ``mask`` entry is 0 set to zero, out of place; the rows and columns past the last
    whole patch are kept.  ``mask``: (B, V, P) fp32 on the images' device."""
    b, v, c, h, w = _patch_images(images)
    p = (h // PATCH_SIZE) * (w // PATCH_SIZE)
    if not isinstance(mask, torch.Tensor) or mask.device != images.device or mask.dtype != torch.float32 or tuple(mask.shape) != (b, v, p):
        raise ValueError(f"mask must be a float32 ({b}, {v}, {p}) tensor on the images' device")
    m = mask.contiguous()
    out = torch.empty_like(images)
    with torch.cuda.device(images.device):
        check(lib.lpb_patch_mask_apply(_ptr(images), b, v, c, h, w, _OUT_FORMATS[images.dtype], _ptr(m), _ptr(out), _stream()))
    return out


def _bbox_table(bboxes, name: str) -> torch.Tensor:
    b = _cuda_f32(bboxes, name)
    if b.dim() != 2 or b.shape[1] != 4 or b.shape[0] < 1:
        raise ValueError(f"`{name}` must be (N >= 1, 4) [x, y, h, w]; got {tuple(b.shape)}")
    return b


def frames_crop_normalize(frames, bboxes, size, cursor=None, row0: int = 0, mean=IMAGENET_MEAN, std=IMAGENET_STD,
                          channels_last=False, dtype=torch.float32):
    """Per-frame crop to a box, bilinear resize to ``size`` and (for uint8 input) ImageNet normalisation, one launch.

    ``frames``: uint8 (F, H, W, 3) decoded RGB, or fp32 (F, 3, H, W) already normalised (crop + resize only).
    ``bboxes``: (N, 4) [x, y, h, w] device table; frame f uses row min(r0 + f, N - 1) with r0 = ``cursor`` (int64 device
    tensor, read only) or ``row0``.  Returns (frames (F, 3, h, w) [or (F, h, w, 3)], clamped boxes (F, 4) fp32)."""
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda:
        raise RuntimeError("lpb200: `frames` must be a CUDA tensor (this package has no CPU fallback)")
    if frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3:
        in_f32 = 0
        f, h, w, _ = frames.shape
    elif frames.dtype == torch.float32 and frames.dim() == 4 and frames.shape[1] == 3:
        in_f32 = 1
        f, _, h, w = frames.shape
    else:
        raise ValueError(f"frames must be uint8 (F, H, W, 3) or float32 (F, 3, H, W); got {tuple(frames.shape)} {frames.dtype}")
    fmt = _out_format(dtype)
    if int(row0) < 0:
        raise ValueError(f"row0 must be >= 0; got {row0}")
    b = _bbox_table(bboxes, "bboxes")
    if cursor is not None and (not cursor.is_cuda or cursor.dtype != torch.int64 or cursor.numel() != 1):
        raise ValueError("cursor must be a one-element int64 CUDA tensor")
    x = frames.contiguous()
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((f, oh, ow, 3) if channels_last else (f, 3, oh, ow), device=x.device, dtype=dtype)
    boxes_out = torch.empty((f, 4), device=x.device, dtype=torch.float32)
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(x.device):
        check(lib.lpb_frames_crop_normalize(_ptr(x), in_f32, f, h, w, _ptr(b), b.shape[0], _ptr(cursor), int(row0), oh, ow, m3, s3,
                                            int(bool(channels_last)), fmt, _ptr(out), _ptr(boxes_out), _stream()))
    return out, boxes_out


def frames_crop_normalize_ragged(arena, slot_bytes: int, frames: int, cursor, videos, videos_host, bboxes, size,
                                 mean=IMAGENET_MEAN, std=IMAGENET_STD, channels_last=False, dtype=torch.float32):
    """``frames_crop_normalize`` of uint8 frames from videos of several sizes, in the arena of
    ``frames_normalize_ragged``: frame f is cropped to box row min(cursor + f, N - 1) of ``bboxes`` and clamped to its
    own video's size.  Each frame's output and clamped box are bit-identical to ``frames_crop_normalize`` on its own
    video alone.  Returns (frames (F, 3, h, w) [or (F, h, w, 3)], clamped boxes (F, 4) fp32)."""
    host = _ragged(arena, slot_bytes, frames, cursor, videos, videos_host)
    fmt, f, dev = _out_format(dtype), int(frames), arena.device
    b = _bbox_table(bboxes, "bboxes")
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((f, oh, ow, 3) if channels_last else (f, 3, oh, ow), device=dev, dtype=dtype)
    boxes_out = torch.empty((f, 4), device=dev, dtype=torch.float32)
    m3, s3 = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(dev):
        check(lib.lpb_frames_crop_normalize_ragged(_ptr(arena), int(slot_bytes), f, _ptr(cursor), _ptr(videos), _ptr(host),
                                                   videos.shape[0], _ptr(b), b.shape[0], oh, ow, m3, s3,
                                                   int(bool(channels_last)), fmt, _ptr(out), _ptr(boxes_out), _stream()))
    return out, boxes_out


def bboxes_from_keypoints(keypoints, anchor_indices=(), crop_ratio=None, crop_height=None, crop_width=None):
    """(N, K, 2) keypoints or an (N, 3K) prediction table (read in place) -> (N, 4) [x, y, h, w] boxes, one launch.
    ``anchor_indices`` are summed in the order given; empty = all keypoints.  Exactly one of ``crop_ratio`` or
    (``crop_height``, ``crop_width``)."""
    kp = _cuda_f32(keypoints, "keypoints")
    if kp.dim() == 3 and kp.shape[2] == 2:
        n, k, point_stride = kp.shape[0], kp.shape[1], 2
    elif kp.dim() == 2 and kp.shape[1] % 3 == 0:
        n, k, point_stride = kp.shape[0], kp.shape[1] // 3, 3
    else:
        raise ValueError(f"keypoints must be (N, K, 2) or an (N, 3K) prediction table; got {tuple(kp.shape)}")
    anchors = [int(i) for i in anchor_indices]
    arr = (C.c_int32 * max(len(anchors), 1))(*anchors)
    out = torch.empty((n, 4), device=kp.device, dtype=torch.float32)
    with torch.cuda.device(kp.device):
        check(lib.lpb_bboxes_from_keypoints(_ptr(kp), n, k, k * point_stride, point_stride, arr, len(anchors),
                                            float(crop_ratio or 0.0), int(crop_height or 0), int(crop_width or 0), _ptr(out), _stream()))
    return out


def bboxes_rolling_median(bboxes, window: int = 5):
    """Centred rolling median of each column of (N, 4) boxes, rounded half to even (pandas' ``rolling(window,
    center=True, min_periods=1).median().round(0)``), one launch."""
    b = _cuda_f32(bboxes, "bboxes")
    if b.dim() != 2 or b.shape[1] != 4:
        raise ValueError(f"bboxes must be (N, 4); got {tuple(b.shape)}")
    out = torch.empty_like(b)
    with torch.cuda.device(b.device):
        check(lib.lpb_bboxes_rolling_median(_ptr(b), b.shape[0], int(window), _ptr(out), _stream()))
    return out


def pack_predictions(keypoints, confidences, table, cursor=None, row0: int = 0):
    """Write one chunk's (keypoints (T, 2K), confidences (T, K)) into rows of ``table`` (N, 3K) at the device cursor
    (int64 tensor, advanced by T) or at ``row0``.  Mutates ``table`` (and ``cursor``)."""
    kp = _cuda_f32(keypoints, "keypoints")
    cf = _cuda_f32(confidences, "confidences")
    t, k = cf.shape
    if table.dtype != torch.float32 or not table.is_contiguous() or table.shape[1] != 3 * k:
        raise ValueError(f"table must be contiguous fp32 (N, {3 * k}); got {tuple(table.shape)} {table.dtype}")
    with torch.cuda.device(kp.device):
        check(lib.lpb_pack_predictions(_ptr(kp), _ptr(cf), t, k, _ptr(table), table.shape[0], _ptr(cursor), int(row0), _stream()))
    return table


def pack_context_predictions(kp_sf, conf_sf, kp_mf, conf_mf, bbox, model_height, model_width, table, step, cursor=None,
                             frame0: int = 0):
    """Context-model rows of one call's output frames (frame ``c - 2 + i`` for i < T, c = ``cursor`` or ``frame0``, the
    frames fed before the call): per keypoint the more confident of the single-frame (``*_sf``) and multi-frame
    (``*_mf``) predictions (a NaN keeps sf), mapped model -> frame with ``bbox`` (T, 4), written to every row of
    ``table`` (N, 3K) the reference's row rule assigns to that frame for ``sequence_length = step + 4`` (see
    ``lpb_pack_context_predictions``).  Mutates ``table`` and advances ``cursor`` by T."""
    kps, cfs = _cuda_f32(kp_sf, "kp_sf"), _cuda_f32(conf_sf, "conf_sf")
    kpm, cfm = _cuda_f32(kp_mf, "kp_mf"), _cuda_f32(conf_mf, "conf_mf")
    bb = _cuda_f32(bbox, "bbox")
    t, k = cfs.shape
    if kps.shape != (t, 2 * k) or kpm.shape != (t, 2 * k) or cfm.shape != (t, k) or bb.shape != (t, 4):
        raise ValueError(f"shapes: kp_sf {tuple(kps.shape)}, kp_mf {tuple(kpm.shape)} (T, 2K); conf_sf {tuple(cfs.shape)}, "
                         f"conf_mf {tuple(cfm.shape)} (T, K); bbox {tuple(bb.shape)} (T, 4)")
    if not isinstance(table, torch.Tensor) or not table.is_cuda:
        raise RuntimeError("lpb200: `table` must be a CUDA tensor (this package has no CPU fallback)")
    if table.dtype != torch.float32 or not table.is_contiguous() or table.dim() != 2 or table.shape[1] != 3 * k:
        raise ValueError(f"table must be contiguous fp32 (N, {3 * k}); got {tuple(table.shape)} {table.dtype}")
    if cursor is not None and (not cursor.is_cuda or cursor.dtype != torch.int64 or cursor.numel() != 1):
        raise ValueError("cursor must be a one-element int64 CUDA tensor")
    with torch.cuda.device(kps.device):
        check(lib.lpb_pack_context_predictions(_ptr(kps), _ptr(cfs), _ptr(kpm), _ptr(cfm), t, k, _ptr(bb), float(model_height),
                                               float(model_width), _ptr(table), table.shape[0], _ptr(cursor), int(frame0),
                                               int(step), _stream()))
    return table


def context_segments(lengths, step: int) -> torch.Tensor:
    """(S, 3) int64 host table (row0, N, R) of videos of ``lengths`` frames back to back, R the rows a context reader of
    step ``step`` produces for each (what ``lpb_pack_context_predictions_segments`` reads)."""
    t, rows, row0 = int(step), [], 0
    for n in (int(v) for v in lengths):
        rows.append((row0, n, n if t == 1 else t * (-(-(n - t - 4) // t) + 1)))
        row0 += n
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 3)


def pack_context_predictions_segments(kp_sf, conf_sf, kp_mf, conf_mf, bbox, model_height, model_width, table, step, cursor,
                                      segments, segments_host, window_index=None):
    """``pack_context_predictions`` for a list of videos back to back in ``table``: ``segments`` is the (S, 3) device
    copy of ``segments_host`` (``context_segments``).  Each output frame goes to the rows of its own video; frames whose
    windows cross a video boundary write nothing.  With ``window_index`` ((step, 5) int32 device tensor) the cursor
    advance also writes the next chunk's window table (see ``lpb_pack_context_predictions_segments``).  Mutates
    ``table``, ``cursor`` (advanced by T) and ``window_index``."""
    kps, cfs = _cuda_f32(kp_sf, "kp_sf"), _cuda_f32(conf_sf, "conf_sf")
    kpm, cfm = _cuda_f32(kp_mf, "kp_mf"), _cuda_f32(conf_mf, "conf_mf")
    bb = _cuda_f32(bbox, "bbox")
    t, k = cfs.shape
    if kps.shape != (t, 2 * k) or kpm.shape != (t, 2 * k) or cfm.shape != (t, k) or bb.shape != (t, 4):
        raise ValueError(f"shapes: kp_sf {tuple(kps.shape)}, kp_mf {tuple(kpm.shape)} (T, 2K); conf_sf {tuple(cfs.shape)}, "
                         f"conf_mf {tuple(cfm.shape)} (T, K); bbox {tuple(bb.shape)} (T, 4)")
    if not isinstance(table, torch.Tensor) or not table.is_cuda:
        raise RuntimeError("lpb200: `table` must be a CUDA tensor (this package has no CPU fallback)")
    if table.dtype != torch.float32 or not table.is_contiguous() or table.dim() != 2 or table.shape[1] != 3 * k:
        raise ValueError(f"table must be contiguous fp32 (N, {3 * k}); got {tuple(table.shape)} {table.dtype}")
    if cursor is None or not cursor.is_cuda or cursor.dtype != torch.int64 or cursor.numel() != 1:
        raise ValueError("cursor must be a one-element int64 CUDA tensor")
    seg_host = segments_host.contiguous()
    if (not segments.is_cuda or segments.dtype != torch.int64 or not segments.is_contiguous() or seg_host.is_cuda
            or seg_host.dtype != torch.int64 or segments.dim() != 2 or segments.shape[1] != 3 or seg_host.shape != segments.shape):
        raise ValueError("segments must be an (S, 3) int64 CUDA tensor and segments_host its (S, 3) int64 host copy")
    if window_index is not None and (not window_index.is_cuda or window_index.dtype != torch.int32
                                     or not window_index.is_contiguous() or tuple(window_index.shape) != (int(step), 5)):
        raise ValueError(f"window_index must be a contiguous ({int(step)}, 5) int32 CUDA tensor")
    with torch.cuda.device(kps.device):
        check(lib.lpb_pack_context_predictions_segments(
            _ptr(kps), _ptr(cfs), _ptr(kpm), _ptr(cfm), t, k, _ptr(bb), float(model_height), float(model_width), _ptr(table),
            table.shape[0], _ptr(cursor), _ptr(segments), _ptr(seg_host), segments.shape[0], int(step), _ptr(window_index),
            _stream()))
    return table


CONTEXT_RING_SLOTS = 5  # LPB_CONTEXT_RING_SLOTS (include/lpb200.h)


def _ring_buffer(t, shape, name: str, dtype=torch.float32) -> None:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"lpb200: `{name}` must be a CUDA tensor (this package has no CPU fallback)")
    if t.dtype != dtype or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must be a contiguous {dtype} {tuple(shape)} tensor; got {tuple(t.shape)} {t.dtype}")


def context_ring_push(wf, wb, kp_sf, conf_sf, bbox, ring_wf, ring_wb, ring_kp, ring_conf, ring_box, count, window_index):
    """One frame's W_f / W_b maps (1, K, H, W), single-frame decode (1, 2K) / (1, K) and box (1, 4) into slot
    ``count mod 5`` of the ring (``ring_wf`` / ``ring_wb`` (5, K, H, W), ``ring_kp`` (5, 2K), ``ring_conf`` (5, K),
    ``ring_box`` (5, 4)), and the (1, 5) int32 ``window_index`` of frames count - 4 .. count for ``crnn_combine`` over the
    ring (``lpb_context_ring_push``).  ``count`` (one-element int64) is read, not advanced.  Mutates the ring and
    ``window_index``."""
    wf, wb, kp_sf, conf_sf, bbox = (_cuda_f32(t, n) for t, n in ((wf, "wf"), (wb, "wb"), (kp_sf, "kp_sf"),
                                                                   (conf_sf, "conf_sf"), (bbox, "bbox")))
    k, h, w = wf.shape[1:] if wf.dim() == 4 else (0, 0, 0)
    r = CONTEXT_RING_SLOTS
    for t, shape, name in ((wf, (1, k, h, w), "wf"), (wb, (1, k, h, w), "wb"), (kp_sf, (1, 2 * k), "kp_sf"),
                           (conf_sf, (1, k), "conf_sf"), (bbox, (1, 4), "bbox"), (ring_wf, (r, k, h, w), "ring_wf"),
                           (ring_wb, (r, k, h, w), "ring_wb"), (ring_kp, (r, 2 * k), "ring_kp"),
                           (ring_conf, (r, k), "ring_conf"), (ring_box, (r, 4), "ring_box")):
        _ring_buffer(t, shape, name)
    _ring_buffer(count, (1,), "count", torch.int64)
    _ring_buffer(window_index, (1, r), "window_index", torch.int32)
    with torch.cuda.device(wf.device):
        check(lib.lpb_context_ring_push(_ptr(wf), _ptr(wb), _ptr(kp_sf), _ptr(conf_sf), _ptr(bbox), k, h, w, _ptr(ring_wf),
                                        _ptr(ring_wb), _ptr(ring_kp), _ptr(ring_conf), _ptr(ring_box), _ptr(count),
                                        _ptr(window_index), _stream()))


def context_ring_select(ring_kp, ring_conf, ring_box, kp_mf, conf_mf, model_height, model_width, out, count):
    """Frame count - 2 of the ring: per keypoint the more confident of its single-frame decode (ring slot
    ``(count - 2) mod 5``) and the multi-frame decode ``kp_mf`` (1, 2K) / ``conf_mf`` (1, K) (a NaN keeps single-frame),
    mapped to the frame with that slot's box, into ``out`` (K, 3); then ``count`` += 1 (``lpb_context_ring_select``)."""
    kp_mf, conf_mf = _cuda_f32(kp_mf, "kp_mf"), _cuda_f32(conf_mf, "conf_mf")
    r, k = CONTEXT_RING_SLOTS, ring_conf.shape[-1]
    for t, shape, name in ((ring_kp, (r, 2 * k), "ring_kp"), (ring_conf, (r, k), "ring_conf"), (ring_box, (r, 4), "ring_box"),
                           (kp_mf, (1, 2 * k), "kp_mf"), (conf_mf, (1, k), "conf_mf"), (out, (k, 3), "out")):
        _ring_buffer(t, shape, name)
    _ring_buffer(count, (1,), "count", torch.int64)
    with torch.cuda.device(out.device):
        check(lib.lpb_context_ring_select(_ptr(ring_kp), _ptr(ring_conf), _ptr(ring_box), _ptr(kp_mf), _ptr(conf_mf), k,
                                          float(model_height), float(model_width), _ptr(out), _ptr(count), _stream()))
    return out


def plane_softmax_backward(probs: torch.Tensor, grad_probs: torch.Tensor) -> torch.Tensor:
    p = _cuda_f32(probs, "probs")
    g = _cuda_f32(grad_probs, "grad_probs")
    b, k, h, w = p.shape
    out = torch.empty_like(p)
    with torch.cuda.device(p.device):
        check(lib.lpb_plane_softmax_bwd(_ptr(p), _ptr(g), b * k, h * w, _ptr(out), _stream()))
    return out


# =====================================================================================
# heatmap losses
# =====================================================================================
class _HeatmapLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, targets, preds, kind):
        b, k, h, w = preds.shape
        out = torch.empty((2,), device=preds.device, dtype=torch.float32)
        ws = torch.empty((b * k * 2,), device=preds.device, dtype=torch.float32)
        with torch.cuda.device(preds.device):
            check(lib.lpb_heatmap_loss_fwd(_ptr(targets), _ptr(preds), b * k, h, w, kind, _ptr(out), _ptr(ws), _stream()))
        ctx.save_for_backward(targets, preds, ws, out)
        ctx.kind = kind
        loss, count = out[0].clone(), out[1].clone()
        ctx.mark_non_differentiable(count)
        return loss, count

    @staticmethod
    def backward(ctx, g, _g_count):
        targets, preds, ws, out = ctx.saved_tensors
        b, k, h, w = preds.shape
        gp = torch.empty_like(preds)
        gg = g.reshape(1).contiguous().float()
        with torch.cuda.device(preds.device):
            check(lib.lpb_heatmap_loss_bwd(_ptr(targets), _ptr(preds), b * k, h, w, ctx.kind, _ptr(ws), _ptr(out), _ptr(gg), _ptr(gp), _stream()))
        return None, gp, None


def heatmap_loss(targets, preds, kind: str = "mse", return_count: bool = False):
    """mean heatmap loss over planes whose target is not all-zero; optionally also that plane count."""
    t = _cuda_f32(targets, "heatmaps_targ")
    p = _cuda_f32(preds, "heatmaps_pred")
    if t.shape != p.shape or t.dim() != 4:
        raise ValueError(f"heatmap shapes {tuple(t.shape)} vs {tuple(p.shape)}")
    loss, count = _HeatmapLoss.apply(t.detach(), p, _KIND[kind])
    return (loss, count) if return_count else loss


class _HeatmapMseFromKeypoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kp, vis, preds, height, width, sigma):
        b, k, oh, ow = preds.shape
        out = torch.empty((2,), device=preds.device, dtype=torch.float32)
        ws = torch.empty((b * k * 2,), device=preds.device, dtype=torch.float32)
        with torch.cuda.device(preds.device):
            check(lib.lpb_heatmap_mse_from_keypoints_fwd(_ptr(kp), _ptr(vis), _ptr(preds), b * k, height, width, oh, ow, sigma, _ptr(out), _ptr(ws), _stream()))
        ctx.save_for_backward(kp, vis, preds, out)
        ctx.meta = (height, width, sigma)
        return out[0].clone()

    @staticmethod
    def backward(ctx, g):
        kp, vis, preds, out = ctx.saved_tensors
        return None, None, MseKeypointGrad(kp, vis, preds, out, g.reshape(1).contiguous().float(), ctx.meta), None, None, None


class MseKeypointGrad(torch.Tensor):
    """d loss / d preds of ``heatmap_mse_from_keypoints``, held as what it is computed from (keypoints, visibility, the
    preds, the forward's out, the upstream gradient) rather than as a dense (B, K, h, w) fp32 tensor.

    The bf16 head's backward consumes it as it is when ``preds`` is that head's own output: its kernels rebuild the values
    where they read them (``lpb_head_bwd_bf16_targets``), so the dense gradient is never written.  Any other use -- a
    torch op, autograd adding a second gradient, ``record_stream``, a hook, the tensor ``torch.autograd.grad`` hands back,
    the fp32 head -- goes through ``__torch_dispatch__`` (or ``materialize``), which writes the dense gradient once with
    ``lpb_heatmap_mse_from_keypoints_bwd``, keeps it, and runs the op on it: the same values bit for bit."""

    __torch_function__ = torch._C._disabled_torch_function_impl

    @staticmethod
    def __new__(cls, kp, vis, preds, fwd_out, grad_out, meta):
        t = torch.Tensor._make_wrapper_subclass(cls, preds.shape, strides=preds.stride(), dtype=preds.dtype, device=preds.device)
        t.src = (kp, vis, preds, fwd_out, grad_out, meta)
        t.dense = None
        return t

    def materialize(self) -> torch.Tensor:
        """The dense gradient (written on the current stream at the first call)."""
        if self.dense is None:
            kp, vis, preds, out, gg, (height, width, sigma) = self.src
            b, k, oh, ow = preds.shape
            gp = torch.empty_like(preds)
            with torch.cuda.device(preds.device):
                check(lib.lpb_heatmap_mse_from_keypoints_bwd(_ptr(kp), _ptr(vis), _ptr(preds), b * k, height, width, oh, ow, sigma, _ptr(out), _ptr(gg), _ptr(gp), _stream()))
            self.dense = gp
        return self.dense

    def implicit_for(self, heatmaps: torch.Tensor) -> bool:
        """Whether a backward that owns ``heatmaps`` may take this gradient implicitly: not yet materialised, and the loss
        read exactly ``heatmaps`` (same memory, shape and strides)."""
        preds = self.src[2]
        return (self.dense is None and preds.data_ptr() == heatmaps.data_ptr() and preds.shape == heatmaps.shape
                and preds.stride() == heatmaps.stride() and preds.dtype == heatmaps.dtype)

    def targets(self) -> MseTargets:
        """The ``lpb_mse_targets`` descriptor of this gradient (device pointers; the tensors stay alive with ``self``)."""
        kp, vis, _, out, gg, (height, width, sigma) = self.src
        return MseTargets(kp.data_ptr(), vis.data_ptr() if vis is not None else None, height, width, sigma, out.data_ptr(), gg.data_ptr())

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        dense = lambda x: x.materialize() if isinstance(x, MseKeypointGrad) else x
        return func(*torch.utils._pytree.tree_map(dense, args), **torch.utils._pytree.tree_map(dense, kwargs or {}))


def heatmap_mse_from_keypoints(keypoints, preds, height, width, sigma=1.25, visibility=None):
    """Fused target generation + HeatmapMSELoss (targets never written to HBM); differentiable in ``preds``."""
    kp = _cuda_f32(keypoints, "keypoints").detach()
    p = _cuda_f32(preds, "heatmaps_pred")
    vis = visibility.to(torch.int32).contiguous() if visibility is not None else None
    return _HeatmapMseFromKeypoints.apply(kp, vis, p, float(height), float(width), float(sigma))


class _HeatmapLossFromKeypoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kp, vis, preds, height, width, sigma, kind):
        b, k, oh, ow = preds.shape
        out = torch.empty((2,), device=preds.device, dtype=torch.float32)
        ws = torch.empty((b * k * 2,), device=preds.device, dtype=torch.float32)
        with torch.cuda.device(preds.device):
            check(lib.lpb_heatmap_loss_from_keypoints_fwd(_ptr(kp), _ptr(vis), _ptr(preds), b * k, height, width, oh, ow, sigma, kind,
                                                          _ptr(out), _ptr(ws), _stream()))
        ctx.save_for_backward(kp, vis, preds, out)
        ctx.meta = (height, width, sigma, kind)
        loss, count = out[0].clone(), out[1].clone()
        ctx.mark_non_differentiable(count)
        return loss, count

    @staticmethod
    def backward(ctx, g, _g_count):
        kp, vis, preds, out = ctx.saved_tensors
        height, width, sigma, kind = ctx.meta
        b, k, oh, ow = preds.shape
        gp = torch.empty_like(preds)
        gg = g.reshape(1).contiguous().float()
        with torch.cuda.device(preds.device):
            check(lib.lpb_heatmap_loss_from_keypoints_bwd(_ptr(kp), _ptr(vis), _ptr(preds), b * k, height, width, oh, ow, sigma, kind,
                                                          _ptr(out), _ptr(gg), _ptr(gp), _stream()))
        return None, None, gp, None, None, None, None


def heatmap_loss_from_keypoints(kind: str, keypoints, preds, height, width, sigma=1.25, visibility=None, return_count: bool = False):
    """Fused target generation + HeatmapMSELoss / KLLoss / JSLoss (``kind`` "mse" | "kl" | "js"): the Gaussian targets of
    ``keypoints`` (B, K, 2) image pixels are made where ``preds`` (B, K, oh, ow) is read and never written; differentiable
    in ``preds``.  With ``return_count`` also the number of kept planes (a non-differentiable device scalar).

    "mse" without the count is ``heatmap_mse_from_keypoints`` (whose gradient the bf16 head takes implicitly); the other
    kinds, and "mse" with the count, write the dense gradient once in the backward."""
    if kind == "mse" and not return_count:
        return heatmap_mse_from_keypoints(keypoints, preds, height, width, sigma, visibility)
    kp = _cuda_f32(keypoints, "keypoints").detach()
    p = _cuda_f32(preds, "heatmaps_pred")
    vis = visibility.to(torch.int32).contiguous() if visibility is not None else None
    planes = p.shape[0] * p.shape[1] if p.dim() == 4 else -1
    if planes < 0 or kp.numel() != 2 * planes or (vis is not None and vis.numel() != planes):
        raise ValueError(f"heatmap_loss_from_keypoints: keypoints {tuple(kp.shape)}, visibility "
                         f"{None if vis is None else tuple(vis.shape)} do not match preds {tuple(p.shape)} (B, K, h, w)")
    loss, count = _HeatmapLossFromKeypoints.apply(kp, vis, p, float(height), float(width), float(sigma), _KIND[kind])
    return (loss, count) if return_count else loss


class _TemporalHeatmapLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hm, cf, eps, kind, prob_threshold):
        t, k, h, w = hm.shape
        out = torch.empty((1,), device=hm.device, dtype=torch.float32)
        ws = torch.empty((max(t - 1, 1) * k,), device=hm.device, dtype=torch.float32)
        with torch.cuda.device(hm.device):
            check(lib.lpb_temporal_heatmap_loss_fwd(_ptr(hm), _ptr(cf), t, k, h, w, kind, _ptr(eps), float(prob_threshold), _ptr(out), _ptr(ws), _stream()))
        ctx.save_for_backward(hm, cf, eps, ws)
        ctx.meta = (kind, float(prob_threshold))
        return out[0]

    @staticmethod
    def backward(ctx, g):
        hm, cf, eps, ws = ctx.saved_tensors
        kind, thr = ctx.meta
        t, k, h, w = hm.shape
        gh = torch.empty_like(hm)
        gg = g.reshape(1).contiguous().float()
        with torch.cuda.device(hm.device):
            check(lib.lpb_temporal_heatmap_loss_bwd(_ptr(hm), _ptr(cf), _ptr(ws), t, k, h, w, kind, _ptr(eps), thr, _ptr(gg), _ptr(gh), _stream()))
        return gh, None, None, None, None


def temporal_heatmap_loss(heatmaps, confidences, kind: str, epsilon: torch.Tensor, prob_threshold: float):
    """TemporalHeatmapLoss (mse | kl) over consecutive frames; differentiable in ``heatmaps``."""
    hm = _cuda_f32(heatmaps, "heatmaps_pred")
    cf = _cuda_f32(confidences, "confidences").detach()
    k = hm.shape[1]
    eps = _cuda_f32(epsilon.to(hm.device).reshape(-1).expand(k) if epsilon.numel() in (1, k) else epsilon, "epsilon")
    if hm.shape[0] < 2:
        raise ValueError("temporal heatmap loss needs at least two frames")
    return _TemporalHeatmapLoss.apply(hm, cf, eps, _KIND[kind], float(prob_threshold))


# =====================================================================================
# unsupervised losses on (T, K, 2)
# =====================================================================================
class PcaParams:
    """Device-side parameters of one PCA loss (mirror of ``lpb_pca_desc``)."""

    def __init__(self, kp_index, n_sel, n_views, centering, mean, kept, epsilon, device):
        # the index range stays on the host, so that unsup_losses can check it against K without a device sync
        idx = np.asarray(kp_index).reshape(-1)
        self.kp_index_min = int(idx.min()) if idx.size else 0
        self.kp_index_max = int(idx.max()) if idx.size else -1
        self.kp_index = torch.as_tensor(kp_index, dtype=torch.int32, device=device).contiguous()
        self.mean = torch.as_tensor(mean, dtype=torch.float32, device=device).contiguous()
        self.kept = torch.as_tensor(kept, dtype=torch.float32, device=device).contiguous().reshape(-1, self.mean.numel())
        self.n_sel, self.n_views = int(n_sel), int(n_views)
        self.centering = {None: 0, "mean": 1, "median": 2}[centering]
        self.epsilon = float(epsilon)
        d = 2 * self.n_views if self.n_views > 0 else 2 * self.n_sel
        if self.mean.numel() != d or self.kept.shape[1] != d:
            raise ValueError(f"PCA parameter dimension mismatch: D={d}, mean={self.mean.numel()}, kept={tuple(self.kept.shape)}")

    def desc(self) -> PcaDesc:
        return PcaDesc(self.kp_index.data_ptr(), self.n_sel, self.n_views, self.centering, self.kept.shape[0],
                       self.mean.data_ptr(), self.kept.data_ptr(), self.epsilon)


class _UnsupLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, confidences, temporal_eps, prob_threshold, temporal_on, sv, mv):
        n_clips, t, k2 = keypoints.shape
        out = torch.empty((n_clips, 4), device=keypoints.device, dtype=torch.float32)
        dsv = sv.desc() if sv is not None else None
        dmv = mv.desc() if mv is not None else None
        with torch.cuda.device(keypoints.device):
            check(lib.lpb_unsup_losses_fwd(_ptr(keypoints), _ptr(confidences), n_clips, t, k2 // 2, _ptr(temporal_eps), float(prob_threshold), int(temporal_on),
                                           C.byref(dsv) if dsv else None, C.byref(dmv) if dmv else None, _ptr(out), _stream()))
        ctx.save_for_backward(keypoints, confidences, temporal_eps)
        ctx.meta = (float(prob_threshold), int(temporal_on), sv, mv)
        return out

    @staticmethod
    def backward(ctx, g):
        keypoints, confidences, temporal_eps = ctx.saved_tensors
        thr, temporal_on, sv, mv = ctx.meta
        n_clips, t, k2 = keypoints.shape
        gk = torch.empty_like(keypoints)
        dsv = sv.desc() if sv is not None else None
        dmv = mv.desc() if mv is not None else None
        gg = g.contiguous().float()
        with torch.cuda.device(keypoints.device):
            check(lib.lpb_unsup_losses_bwd(_ptr(keypoints), _ptr(confidences), n_clips, t, k2 // 2, _ptr(temporal_eps), thr, temporal_on,
                                           C.byref(dsv) if dsv else None, C.byref(dmv) if dmv else None, _ptr(gg), _ptr(gk), _stream()))
        return gk, None, None, None, None, None, None


def unsup_losses(keypoints, confidences=None, temporal_eps=None, prob_threshold=0.0, pca_singleview: PcaParams | None = None,
                 pca_multiview: PcaParams | None = None):
    """One launch for the unsupervised loss stack.  keypoints (n_clips, T, 2K) or (T, 2K).

    Returns (n_clips, 4) = [temporal, pca_singleview, pca_multiview, 0] per clip (or (4,) for 2-D input).
    A NaN keypoint makes the losses that read it NaN, as in the reference.
    """
    k = keypoints.shape[-1] // 2
    for name, p in (("pca_singleview", pca_singleview), ("pca_multiview", pca_multiview)):
        if p is not None and p.n_sel > 0 and (p.kp_index_min < 0 or p.kp_index_max >= k):
            raise ValueError(f"{name}: keypoint indices span [{p.kp_index_min}, {p.kp_index_max}], outside [0, {k}) "
                             f"for {k} keypoints")
    kp = _cuda_f32(keypoints, "keypoints_pred")
    squeeze = kp.dim() == 2
    if squeeze:
        kp = kp[None]
    cf = None
    if confidences is not None:
        cf = _cuda_f32(confidences, "confidences").reshape(kp.shape[0], kp.shape[1], -1)
    k = kp.shape[2] // 2
    te = None
    if temporal_eps is not None:
        te = torch.as_tensor(temporal_eps, dtype=torch.float32, device=kp.device).reshape(-1)
        te = (te.expand(k) if te.numel() == 1 else te).contiguous()
        if te.numel() != k:
            raise ValueError(f"temporal epsilon has {te.numel()} entries for {k} keypoints")
    out = _UnsupLosses.apply(kp, cf, te, prob_threshold, te is not None, pca_singleview, pca_multiview)
    return out[0] if squeeze else out


# =====================================================================================
# calibrated multi-view geometry (csrc/cameras.cu)
# =====================================================================================
_DIST_PARAMS = (4, 5, 8, 12)


def _camera_tensors(intrinsics, extrinsics, dist, b, v):
    """Batch-dict camera tensors -> contiguous fp32 CUDA tensors of the checked shapes (no gradient: batch data)."""
    k = _cuda_f32(intrinsics, "intrinsics").detach()
    e = _cuda_f32(extrinsics, "extrinsics").detach()
    d = _cuda_f32(dist, "dist").detach()
    if tuple(k.shape) != (b, v, 3, 3) or tuple(e.shape) != (b, v, 3, 4) or d.dim() != 3 or tuple(d.shape[:2]) != (b, v):
        raise ValueError(f"cameras for {b} x {v} views: intrinsics {tuple(k.shape)} (want (B, V, 3, 3)), extrinsics "
                         f"{tuple(e.shape)} (want (B, V, 3, 4)), dist {tuple(d.shape)} (want (B, V, P))")
    if d.shape[-1] not in _DIST_PARAMS:
        raise ValueError(f"dist has {d.shape[-1]} coefficients per view; supported: 4, 5, 8 or 12 (tilt distortion, 14, is not)")
    return k, e, d


class _TriangulatePairs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pts, k, e, d):
        b, v, n, _ = pts.shape
        out = torch.empty((b, v * (v - 1) // 2, n, 3), device=pts.device, dtype=torch.float32)
        with torch.cuda.device(pts.device):
            check(lib.lpb_triangulate_pairs_fwd(_ptr(pts), _ptr(k), _ptr(e), _ptr(d), b, v, n, d.shape[-1], _ptr(out), _stream()))
        ctx.save_for_backward(pts, k, e, d)
        return out

    @staticmethod
    def backward(ctx, g):
        pts, k, e, d = ctx.saved_tensors
        b, v, n, _ = pts.shape
        g = g.contiguous().float()
        gp = torch.empty_like(pts)
        with torch.cuda.device(pts.device):
            check(lib.lpb_triangulate_pairs_bwd(_ptr(pts), _ptr(k), _ptr(e), _ptr(d), _ptr(g), b, v, n, d.shape[-1], _ptr(gp), _stream()))
        return gp, None, None, None


def triangulate_pairs(points, intrinsics, extrinsics, dist):
    """(B, V, K, 2) frame pixels -> (B, V(V-1)/2, K, 3): undistort, then DLT per camera pair (combinations order).
    Differentiable in ``points``."""
    pts = _cuda_f32(points, "points")
    if pts.dim() != 4 or pts.shape[-1] != 2 or pts.shape[1] < 2:
        raise ValueError(f"points must be (batch, num_views >= 2, num_keypoints, 2); got {tuple(pts.shape)}")
    k, e, d = _camera_tensors(intrinsics, extrinsics, dist, pts.shape[0], pts.shape[1])
    return _TriangulatePairs.apply(pts, k, e, d)


class _ProjectPoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p3, n_pairs, k, e, d, bbox, model_height, model_width):
        b, v = k.shape[:2]
        n = p3.shape[-2]
        out = torch.empty((b, v, n, 2), device=p3.device, dtype=torch.float32)
        with torch.cuda.device(p3.device):
            check(lib.lpb_project_points_fwd(_ptr(p3), n_pairs, _ptr(k), _ptr(e), _ptr(d), _ptr(bbox), model_height, model_width,
                                             b, v, n, d.shape[-1], _ptr(out), _stream()))
        ctx.save_for_backward(p3, k, e, d, bbox)
        ctx.meta = (n_pairs, model_height, model_width)
        return out

    @staticmethod
    def backward(ctx, g):
        p3, k, e, d, bbox = ctx.saved_tensors
        n_pairs, mh, mw = ctx.meta
        b, v = k.shape[:2]
        g = g.contiguous().float()
        gp = torch.empty_like(p3)
        with torch.cuda.device(p3.device):
            check(lib.lpb_project_points_bwd(_ptr(p3), n_pairs, _ptr(k), _ptr(e), _ptr(d), _ptr(bbox), mh, mw, _ptr(g),
                                             b, v, p3.shape[-2], d.shape[-1], _ptr(gp), _stream()))
        return gp, None, None, None, None, None, None, None


def project_points(points_3d, intrinsics, extrinsics, dist, mean_over_pairs=False, bbox=None, model_size=None):
    """(B, K, 3) world points -> (B, V, K, 2) frame pixels (pinhole K E, then distortion where a view has any).

    ``mean_over_pairs``: ``points_3d`` is (B, pairs, K, 3) and is averaged over the pair axis first (NaN-propagating, as
    ``torch.mean(dim=1)``).  ``bbox`` (B, 4V) with ``model_size`` (height, width): the result is in model coordinates
    (``frame_to_model``).  One launch each way; differentiable in ``points_3d``."""
    if mean_over_pairs and points_3d.dim() == 4 and points_3d.shape[1] == 0:
        # the kernels read n_pairs = 0 as "no pair axis": a zero-width slice would project its parent's first points
        raise ValueError(f"points_3d has no pairs to average over: {tuple(points_3d.shape)}")
    p3 = _cuda_f32(points_3d, "points_3d")
    if p3.shape[-1] != 3 or p3.dim() != (4 if mean_over_pairs else 3):
        raise ValueError(f"points_3d must be {'(batch, pairs, num_keypoints, 3)' if mean_over_pairs else '(batch, num_keypoints, 3)'}; got {tuple(p3.shape)}")
    b, v = p3.shape[0], intrinsics.shape[1]
    k, e, d = _camera_tensors(intrinsics, extrinsics, dist, b, v)
    bb, mh, mw = None, 0.0, 0.0
    if bbox is not None:
        bb = _cuda_f32(bbox, "bbox").detach()
        if tuple(bb.shape) != (b, 4 * v) or model_size is None:
            raise ValueError(f"bbox must be (batch, 4 * num_views) = ({b}, {4 * v}) with a model_size; got {tuple(bb.shape)}")
        mh, mw = float(model_size[0]), float(model_size[1])
    return _ProjectPoints.apply(p3, p3.shape[1] if mean_over_pairs else 0, k, e, d, bb, mh, mw)


class _FrameToModel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kp, bbox, model_height, model_width):
        b, v, n, _ = kp.shape
        out = torch.empty_like(kp)
        with torch.cuda.device(kp.device):
            check(lib.lpb_frame_to_model(_ptr(kp), b, v, n, _ptr(bbox), model_height, model_width, 0, _ptr(out), _stream()))
        ctx.save_for_backward(bbox)
        ctx.meta = (model_height, model_width)
        return out

    @staticmethod
    def backward(ctx, g):
        (bbox,) = ctx.saved_tensors
        mh, mw = ctx.meta
        g = g.contiguous().float()
        b, v, n, _ = g.shape
        gi = torch.empty_like(g)
        with torch.cuda.device(g.device):
            check(lib.lpb_frame_to_model(_ptr(g), b, v, n, _ptr(bbox), mh, mw, 1, _ptr(gi), _stream()))
        return gi, None, None, None


def frame_to_model(keypoints, bbox, model_height, model_width):
    """(B, V, K, 2) frame pixels -> model pixels with per-view bbox [x, y, h, w] (B, 4V); differentiable in keypoints."""
    kp = _cuda_f32(keypoints, "frame_keypoints")
    if kp.dim() != 4 or kp.shape[-1] != 2:
        raise ValueError(f"frame_keypoints must be (batch, num_views, num_keypoints, 2); got {tuple(kp.shape)}")
    bb = _cuda_f32(bbox, "bbox").detach()
    if tuple(bb.shape) != (kp.shape[0], 4 * kp.shape[1]):
        raise ValueError(f"bbox must be (batch, 4 * num_views) = ({kp.shape[0]}, {4 * kp.shape[1]}); got {tuple(bb.shape)}")
    return _FrameToModel.apply(kp, bb, float(model_height), float(model_width))


class _PairwiseProjectionsLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, targ, pred):
        b, p, n, _ = pred.shape
        out = torch.empty((2,), device=pred.device, dtype=torch.float32)
        with torch.cuda.device(pred.device):
            check(lib.lpb_pairwise_projections_loss_fwd(_ptr(targ), _ptr(pred), b, p, n, _ptr(out), _stream()))
        ctx.save_for_backward(targ, pred, out)
        loss, count = out[0].clone(), out[1].clone()
        ctx.mark_non_differentiable(count)
        return loss, count

    @staticmethod
    def backward(ctx, g, _g_count):
        targ, pred, out = ctx.saved_tensors
        b, p, n, _ = pred.shape
        gp = torch.empty_like(pred)
        gg = g.reshape(1).contiguous().float()
        with torch.cuda.device(pred.device):
            check(lib.lpb_pairwise_projections_loss_bwd(_ptr(targ), _ptr(pred), b, p, n, _ptr(out), _ptr(gg), _ptr(gp), _stream()))
        return None, gp


def pairwise_projections_loss(targets, preds, return_count=False):
    """Mean L2 distance between targets (B, K, 3) and per-pair predictions (B, pairs, K, 3) over entries with neither
    side NaN; 0 (with a zero gradient) when there is none.  Differentiable in ``preds``."""
    t = _cuda_f32(targets, "keypoints_targ_3d").detach()
    p = _cuda_f32(preds, "keypoints_pred_3d")
    if t.dim() != 3 or p.dim() != 4 or t.shape[-1] != 3 or p.shape[-1] != 3 or t.shape[0] != p.shape[0] or t.shape[1] != p.shape[2]:
        raise ValueError(f"targets (batch, num_keypoints, 3) vs predictions (batch, pairs, num_keypoints, 3): {tuple(t.shape)} / {tuple(p.shape)}")
    loss, count = _PairwiseProjectionsLoss.apply(t, p)
    return (loss, count) if return_count else loss


# =====================================================================================
# coordinate-regression models (csrc/regression.cu)
# =====================================================================================
_FEATURE_FORMAT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}  # LPB_OUT_* (lpb200.h)


class _RegressionHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, layout, weight, bias):
        b, c, h, w = features.shape
        n = weight.shape[0]
        pooled = torch.empty((b, c), device=features.device, dtype=torch.float32)
        out = torch.empty((b, n), device=features.device, dtype=torch.float32)
        fmt = _FEATURE_FORMAT[features.dtype]
        with torch.cuda.device(features.device):
            check(lib.lpb_regression_head_fwd(_ptr(features), fmt, layout, b, c, h, w, _ptr(weight), _ptr(bias), n, _ptr(pooled),
                                              _ptr(out), _stream()))
        ctx.save_for_backward(pooled, weight)
        ctx.meta = (fmt, layout, tuple(features.shape), features.dtype)
        return out

    @staticmethod
    def backward(ctx, g):
        pooled, weight = ctx.saved_tensors
        fmt, layout, (b, c, h, w), dtype = ctx.meta
        n = weight.shape[0]
        g = g.contiguous().float()
        dfeat = dw = db = ws = None
        if ctx.needs_input_grad[0]:
            memory = torch.channels_last if layout == FEATURES_NHWC else torch.contiguous_format
            dfeat = torch.empty((b, c, h, w), device=g.device, dtype=dtype, memory_format=memory)
            ws = torch.empty((b, c), device=g.device, dtype=torch.float32)
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            dw, db = torch.empty_like(weight), torch.empty((n,), device=g.device, dtype=torch.float32)
        with torch.cuda.device(g.device):
            check(lib.lpb_regression_head_bwd(_ptr(g), _ptr(pooled), _ptr(weight), fmt, layout, b, c, h, w, n, _ptr(dfeat), _ptr(dw),
                                              _ptr(db), _ptr(ws), _stream()))
        return dfeat, None, dw, db


def regression_head(features, weight, bias):
    """``mean over (h, w) of features`` then ``nn.Linear``: (B, C, h, w) -> (B, N) fp32, forward and both gradients in
    ``liblpb200.so``.  Features in bf16, fp16 or fp32, NCHW or channels-last (read in place, ``feature_layout``); the
    gradient comes back in the same dtype and layout.  Differentiable in features, weight and bias."""
    if not isinstance(features, torch.Tensor) or not features.is_cuda:
        raise RuntimeError("lpb200: `features` must be a CUDA tensor (this package has no CPU fallback)")
    if features.dim() != 4:
        raise ValueError(f"features must be (batch, channels, height, width); got {tuple(features.shape)}")
    if features.dtype not in _FEATURE_FORMAT:
        raise ValueError(f"features must be float32, bfloat16 or float16; got {features.dtype}")
    if weight.dim() != 2 or weight.shape[1] != features.shape[1] or bias.shape != (weight.shape[0],):
        raise ValueError(f"weight (N, C) / bias (N,) for C = {features.shape[1]}: {tuple(weight.shape)} / {tuple(bias.shape)}")
    layout = feature_layout(features)
    f = features if layout == FEATURES_NHWC else features.contiguous()
    return _RegressionHead.apply(f, layout, _cuda_f32(weight, "weight"), _cuda_f32(bias, "bias"))


class _RegressionLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, targ, pred):
        out = torch.empty((4,), device=pred.device, dtype=torch.float32)
        with torch.cuda.device(pred.device):
            check(lib.lpb_regression_losses_fwd(_ptr(targ), _ptr(pred), pred.numel(), _ptr(out), _stream()))
        ctx.save_for_backward(targ, pred, out)
        mse, kept, rmse, pairs = (out[i].clone() for i in range(4))
        ctx.mark_non_differentiable(kept, rmse, pairs)
        return mse, kept, rmse, pairs

    @staticmethod
    def backward(ctx, g, _g_kept, _g_rmse, _g_pairs):
        targ, pred, out = ctx.saved_tensors
        gp = torch.empty_like(pred)
        gg = g.reshape(1).contiguous().float()
        with torch.cuda.device(pred.device):
            check(lib.lpb_regression_losses_bwd(_ptr(targ), _ptr(pred), pred.numel(), _ptr(out), _ptr(gg), _ptr(gp), _stream()))
        return None, gp


def regression_losses(targets, preds):
    """``(mse, kept, rmse, pairs)`` of (B, 2K) keypoint targets and predictions in one launch, with no host sync.

    ``mse``: mean of (t - p)^2 over the entries whose target is not NaN (NaN when there is none), differentiable in
    ``preds``.  ``rmse``: the reference's diagnostic, the kept squared errors compacted in order and paired as (x, y),
    mean of sqrt(pair mean); NaN when nothing is kept or an odd number is.  ``kept`` / ``pairs``: the counts."""
    t = _cuda_f32(targets, "keypoints_targ").detach()
    p = _cuda_f32(preds, "keypoints_pred")
    if t.shape != p.shape:
        raise ValueError(f"keypoint targets {tuple(t.shape)} and predictions {tuple(p.shape)} differ in shape")
    return _RegressionLosses.apply(t, p)
