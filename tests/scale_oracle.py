"""float64 references of the hot path for batch-size (scale) tests.  TEST INFRASTRUCTURE ONLY.

Every function computes in float64 on the device of its inputs (or the ``device`` it is given), so the result does not
depend on TF32 / cuDNN settings and no global flag is touched.  Large inputs are processed in chunks of planes or
frames so that peak memory stays around 2 GB.  The functions restate the CPU oracle (``oracle/lp_oracle.py``) where that
one is fixed to float32 or to the CPU, and reuse it where it keeps dtype and device; ``tests/test_scale_oracle.py``
pins every function here to the oracle and to the golden vectors.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import lp_oracle as O

F64 = torch.float64
_CHUNK_ELEMS = 1 << 25  # float64 elements of one chunk's largest intermediate (256 MB)

_DECODE_OFFSET = {1: 0.5, 2: 1.5, 3: 2.5}  # lightning_pose/models/heads/heatmap.py:131-136
_U_CACHE: dict = {}


def upsample_op(n: int, ds: int, device) -> torch.Tensor:
    """(n * 2^ds, n) float64 matrix U with upsample^ds(h) = U_H h U_W^T (pinned by the golden ``U_*`` matrices)."""
    key = (n, ds, str(device))
    if key not in _U_CACHE:
        _U_CACHE[key] = torch.from_numpy(O.upsample_matrix_1d(n, ds)).to(device=device, dtype=F64)
    return _U_CACHE[key]


def _chunk(per_item: int) -> int:
    return max(1, _CHUNK_ELEMS // max(1, per_item))


# ------------------------------------------------------------------------------------------------
# soft-argmax decode
# ------------------------------------------------------------------------------------------------
def _window_sums(p: torch.Tensor, cx: torch.Tensor, cy: torch.Tensor, r: int = 2) -> torch.Tensor:
    """sum of the (2r+1)^2 window of the planes p (n, H, W) around integer centres (cx, cy), zero outside the plane."""
    n, hh, ww = p.shape
    padded = F.pad(p, (r, r, r, r))
    offs = torch.arange(2 * r + 1, device=p.device)
    rows = (cy.long()[:, None] + offs[None, :]).clamp(0, hh + 2 * r - 1)
    cols = (cx.long()[:, None] + offs[None, :]).clamp(0, ww + 2 * r - 1)
    idx = torch.arange(n, device=p.device)[:, None, None]
    return padded[idx, rows[:, :, None], cols[:, None, :]].sum((-1, -2))


def _decode_planes(h: torch.Tensor, ds: int, temperature: float, trunc_eps: float):
    n, hh, ww = h.shape
    uh, uw = upsample_op(hh, ds, h.device), upsample_op(ww, ds, h.device)
    field = torch.matmul(torch.matmul(uh, h), uw.T)  # (n, H, W)
    big_h, big_w = field.shape[-2:]
    p = torch.softmax(field.reshape(n, -1) * temperature, -1).reshape(n, big_h, big_w)
    cols = torch.arange(big_w, device=h.device, dtype=F64)
    rows = torch.arange(big_h, device=h.device, dtype=F64)
    x = (p.sum(1) * cols).sum(-1)
    y = (p.sum(2) * rows).sum(-1)
    pre = torch.stack([x, y], -1)
    with torch.no_grad():
        # confidence window at trunc() of the pre-offset coordinates (lightning_pose/data/heatmaps.py:90-142); the
        # alternatives take the window on the other side of an integer within trunc_eps of a coordinate
        confs = []
        for sx, sy in ((0.0, 0.0), (-trunc_eps, 0.0), (trunc_eps, 0.0), (0.0, -trunc_eps), (0.0, trunc_eps),
                       (-trunc_eps, -trunc_eps), (-trunc_eps, trunc_eps), (trunc_eps, -trunc_eps), (trunc_eps, trunc_eps)):
            confs.append(_window_sums(p, torch.trunc(x.detach() + sx), torch.trunc(y.detach() + sy)))
        conf_alt = torch.stack(confs, -1)
    return pre, conf_alt


def decode_ref(hm: torch.Tensor, ds: int, temperature: float = 1000.0, trunc_eps: float = 1e-3):
    """Soft-argmax decode of (B, K, h, w) heatmaps in float64.

    Returns ``(preds (B, 2K), conf (B, K), pre (B, K, 2), conf_alt (B, K, 9))``: preds after the ``{0.5, 1.5, 2.5}``
    offset; ``pre`` the coordinates before it; ``conf`` the window sum at trunc(pre); ``conf_alt[..., i]`` the window
    sums at trunc(pre + s) for the nine shifts s in {-eps, 0, eps}^2 (index 0 is ``conf``).  Where no coordinate lies
    within ``trunc_eps`` of an integer all nine are equal.  Differentiable in ``hm`` through ``preds`` / ``pre``.
    """
    b, k, hh, ww = hm.shape
    flat = hm.reshape(b * k, hh, ww).to(F64)
    step = _chunk(hh * ww * 4**ds)
    pres, alts = [], []
    for i in range(0, b * k, step):
        pre, alt = _decode_planes(flat[i : i + step], ds, temperature, trunc_eps)
        pres.append(pre)
        alts.append(alt)
    pre = torch.cat(pres).reshape(b, k, 2)
    conf_alt = torch.cat(alts).reshape(b, k, 9)
    preds = (pre - _DECODE_OFFSET[ds]).reshape(b, 2 * k)
    return preds, conf_alt[..., 0], pre, conf_alt


def decode_grad_ref(hm: torch.Tensor, ds: int, temperature: float, grad_xy: torch.Tensor) -> torch.Tensor:
    """d sum(preds * grad_xy) / d hm by float64 autograd of ``decode_ref``, chunk by chunk; (B, K, h, w) float64."""
    b, k, hh, ww = hm.shape
    flat = hm.reshape(b * k, hh, ww)
    g = grad_xy.reshape(b * k, 2).to(F64)
    out = torch.empty((b * k, hh, ww), device=hm.device, dtype=F64)
    step = _chunk(hh * ww * 4**ds * 3)
    for i in range(0, b * k, step):
        x = flat[i : i + step].to(F64).requires_grad_(True)
        pre, _ = _decode_planes(x, ds, temperature, 0.0)
        (out[i : i + step],) = torch.autograd.grad((pre * g[i : i + step]).sum(), x)
    return out.reshape(b, k, hh, ww)


# ------------------------------------------------------------------------------------------------
# heatmap head
# ------------------------------------------------------------------------------------------------
def operand_round(t: torch.Tensor, dtype) -> torch.Tensor:
    """t rounded to the 16-bit ``dtype`` (round to nearest even, from its float32 value), straight-through for autograd."""
    return t + (t.detach().float().to(dtype).to(t.dtype) - t.detach())


def head_ref(feats: torch.Tensor, weights, biases, softmax: bool = True, operands=torch.bfloat16, mids: list | None = None):
    """PixelShuffle(2) + ConvTranspose2d(k3, s2, p1, op1) per layer [+ spatial softmax], float64, on feats' device.

    ``operands`` (None, ``torch.bfloat16`` or ``torch.float16``): the weights and the inputs of layers after the first are
    rounded to that dtype where the tensor-core kernels round them (the features are taken as given).  The fp16 route
    also rounds the biases of layers after the first, which ride on the constant-one channel as fp16 operands; the bf16
    reference leaves them unrounded.  Differentiable in every input.  ``mids``: if a list, the input of every layer after
    the first is appended to it (with ``retain_grad``)."""
    x = F.pixel_shuffle(feats.to(F64), 2)
    for i, (w, b) in enumerate(zip(weights, biases)):
        w = w.to(device=x.device, dtype=F64)
        b = b.to(device=x.device, dtype=F64)
        if i:
            if mids is not None:
                x.retain_grad()
                mids.append(x)
            if operands is not None:
                x = operand_round(x, operands)
            if operands == torch.float16:
                b = operand_round(b, operands)
        x = F.conv_transpose2d(x, w if operands is None else operand_round(w, operands), b, stride=2, padding=1, output_padding=1)
    if softmax:
        n, c, hh, ww = x.shape
        x = torch.softmax(x.reshape(n, c, -1), -1).reshape(n, c, hh, ww)
    return x


def head_ref_chunked(feats: torch.Tensor, weights, biases, softmax: bool = True, operands=torch.bfloat16) -> torch.Tensor:
    """``head_ref`` without autograd, frame chunk by frame chunk."""
    out = []
    step = _chunk(feats[0].numel() * 8)
    with torch.no_grad():
        for i in range(0, feats.shape[0], step):
            out.append(head_ref(feats[i : i + step], weights, biases, softmax, operands))
    return torch.cat(out)


def head_grad_ref(feats, weights, biases, grad_out, softmax: bool = True, operands=torch.bfloat16, want_mid_grad=False):
    """float64 autograd of sum(head_ref(...) * grad_out), frame chunk by frame chunk.

    Returns (dfeat, [dw], [db][, per-channel L2 norm of d(input of the last layer)] )."""
    ws = [w.detach().to(F64).requires_grad_(True) for w in weights]
    bs = [b.detach().to(F64).requires_grad_(True) for b in biases]
    dfeat = torch.empty(feats.shape, device=feats.device, dtype=F64)
    sq = None
    step = _chunk(feats[0].numel() * 8)
    for i in range(0, feats.shape[0], step):
        f = feats[i : i + step].detach().to(F64).requires_grad_(True)
        mids: list = []
        y = head_ref(f, ws, bs, softmax, operands, mids=mids if want_mid_grad else None)
        (y * grad_out[i : i + step].to(F64)).sum().backward()
        dfeat[i : i + step] = f.grad
        if want_mid_grad:
            s = mids[-1].grad.pow(2).sum((0, 2, 3))
            sq = s if sq is None else sq + s
    res = (dfeat, [w.grad for w in ws], [b.grad for b in bs])
    return res + (sq.sqrt(),) if want_mid_grad else res


# ------------------------------------------------------------------------------------------------
# loss stack
# ------------------------------------------------------------------------------------------------
def gaussian_targets_ref(keypoints, height, width, output_shape, sigma=1.25, visibility=None) -> torch.Tensor:
    """``O.gaussian_targets`` (lightning_pose/data/heatmaps.py:37-87) in float64 on the keypoints' device."""
    oh, ow = int(output_shape[0]), int(output_shape[1])
    dev = keypoints.device
    kp = keypoints.detach().to(F64)
    x = kp[..., 0] * (ow / width)
    y = kp[..., 1] * (oh / height)
    bad = torch.isnan(x) | (x < -1) | (x > ow + 1) | (y < -1) | (y > oh + 1)
    xc = torch.clamp(x, -1, ow + 1)[..., None, None]
    yc = torch.clamp(y, -1, oh + 1)[..., None, None]
    cols = torch.arange(ow, dtype=F64, device=dev)
    rows = torch.arange(oh, dtype=F64, device=dev)[:, None]
    g = torch.exp(-((cols - xc) ** 2 + (rows - yc) ** 2) / (2.0 * sigma**2))
    g = g / g.sum(dim=(2, 3), keepdim=True)
    zero = torch.zeros((), dtype=F64, device=dev)
    if visibility is None:
        return torch.where(bad[..., None, None], zero, g)
    vis = visibility.to(dev)[..., None, None]
    g = torch.where(vis == 0, zero, g)
    g = torch.where(vis == 1, torch.full((), 1.0 / (oh * ow), dtype=F64, device=dev), g)
    return torch.where((vis == 2) & bad[..., None, None], zero, g)


def _plane_terms(t: torch.Tensor, p: torch.Tensor, kind: str) -> torch.Tensor:
    """per-plane loss sum of (n, h, w) targets / predictions (losses.py:314-335, :360-378, :404-423)."""
    if kind == "mse":
        return ((t - p) ** 2).sum((-1, -2)) * (t.shape[-1] * t.shape[-2])
    tt, pp = t + 1e-10, p + 1e-10
    if kind == "kl":
        return (tt * (torch.log(tt) - torch.log(pp))).sum((-1, -2))
    m = 0.5 * (tt + pp)
    lm = torch.log(m)
    return 0.5 * (tt * (torch.log(tt) - lm) + pp * (torch.log(pp) - lm)).sum((-1, -2))


def heatmap_loss_ref(targets: torch.Tensor, preds: torch.Tensor, kind: str, with_grad: bool = False):
    """HeatmapMSE/KL/JS loss over the planes whose target is not all-zero (losses.py:246-249), float64.

    The MSE is the mean over the kept planes' pixels (so the plane sum above is divided by h*w again); KL / JS the mean
    over kept planes.  ``with_grad``: also d loss / d preds (float64 autograd, plane chunk by plane chunk)."""
    b, k, hh, ww = preds.shape
    t = targets.reshape(b * k, hh, ww)
    p = preds.reshape(b * k, hh, ww)
    keep = ~torch.all(t == 0, dim=(-1, -2))
    n_keep = int(keep.sum())
    denom = n_keep * (hh * ww if kind == "mse" else 1)
    step = _chunk(hh * ww * 6)
    total = torch.zeros((), dtype=F64, device=preds.device)
    grad = torch.zeros((b * k, hh, ww), dtype=F64, device=preds.device) if with_grad else None
    for i in range(0, b * k, step):
        ti = t[i : i + step].to(F64)
        pi = p[i : i + step].to(F64).requires_grad_(with_grad)
        v = (_plane_terms(ti, pi, kind) * keep[i : i + step]).sum() / denom
        if with_grad:
            (grad[i : i + step],) = torch.autograd.grad(v, pi)
        total = total + v.detach()
    return (total, grad.reshape(b, k, hh, ww)) if with_grad else total


def temporal_loss_ref(keypoints, confidences=None, epsilon=0.0, prob_threshold=0.0) -> torch.Tensor:
    """``O.temporal_loss`` (losses.py:608-703) on (T, 2K) keypoints, float64 on their device, differentiable."""
    kp = keypoints.to(F64)
    t = kp.shape[0]
    n = torch.linalg.norm(torch.diff(kp, dim=0).reshape(t - 1, -1, 2), ord=2, dim=2)
    if confidences is not None:
        low = confidences < prob_threshold
        n = n.masked_fill(low[:-1] | low[1:], 0.0)
    eps = torch.as_tensor(epsilon, dtype=F64, device=kp.device)
    return F.relu(n - eps).mean()


def pca_singleview_ref(keypoints, columns, centering, mean, kept, epsilon) -> torch.Tensor:
    """single-view PCA loss (losses.py:548-573, utils/pca.py:124-163, :266-309) in float64 (the oracle keeps dtype)."""
    kp = keypoints.to(F64)
    data = O.pca_format_singleview(kp, list(columns), centering)
    return O.pca_loss(data, mean.to(kp.device, F64), kept.to(kp.device, F64), float(epsilon))


def pca_multiview_ref(keypoints, mirrored_column_matches, mean, kept, epsilon) -> torch.Tensor:
    """multi-view PCA loss (losses.py:548-573, utils/pca.py:97-122) in float64 (the oracle keeps dtype)."""
    kp = keypoints.to(F64)
    data = O.pca_format_multiview(kp, [list(v) for v in mirrored_column_matches])
    return O.pca_loss(data, mean.to(kp.device, F64), kept.to(kp.device, F64), float(epsilon))


# ------------------------------------------------------------------------------------------------
# MHCRNN context head
# ------------------------------------------------------------------------------------------------
def crnn_ref(features: torch.Tensor, params: dict, upsampling_factor: int, softmax: bool = True) -> torch.Tensor:
    """``O.mhcrnn_multiframe`` (heads/heatmap_mhcrnn.py:268-316) in float64 on the features' device: (frames, batch,
    C, h, w) -> (batch, K, H, W); ``softmax=False`` returns the logits (x_f + x_b) / 2."""
    p = {key: tuple(t.to(device=features.device, dtype=F64) for t in tup) for key, tup in params.items()}
    x = features.to(F64)
    if softmax:
        return O.mhcrnn_multiframe(x, p, upsampling_factor)
    frames, batch = x.shape[:2]
    ct = lambda z, wb: F.conv_transpose2d(z, wb[0], wb[1], stride=2, padding=1, output_padding=1)
    y = F.pixel_shuffle(x.reshape(frames * batch, *x.shape[2:]), 2)
    if upsampling_factor == 2:
        y = ct(y, p["W_pre"])
    y = y.reshape(frames, batch, *y.shape[1:])
    wf = torch.stack([ct(y[t], p["W_f"]) for t in range(frames)]).flatten(0, 1)
    wb = torch.stack([ct(y[t], p["W_b"]) for t in range(frames)]).flatten(0, 1)
    idx = torch.arange(frames, device=x.device)[None, :] * batch + torch.arange(batch, device=x.device)[:, None]
    return crnn_combine_ref(wf, wb, idx, p["H_f"], p["H_b"])


def context_ref(feats: torch.Tensor, params: dict, upsampling_factor: int, idx: torch.Tensor, operands=torch.bfloat16,
                mids: list | None = None):
    """The context head as its kernels compute it, in float64: the W_f and W_b maps of every frame (N, C, h, w) by two
    ``head_ref`` logit heads, W_pre + W_f and W_pre + W_b (``upsampling_factor`` 2) or W_f and W_b alone, with the
    tensor-core kernels' operand roundings (``operands``; None: none); then ``crnn_combine_ref`` over the (M, 5) window
    table ``idx`` and the plane softmax.  Returns ``(heatmaps (M, K, H, W), wf, wb)``, the maps (N, K, H, W) with
    ``retain_grad`` where they need a gradient, so that their per-channel gradient norms can bound the W_f / W_b bias
    gradients.  ``mids``: as ``head_ref``'s (the W_pre outputs of the W_f run, then of the W_b run).  Differentiable in
    every input."""
    maps = []
    for key in ("W_f", "W_b"):
        layers = ([params["W_pre"]] if upsampling_factor == 2 else []) + [params[key]]
        m = head_ref(feats, [w for w, _ in layers], [b for _, b in layers], softmax=False, operands=operands, mids=mids)
        if m.requires_grad:
            m.retain_grad()
        maps.append(m)
    logits = crnn_combine_ref(maps[0], maps[1], idx, params["H_f"], params["H_b"])
    n, k, hh, ww = logits.shape
    return torch.softmax(logits.reshape(n, k, -1), -1).reshape(n, k, hh, ww), maps[0], maps[1]


def crnn_combine_ref(wf, wb, idx, h_f_params, h_b_params) -> torch.Tensor:
    """(x_f + x_b) / 2 of the bidirectional recurrence over the five context slots of every window, float64.

    ``wf`` / ``wb`` (N, K, H, W): W_f(x_t) / W_b(x_t) of N frames; ``idx`` (M, 5) frame of each slot; ``h_*_params`` =
    (conv w, conv b, convT w, convT b) of H_f / H_b (grouped, kernel = stride = 2; heads/heatmap_mhcrnn.py:268-316).
    Differentiable in the maps and parameters."""
    k = wf.shape[1]
    wf, wb = wf.to(F64), wb.to(F64)
    hf = [t.to(device=wf.device, dtype=F64) for t in h_f_params]
    hb = [t.to(device=wf.device, dtype=F64) for t in h_b_params]
    idx = idx.long().to(wf.device)

    def hidden(z, hp):
        z = F.conv2d(z, hp[0], hp[1], stride=2, groups=k)
        return F.conv_transpose2d(z, hp[2], hp[3], stride=2, groups=k)

    xf = wf[idx[:, 0]]
    for t in range(1, idx.shape[1]):
        xf = wf[idx[:, t]] + hidden(xf, hf)
    last = idx.shape[1] - 1
    xb = wb[idx[:, last]]
    for t in range(last - 1, -1, -1):
        xb = wb[idx[:, t]] + hidden(xb, hb)
    return (xf + xb) / 2
