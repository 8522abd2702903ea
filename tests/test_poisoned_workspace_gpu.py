"""GPU: every entry of ``ops.py`` gives the same bits whatever its new outputs and workspaces held before the call.

Each case runs one entry (or one entry's forward and backward) under ``poison_support.same_under_poison``: every
``torch.empty`` / ``torch.empty_like`` of the call filled with 0x00, then 0xFF (NaN in every float type, -1 in int32),
then 0x7F (3.39e38 fp32 / bf16, NaN fp16, 0x7F7F7F7F int32).  The inputs are made outside the poison.  Shapes are small,
plus one batch past one wave (2 S + 7 frames, S the SM count) for the head and the decode, and shapes whose last band or
chunk is short.

Audit, from the code, of what each entry reads from memory it allocates (the integer workspaces first: a stale -1 or
0x7F7F7F7F index would read out of bounds):

- 16-bit head forward (``_head_forward_16``, one / two / three deconvs): ``ws`` packed weights written by the prep
  launch; the row-layout pads of the staged features and of ``mid`` / ``mid2`` cleared by prep; k1a and the banded
  kernels read staged rows only where the tile group / band owns them; split-softmax statistics written per
  (frame, group, band) before the combine reads them.  ``band_max``: every slot written by its epilogue warp.  No
  integer workspace.
- bf16 head backward (``head_backward_bf16``, ``lpb_head3_bwd``): ``dw*`` / ``db*`` stored (not accumulated) by the
  fixed-order ``reduce_partials`` from per-CTA partials each CTA writes (a memset only for B = 0); b2d's short last chunk stages stale rows that feed only accumulator rows the epilogue skips
  (head_bwd_bf16.cu, b2d).  The decode overflow planes (``gov``) are read only where the window meta's flag is 2.  No
  integer workspace.
- ``decode_backward_windows``: ``queue`` counter cleared by memset; ``meta`` written for every plane; ``win`` read only
  where flag is 1; ``overflow`` written and read only where flag is 2 (the comment at ops.decode_backward_windows).
- ``decode_forward``: the queue and its counter ([2 n + 1] int32) cleared by memset before the warp kernel.
- fp32 route: ``convt_backward_f32``'s ``dw`` / ``db`` are stored by the fixed-order ``reduce_partials`` from the
  partials workspace, which every slot writes first (a memset only for B = 0).  ``plane_softmax_*`` and ``upsample2x`` write every output, read none.
- losses / targets: the per-plane ``ws`` [2 B K] of the heatmap losses written by the forward before its reduction and
  the backward read it; ``temporal_heatmap_loss`` ``ws`` likewise.
- ``crnn_combine`` backward: ``start`` / ``cnt`` / ``pairs`` (int32) written by ``crnn_pairs_kernel`` (cnt cleared in
  the kernel, start[0] set, each pair list placed then sorted) before ``crnn_dmaps_kernel`` reads them; the float
  partials written before ``reduce_partials``.  ``context_gather`` writes every output element.
- regression head: ``ws`` (B, C) written by the backward's column-sum kernel before the broadcast reads it.  Geometry
  (``triangulate_pairs``, ``project_points``, ``frame_to_model``, ``pairwise_projections_loss``), patch masks, ingest and
  the crop boxes (``bboxes_from_keypoints``, ``bboxes_rolling_median``) write every output element and have no
  workspace.  ``draw_dlc_params`` fills each of its six columns from the generator.
- predictors: the chunk graph's buffers are allocated before capture, some by ``torch.empty``; the run must give the
  same table whatever they held.

Every ``ops.py`` entry that allocates with ``torch.empty`` has a case below.  The ``register_fake`` functions allocate
fake tensors for tracing, with no device memory.  ``pack_predictions`` and the context packers allocate nothing (they
write into the caller's table); the predictor cases run them."""
import math

import pytest
import torch

from head_support import features, gen, head_params, make_head, softmax_split
from poison_support import same_under_poison

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CL = torch.channels_last


@pytest.fixture(scope="module")
def ops():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops as o

    return o


@pytest.fixture(scope="module")
def lib(ops):
    from lightning_pose_b200._lib import lib as l

    return l


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


# ------------------------------------------------------------------------------------------------
# the 16-bit head
# ------------------------------------------------------------------------------------------------
# name -> (B or "wave", C, H, W, deconv channels): a k1a row (bands of 7 and 6), banded two- and one-deconv rows with
# short last bands, a wide row (keypoint groups), three deconvs, and config 2 past one wave
FWD_ROWS = {
    "k1a_13x8": (3, 128, 13, 8, (17, 17)),
    "2d_8x5": (3, 128, 8, 5, (17, 17)),
    "1d_9x8": (3, 128, 9, 8, (20,)),
    "wide_k40": (3, 512, 8, 8, (40, 40)),
    "three_8_8_17": (3, 512, 8, 8, (8, 8, 17)),
    "cfg2_wave": ("wave", 2048, 12, 12, (17, 17)),
}
FWD_CASES = [(r, torch.bfloat16, False) for r in FWD_ROWS] + [("k1a_13x8", torch.float16, False), ("1d_9x8", torch.float16, False),
                                                              ("2d_8x5", torch.bfloat16, True), ("1d_9x8", torch.float16, True),
                                                              ("three_8_8_17", torch.bfloat16, True)]


def _batch(b, sms):
    return 2 * sms + 7 if b == "wave" else b


def _head16(ops, lib, f, ws, bs, split, ds):
    """heatmaps with band maxima, the plain heatmaps, the logits, the training form's heatmaps (bf16), and the decode of
    the heatmaps with and without the band maxima"""
    layout = ops.feature_layout(f)
    with softmax_split(lib, split):
        hm, hints = ops._head_forward_16(f, ws, bs, True, want_hints=True, layout=layout)
        plain = ops._head_forward_16(f, ws, bs, True, layout=layout)
        logits = ops._head_forward_16(f, ws, bs, False, layout=layout)
        train = ops._head_forward_16(f, ws, bs, True, train=True, layout=layout)[0] if f.dtype == torch.bfloat16 else plain
    full = ops.decode_forward(hm, ds, 1000.0)
    banded = ops.decode_forward(hm, ds, 1000.0, band_max=hints)
    return hm, hints.bits, plain, logits, train, full, banded


@pytest.mark.parametrize("split", [0, 2])
@pytest.mark.parametrize("row,dtype,nhwc", FWD_CASES)
def test_head_forward_16(ops, lib, sms, row, dtype, nhwc, split):
    b, c, h, w, ch = FWD_ROWS[row]
    b = _batch(b, sms)
    head = make_head(c, ch, seed=5)
    ws, bs = head_params(head)
    f = features(b, c, h, w, seed=6, dtype=dtype)
    if nhwc:
        f = f.contiguous(memory_format=CL)
    assert ops.head_16_operand(f, list(ch), train=False)[1] == (ops.FEATURES_NHWC if nhwc else ops.FEATURES_NCHW)
    same_under_poison(_head16, ops, lib, f, ws, bs, split, head.downsample_factor, case=f"{row} {dtype} nhwc={nhwc} split={split}")


# name -> (B or "wave", C, H, W, deconv channels, channels-last)
BWD_ROWS = {
    "cfg2": (3, 2048, 12, 12, (17, 17), False),
    "cfg2_nhwc": (3, 2048, 12, 12, (17, 17), True),
    "vit_1d": (3, 384, 16, 16, (17,), False),
    "wide_k40": (3, 512, 8, 8, (40, 40), False),
    "three_8_8_17": (3, 512, 8, 8, (8, 8, 17), False),
    "cfg2_wave": ("wave", 2048, 12, 12, (17, 17), False),
}
GRAD_KINDS = ["dense", "windows", "windows+dense", "mse", "dense_logits"]


def _head_bwd(ops, head, f, kind, need_dfeat, gout, gkp, kp):
    head.zero_grad(set_to_none=True)
    head.final_softmax = kind != "dense_logits"
    x = f.detach().clone().requires_grad_(need_dfeat)
    if kind in ("dense", "dense_logits"):
        (head(x) * gout).sum().backward()
    elif kind == "mse":
        hm = head(x)
        img = (hm.shape[2] * 2 ** head.downsample_factor, hm.shape[3] * 2 ** head.downsample_factor)
        ops.heatmap_mse_from_keypoints(kp * torch.tensor(img[::-1], device=DEV), hm, img[0], img[1]).backward()
    else:
        hm, xy, _ = head.forward_with_keypoints(x)
        loss = (xy * gkp).sum()
        if kind == "windows+dense":
            loss = loss + (hm * gout).sum()
        loss.backward()
    head.final_softmax = True
    out = [x.grad] if need_dfeat else []
    return out + [p.grad for p in head.parameters() if p.grad is not None]


@pytest.mark.parametrize("kind", GRAD_KINDS)
@pytest.mark.parametrize("row", list(BWD_ROWS))
def test_head_backward_bf16(ops, sms, row, kind):
    b, c, h, w, ch, nhwc = BWD_ROWS[row]
    b = _batch(b, sms)
    head = make_head(c, ch, seed=9)
    f = features(b, c, h, w, seed=10, dtype=torch.bfloat16)
    if nhwc:
        f = f.contiguous(memory_format=CL)
    up = {1: 4, 2: 8, 3: 16}[len(ch)]
    gout = torch.randn(b, ch[-1], up * h, up * w, device=DEV, generator=gen(11))
    gkp = torch.randn(b, 2 * ch[-1], device=DEV, generator=gen(12))
    kp = torch.rand(b, ch[-1], 2, device=DEV, generator=gen(13))
    for need_dfeat in (True, False):
        same_under_poison(_head_bwd, ops, head, f, kind, need_dfeat, gout, gkp, kp, case=f"{row} {kind} dfeat={need_dfeat}")


# ------------------------------------------------------------------------------------------------
# the fp32 route and the decode
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nhwc", [False, True])
def test_fp32_route(ops, nhwc):
    b, c, h, w = 3, 256, 5, 7
    f = torch.randn(b, c, h, w, device=DEV, generator=gen(1)) * 0.5
    if nhwc:
        f = f.contiguous(memory_format=CL)
    head = make_head(c, (17, 17), seed=2)
    ws, bs = head_params(head)
    g = torch.randn(b, 17, 8 * h, 8 * w, device=DEV, generator=gen(3))

    def run():
        out, acts = ops.head_forward_f32(f, ws, bs, final_softmax=False, keep_activations=True)
        probs = out.clone()
        ops.plane_softmax_(probs)
        gl = ops.plane_softmax_backward(probs, g)
        g2 = ops.convt_backward_f32(acts[1], gl, ws[1], shuffle=False)
        g1 = ops.convt_backward_f32(acts[0], g2[0], ws[0], shuffle=True)
        g1b = ops.convt_backward_f32(acts[0], g2[0], ws[0], shuffle=True, need_dx=False, need_db=False)
        one = ops.convt_forward_f32(f, ws[0], None, shuffle=True)
        return out, probs, gl, g2, g1, g1b, one, ops.head_forward_f32(f, ws, bs), ops.upsample2x(probs[:, :, :11, :13])

    same_under_poison(run, case=f"fp32 nhwc={nhwc}")


def _decode_planes(n, h, w, seed):
    """peaked planes, diffuse planes (queued by the warp kernel), and a few NaN planes"""
    g = gen(seed)
    logits = torch.randn(n, 17, h, w, device=DEV, generator=g)
    logits[:, ::3] *= 0.1
    logits[:, 1::3] *= 30.0
    hm = torch.softmax(logits.flatten(2), -1).reshape(logits.shape)
    hm[0, 5] = float("nan")
    hm[-1, 16] = float("nan")
    return hm


@pytest.mark.parametrize("hw,ds", [((24, 24), 2), ((48, 40), 2), ((64, 64), 1), ((32, 32), 3)])
def test_decode(ops, sms, hw, ds):
    n = 2 * sms + 7 if hw in ((24, 24), (48, 40)) else 5
    hm = _decode_planes(n, *hw, seed=hw[0] + ds)
    gxy = torch.randn(n, 17, 2, device=DEV, generator=gen(4))

    def run():
        xy, conf, stats = ops.decode_forward(hm, ds, 1000.0)
        dense = ops._decode_bwd(hm, stats, gxy, ds, 1000.0)
        win, meta, ov = ops.decode_backward_windows(hm, stats, gxy, ds, 1000.0)
        flag = meta[:, 2]
        return xy, conf, stats, dense, meta, win[flag == 1], ov.reshape(-1, *hw)[flag == 2]

    flag = same_under_poison(run, case=f"decode {hw} ds={ds}")[4][:, 2]
    assert bool((flag == 1).any()), "no plane took a gradient window"
    if max(hw) > 32:  # a diffuse plane's gradient does not fit a 32 x 32 window: it takes the overflow buffer
        assert bool((flag == 2).any()), "no plane took the overflow buffer"


# ------------------------------------------------------------------------------------------------
# targets and losses
# ------------------------------------------------------------------------------------------------
def test_targets_and_heatmap_losses(ops):
    b, k, oh, ow = 5, 7, 24, 20
    kp = torch.rand(b, k, 2, device=DEV, generator=gen(5)) * torch.tensor([80.0, 96.0], device=DEV)
    kp[0, 1] = float("nan")
    vis = (torch.rand(b, k, device=DEV, generator=gen(6)) > 0.2).to(torch.int32)
    logits = torch.randn(b, k, oh, ow, device=DEV, generator=gen(7)) * 3
    preds = torch.softmax(logits.flatten(2), -1).reshape(logits.shape)

    def run():
        out = []
        x = kp.clone().requires_grad_(True)
        t = ops.generate_heatmaps(x, 96, 80, (oh, ow), keep_gradients=True)
        (t * logits).sum().backward()
        out += [t, x.grad, ops.generate_heatmaps(kp, 96, 80, (oh, ow), visibility=vis)]
        for kind in ("mse", "kl", "js"):
            p = preds.clone().requires_grad_(True)
            loss, cnt = ops.heatmap_loss(t.detach(), p, kind, return_count=True)
            loss.backward()
            out += [loss, cnt, p.grad]
            for count in (False, True):
                p = preds.clone().requires_grad_(True)
                res = ops.heatmap_loss_from_keypoints(kind, kp, p, 96, 80, visibility=vis, return_count=count)
                (res[0] if count else res).backward()
                out += [res, p.grad.clone() if not isinstance(p.grad, ops.MseKeypointGrad) else p.grad.materialize()]
        for kind in ("mse", "kl"):
            p = preds.clone().requires_grad_(True)
            cf = torch.rand(b, k, device=DEV, generator=gen(8))
            loss = ops.temporal_heatmap_loss(p, cf, kind, torch.tensor([0.01], device=DEV), 0.3)
            loss.backward()
            out += [loss, p.grad]
        out += [ops.keypoints_mask_oob(kp, 96, 80), ops.evaluate_heatmaps_at_location(preds, kp[..., :] / 4)]
        return out

    same_under_poison(run, case="targets and losses")


def test_unsup_losses_and_remap(ops):
    from lightning_pose_b200.ops import PcaParams

    n, t, k = 3, 9, 6
    kp = torch.randn(n, t, 2 * k, device=DEV, generator=gen(9)) * 20 + 50
    cf = torch.rand(n, t, k, device=DEV, generator=gen(10))
    d = 2 * 4
    kept = torch.linalg.qr(torch.randn(d, d, generator=torch.Generator().manual_seed(0)))[0][:3]
    sv = PcaParams([0, 1, 2, 3], 4, 0, "mean", torch.randn(d) * 10 + 50, kept, 1.0, DEV)
    tf = torch.randn(n * t, 2, 3, device=DEV, generator=gen(11)) * 0.1 + torch.tensor([[1.0, 0, 0], [0, 1.0, 0]], device=DEV)
    bb = torch.rand(n * t, 4, device=DEV, generator=gen(12)) * 100 + 10

    def run():
        x = kp.clone().requires_grad_(True)
        losses = ops.unsup_losses(x, cf, temporal_eps=2.0, prob_threshold=0.1, pca_singleview=sv)
        losses.sum().backward()
        y = kp.reshape(n * t, 2 * k).clone().requires_grad_(True)
        r = ops.remap_keypoints(y, tf, bb, 64, 64)
        (r * r).sum().backward()
        return losses, x.grad, r, y.grad

    same_under_poison(run, case="unsup losses and remap")


# ------------------------------------------------------------------------------------------------
# context, regression, geometry, patch masks
# ------------------------------------------------------------------------------------------------
def _crnn_inputs(n, m, k=5, h=4, w=6, hidden=8, seed=13):
    g = gen(seed)
    wf = torch.randn(n, k, h, w, device=DEV, generator=g)
    wb = torch.randn(n, k, h, w, device=DEV, generator=g)
    idx = torch.randint(0, n, (m, 5), device=DEV, generator=g, dtype=torch.int32)

    def params():
        return [torch.randn(k * hidden, 1, 2, 2, device=DEV, generator=g) * 0.3, torch.randn(k * hidden, device=DEV, generator=g) * 0.1,
                torch.randn(k * hidden, 1, 2, 2, device=DEV, generator=g) * 0.3, torch.randn(k, device=DEV, generator=g) * 0.1]

    return wf, wb, idx, params(), params()


def _crnn(ops, wf, wb, idx, hf, hb, gout):
    leaves = [t.clone().requires_grad_(True) for t in [wf, wb, *hf, *hb]]
    out = ops.crnn_combine(leaves[0], leaves[1], idx, leaves[2:6], leaves[6:10])
    (out * gout).sum().backward()
    return [out] + [x.grad for x in leaves]


def test_context(ops):
    n, m = 40, 37
    wf, wb, idx, hf, hb = _crnn_inputs(n, m)
    gout = torch.randn(m, *wf.shape[1:], device=DEV, generator=gen(14))
    seq = {dt: torch.randn(9, 3, 8, 8, device=DEV, generator=gen(15)).to(dt) for dt in (torch.float32, torch.bfloat16, torch.float16)}

    def run():
        out = _crnn(ops, wf, wb, idx, hf, hb, gout)
        for x in seq.values():
            x = x.clone().requires_grad_(True)
            y = ops.context_gather(x, 5)
            (y.float() * torch.arange(y.numel(), device=DEV).reshape(y.shape).float().sin()).sum().backward()
            out += [y, x.grad]
        return out

    same_under_poison(run, case="context")


def _cameras(b, v):
    kmat = torch.tensor([[500.0, 0, 64], [0, 480.0, 60], [0, 0, 1]], device=DEV).expand(b, v, 3, 3).clone()
    e = torch.zeros(b, v, 3, 4, device=DEV)
    for i in range(v):
        a = 0.3 * i
        e[:, i, :3, :3] = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], device=DEV)
        e[:, i, :, 3] = torch.tensor([0.1 * i, 0.0, 5.0], device=DEV)
    d = torch.zeros(b, v, 5, device=DEV)
    d[..., 0] = 0.05
    return kmat, e, d


def test_regression_geometry_patches(ops):
    f32 = torch.randn(4, 64, 5, 7, device=DEV, generator=gen(16))
    weight = torch.randn(12, 64, device=DEV, generator=gen(17)) * 0.1
    bias = torch.randn(12, device=DEV, generator=gen(18))
    targ = torch.randn(4, 12, device=DEV, generator=gen(19))
    targ[1, 3] = float("nan")
    b, v, k = 3, 3, 6
    kmat, e, d = _cameras(b, v)
    pts = torch.rand(b, v, k, 2, device=DEV, generator=gen(20)) * 100 + 10
    p3t = torch.randn(b, k, 3, device=DEV, generator=gen(21))
    bb = torch.tensor([5.0, 6.0, 120.0, 110.0], device=DEV).repeat(b, v)
    images = torch.randn(2, 3, 3, 40, 36, device=DEV, generator=gen(22))
    step = torch.tensor([5], device=DEV, dtype=torch.int64)

    def run():
        out = []
        for dt, fmt in ((torch.float32, None), (torch.bfloat16, None), (torch.float16, CL)):
            x = f32.to(dt, copy=True)
            x = (x.contiguous(memory_format=fmt) if fmt else x).requires_grad_(True)
            wt, bs = weight.clone().requires_grad_(True), bias.clone().requires_grad_(True)
            y = ops.regression_head(x, wt, bs)
            (y * y).sum().backward()
            out += [y, x.grad, wt.grad, bs.grad]
        p = torch.randn(4, 12, device=DEV, generator=gen(23)).requires_grad_(True)
        res = ops.regression_losses(targ, p)
        res[0].backward()
        out += [*res, p.grad]
        x = pts.clone().requires_grad_(True)
        tri = ops.triangulate_pairs(x, kmat, e, d)
        q = tri.detach().clone().requires_grad_(True)
        proj = ops.project_points(q, kmat, e, d, mean_over_pairs=True, bbox=bb, model_size=(64, 64))
        (proj.sum() + tri.sum()).backward()
        y = tri.detach().clone().requires_grad_(True)
        loss = ops.pairwise_projections_loss(p3t, y)
        loss.backward()
        out += [tri, x.grad, proj, q.grad, loss, y.grad]
        x = pts.clone().requires_grad_(True)
        fm = ops.frame_to_model(x, bb, 64, 80)
        (fm * fm).sum().backward()
        out += [fm, x.grad]
        mask = ops.patch_mask_select(images, step, 7, 0, 10, 0.1, 0.5)
        out += [mask, ops.patch_mask_apply(images, mask), ops.patch_mask_apply(images.bfloat16(), mask)]
        return out

    same_under_poison(run, case="regression, geometry, patches")


# ------------------------------------------------------------------------------------------------
# ingest
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [False, True])
def test_ingest(ops, dtype, channels_last):
    g = gen(24)
    frames = torch.randint(0, 256, (5, 37, 51, 3), device=DEV, dtype=torch.uint8, generator=g)
    other = torch.randint(0, 256, (5, 29, 33, 3), device=DEV, dtype=torch.uint8, generator=g)
    boxes = torch.tensor([[3.0, 4.0, 20.0, 30.0], [0.0, 0.0, 37.0, 51.0], [10.0, 12.0, 9.0, 7.0]], device=DEV)
    box = torch.tensor([2, 3, 30, 25], device=DEV, dtype=torch.int32)
    params = torch.tensor([4.0, 1.1, 0.9, 1.1, 0.9, 3.0], device=DEV)
    seed = torch.tensor([1234567], device=DEV, dtype=torch.int64)
    kw = dict(channels_last=channels_last, dtype=dtype)

    def run():
        out = [ops.frames_normalize(frames, (24, 40), **kw), ops.frames_normalize(frames, None, **kw),
               ops.frames_normalize_views([frames, other], (24, 40), **kw),
               *ops.frames_crop_normalize(frames, boxes, (24, 40), row0=1, **kw),
               *ops.frames_crop_resize_cv2(frames, (24, 40), box=box, **kw), *ops.frames_crop_resize_cv2(frames, (24, 40), **kw)]
        if dtype != torch.float16:
            out += list(ops.frames_augment_normalize(frames, (24, 40), params, seed, **kw))
        return out

    same_under_poison(run, case=f"ingest {dtype} cl={channels_last}")


# ------------------------------------------------------------------------------------------------
# predictors
# ------------------------------------------------------------------------------------------------
def _predict(head, k, feats, chunk, use_graph):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    n = feats.shape[0]
    bp = BatchedPredictor(head, k, n, chunk, (128, 128), use_graph=use_graph)
    pad = (-n) % chunk
    f = torch.cat([feats, feats[-1:].expand(pad, *feats.shape[1:])])
    bp.run(f[i : i + chunk] for i in range(0, n + pad, chunk))
    return bp.table


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("kind", ["plain", "context", "three"])
def test_batched_predictor(ops, kind, use_graph):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    k, c, n, chunk = 17, 512, 21, 8
    if kind == "context":
        torch.manual_seed(3)
        head = HeatmapMHCRNNHead("resnet50", c, k).to(DEV).eval()
    else:
        head = make_head(c, (17, 17) if kind == "plain" else (8, 8, 17), seed=4).eval()
    feats = features(n, c, 4, 4, seed=25, dtype=torch.bfloat16)
    with torch.no_grad():
        same_under_poison(_predict, head, k, feats, chunk, use_graph, case=f"predictor {kind} graph={use_graph}")


def test_frame_predictor(ops):
    import torch.nn.functional as F

    from lightning_pose_b200.utils.predictions import FramePredictor

    c = 512
    head = make_head(c, (17, 17), seed=6).eval()
    proj = torch.randn(c, 3, device=DEV, generator=gen(26))
    features_of = lambda x: torch.einsum("ca,bahw->bchw", proj, F.avg_pool2d(x, 32)).to(torch.bfloat16)  # noqa: E731
    frame = torch.randint(0, 256, (150, 170, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).numpy()

    def run():
        fp = FramePredictor(head, 17, (128, 128), features_of=features_of)
        outs = [fp.predict_frame(frame), fp.predict_frame(frame, bbox=(10, 12, 100, 90))]
        return [torch.from_numpy(v.copy()) for o in outs for _, v in sorted(o.items())]

    with torch.no_grad():
        same_under_poison(run, case="frame predictor")


def test_boxes_and_draws(ops):
    """The crop boxes of crop-zoom prediction and the DALI augmentation draw: every output element written."""
    kp = torch.rand(11, 6, 2, device=DEV, generator=gen(27)) * 200
    kp[3, 1] = float("nan")
    table = torch.rand(11, 18, device=DEV, generator=gen(28)) * 200
    boxes = torch.rand(11, 4, device=DEV, generator=gen(29)) * 100 + 20

    def run():
        g = torch.Generator(device=DEV).manual_seed(30)
        return [ops.bboxes_from_keypoints(kp, crop_ratio=1.5), ops.bboxes_from_keypoints(kp, (0, 2, 5), crop_height=64, crop_width=48),
                ops.bboxes_from_keypoints(table, (1, 4), crop_ratio=2.0), ops.bboxes_rolling_median(boxes),
                ops.bboxes_rolling_median(boxes, window=3), *ops.draw_dlc_params(3, DEV, generator=g)]

    same_under_poison(run, case="boxes and draws")
