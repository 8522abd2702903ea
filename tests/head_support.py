"""Shared pieces of the heatmap head's tests.  TEST INFRASTRUCTURE ONLY.

One of each: the random test head, its features and gradients, the softmax-split switch, the restated forward workspace
layout, and the acceptance rules against the float64 references of ``scale_oracle.py``.  Every rule is applied per
keypoint plane / output channel / frame and reports its ratios (error / allowed) to ``_judge``, so that one wrong small
channel cannot hide behind a large one; ``test_head_shapes_gpu.py::test_comparisons_reject_plausible_kernel_bugs`` shows
on the CPU that each rule rejects plausible kernel bugs.  The operand dtype of the features (bf16, fp16) sets the bars."""
import collections
import contextlib

import torch

import scale_oracle as S

F64 = torch.float64
HEAD_CLS = 20  # output channels of one keypoint group (head_prep.cuh)
STAGE_BYTES = 4 * 4 * 80 * 16  # packed weights of one 32-channel K stage (head_prep.cuh)
SOFTMAX_SPLIT = 7  # tuning key of the plane softmax's form: 0 never split, 1 split below one wave (default), 2 always


def _lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


# ------------------------------------------------------------------------------------------------
# the test head, its inputs and gradients
# ------------------------------------------------------------------------------------------------
def make_head(c, channels, seed, gain=3.0, final_softmax=True):
    """A HeatmapHead on the device with deconv output channels ``channels``: one deconv is a ViT head, two or three a
    ResNet-50 head (downsample factor 2 or 1).  Xavier-uniform weights at ``gain``, biases uniform in [-0.3, 0.3]."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    n = len(channels)
    if n == 1:
        head = HeatmapHead("vits_dino", c, channels[0], final_softmax=final_softmax)
    else:
        head = HeatmapHead("resnet50", c, channels[-1], deconv_out_channels=channels[0], downsample_factor=4 - n,
                           final_softmax=final_softmax)
    deconvs = list(head.upsampling_layers)[1:]
    assert [d.weight.shape[1] for d in deconvs] == list(channels)
    for layer in deconvs:
        torch.nn.init.xavier_uniform_(layer.weight, gain=gain)
        torch.nn.init.uniform_(layer.bias, -0.3, 0.3)
    return head.cuda()


def head_params(head):
    """(weights, biases) of the head's deconvs, detached."""
    deconvs = list(head.upsampling_layers)[1:]
    return [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def features(b, c, h, w, seed, dtype, scale=0.5):
    return (torch.randn(b, c, h, w, device="cuda", generator=gen(seed)) * scale).to(dtype)


def grads(head, feats, gout, feature_grad=True):
    """{"dfeat", "dw1", "db1", ...} of sum(head(feats) * gout); without ``feature_grad`` the features are a frozen
    backbone's and no "dfeat" is returned."""
    head.zero_grad(set_to_none=True)
    f = feats.clone().requires_grad_(feature_grad)
    (head(f) * gout).sum().backward()
    out = {"dfeat": f.grad.clone()} if feature_grad else {}
    for i, d in enumerate(list(head.upsampling_layers)[1:], 1):
        out[f"dw{i}"], out[f"db{i}"] = d.weight.grad.clone(), d.bias.grad.clone()
    return out


@contextlib.contextmanager
def softmax_split(lib, value):
    """Pin the plane softmax's form (0: the fused per-frame kernel, with which a frame computes the same bits at any
    batch; 1: split over (frame, band) below one wave, the default; 2: always split), restoring the setting after."""
    saved = lib.lpb_get_tuning(SOFTMAX_SPLIT)
    try:
        assert lib.lpb_set_tuning(SOFTMAX_SPLIT, value) == 0
        yield
    finally:
        lib.lpb_set_tuning(SOFTMAX_SPLIT, saved)


# ------------------------------------------------------------------------------------------------
# the forward workspace, restated
# ------------------------------------------------------------------------------------------------
FwdLayout = collections.namedtuple("FwdLayout", "w2_at mid_at nst2 mid_rows total")


def row_layout(hi, wi):
    """(pitch, lead rows, rows) of the padded row layout of an hi x wi map: every image row followed by a zero column,
    lead rows of zeros before and after the image, the row count rounded up to 8."""
    pp = wi + 1
    lead = pp + 1
    return pp, lead, (hi * pp + 2 * lead + 7) & ~7


def fwd_layout(b, c, h, w, c1, c2):
    """head_fwd_layout (head_rows.cuh): the packed w1 at byte 0, the packed w2 (per keypoint group and K stage), the mid
    activations' 4 * nst2 K-chunks in the row layout of the 4H x 4W map (two-deconv heads), the split-softmax statistics
    per (frame, group, band), and the total workspace bytes."""
    groups = lambda k: -(-k // HEAD_CLS)  # noqa: E731

    def bands(hi, wi):
        r = max(1, min(256 // (wi + 1), hi))
        return -(-hi // r)

    nst2 = -(-max(c1 + 1, HEAD_CLS * groups(c1)) // 32) if c2 else 1
    g1, g2 = groups(c1), (groups(c2) if c2 else 1)
    w2_at = g1 * (c // 128) * STAGE_BYTES
    mid_at = w2_at + g2 * nst2 * STAGE_BYTES
    mid_rows = row_layout(4 * h, 4 * w)[2]
    part_at = mid_at + (b * 4 * nst2 * mid_rows * 16 if c2 else 0)
    part = b * (g2 * bands(4 * h, 4 * w) if c2 else g1 * bands(2 * h, 2 * w)) * HEAD_CLS * 2 * 4
    return FwdLayout(w2_at, mid_at, nst2, mid_rows, part_at + ((part + 255) & ~255))


# ------------------------------------------------------------------------------------------------
# acceptance rules
# ------------------------------------------------------------------------------------------------
WORST: dict = {}  # quantity -> (largest ratio seen, case); printed by each module's headroom fixture

# operand dtype -> (name prefix, heatmaps: largest relative error, and the relative error at most 0.01 % of the pixels may
# exceed; logits: relative bar).  fp16 has 1/8 of bf16's unit roundoff (2^-11 against 2^-8); its bars are bf16's scaled
# by that and rounded up.
BARS = {torch.bfloat16: ("", 3e-2, 1e-2, 1e-2), torch.float16: ("fp16 ", 5e-3, 2e-3, 2e-3)}


def _judge(case, ratios: dict):
    bad = []
    for name, r in ratios.items():
        r = r.detach().to(F64).flatten()
        worst = float(r.max()) if r.numel() else 0.0
        if worst > WORST.get(name, (-1.0, None))[0]:
            WORST[name] = (worst, case)
        if not worst < 1.0:
            bad.append((name, worst, int(r.argmax())))
    assert not bad, f"{case}: (quantity, error / allowed, index) {bad}"


def report_headroom():
    """With ``pytest -s``: the largest error / allowed ratio seen per quantity (how much headroom each rule has)."""
    for name, (ratio, case) in sorted(WORST.items()):
        print(f"headroom {name:44s} {ratio:9.4f}  ({case})")
    WORST.clear()


def check_heatmaps(out, ref, case="", key="heatmaps", dtype=torch.bfloat16):
    """Relative error below the dtype's largest bar (bf16 3e-2) on every pixel, above the lower bar (bf16 1e-2) on under
    0.01 % of the pixels, and every keypoint plane sums to 1 within 1e-5.  The 0.01 % holds over the batch and, per
    plane, with 9 pixels to spare: a mid activation on a rounding boundary that rounds the other way (fp32 summation
    order) moves the 3 x 3 output pixels it feeds, and a plane of fewer than 10^4 pixels would otherwise allow none."""
    prefix, top, over_bar, _ = BARS[dtype]
    key = prefix + key
    out, ref = out.detach().to(F64), ref.to(F64)
    rel = (out - ref).abs() / (ref.abs() + 1e-7)
    over = (rel > over_bar).to(F64)
    _judge(case, {f"{key}: relative error": rel.amax((-1, -2)) / top,
                  f"{key}: pixels over {over_bar:g}": over.mean() / 1e-4,
                  f"{key}: pixels over {over_bar:g} per plane": over.sum((-1, -2)) / (1e-4 * rel[0, 0].numel() + 9),
                  f"{key}: plane sum": (out.sum((-1, -2)) - 1).abs() / 1e-5})


def check_logits(out, ref, case="", dtype=torch.bfloat16):
    """Logits head: within the dtype's bar (bf16 1e-2) of the plane's largest magnitude plus the bar relative, per
    (frame, keypoint) plane."""
    prefix, _, _, bar = BARS[dtype]
    out, ref = out.detach().to(F64), ref.to(F64)
    allowed = bar * ref.abs().amax((-1, -2), keepdim=True) + bar * ref.abs() + 1e-12
    _judge(case, {f"{prefix}logits": ((out - ref).abs() / allowed).amax((-1, -2))})


def check_keypoints(hm, hm_ref, ds, case, bar):
    """The heatmaps and the reference's, each decoded in float64: within ``bar`` px on the planes the reference is
    confident in (confidence above 0.5)."""
    kp, _, _, _ = S.decode_ref(hm, ds)
    kp_ref, cf_ref, _, _ = S.decode_ref(hm_ref, ds)
    d = (kp - kp_ref).abs().reshape(cf_ref.shape + (2,)).amax(-1)
    _judge(case, {f"keypoints within {bar:g} px": d[cf_ref > 0.5] / bar})


def logit_grad(gout, probs=None):
    """d loss / d logits for a dense output gradient: the spatial softmax's backward when ``probs`` is given."""
    g = gout.to(F64)
    if probs is None:
        return g
    p = probs.to(F64)
    return p * (g - (p * g).sum((-1, -2), keepdim=True))


def check_grads(got: dict, ref: dict, gnorm: dict, case="", rel=1e-2, global_scale=(), db_max_rule=None):
    """bf16 backward against float64, per channel.

    ``dfeat``: per frame, ``rel`` times the frame's largest gradient.  ``dw{i}`` [Cin, Cout, 3, 3] (layers counted from 1):
    per output channel, ``rel`` times that channel's largest weight gradient.  ``db{i}``: a bias gradient is its channel's
    output gradient summed over every pixel of every frame.  Behind a softmax that sum cancels exactly, and with a dense
    random gradient it is a sum of random signs, so the channel's own value is no scale for the error.  What sets the
    error is the bf16 rounding of the gradient operand the kernels sum, at most 2^-9 of each element, whose sum over the
    channel is bounded by 4 x 2^-8 of the channel's gradient L2 norm ``gnorm[f"db{i}"][o]``; plus ``rel`` of the
    channel's value, as for the other quantities.
    Quantities named in ``global_scale`` are held to ``rel`` times their largest entry instead, where the caller says why
    no per-channel bound is meaningful.  ``db_max_rule`` (the head's final_softmax) also holds each bias gradient to
    ``rel`` of its largest entry, the last layer's behind a softmax (exactly 0) to ``rel`` of the last weight gradient's
    largest entry: the global rule of the bf16 head's first backward tests, which the per-channel one does not imply."""
    ratios = {}
    last = sum(k.startswith("dw") for k in ref)
    for name, r in ref.items():
        g, r = got[name].detach().to(F64), r.to(F64)
        err = (g - r).abs()
        if name in global_scale:
            ratios[f"{name} (largest entry's scale)"] = err.max() / (rel * r.abs().max() + 1e-9)
        elif name == "dfeat":
            ratios[name] = err.flatten(1).amax(1) / (rel * r.abs().flatten(1).amax(1) + 1e-9)
        elif name.startswith("dw"):
            ratios[name] = err.transpose(0, 1).flatten(1).amax(1) / (rel * r.abs().transpose(0, 1).flatten(1).amax(1) + 1e-9)
        else:
            ratios[name] = err / (rel * r.abs() + 4.0 * 2.0**-8 * gnorm[name].to(F64) + 1e-9)
            if db_max_rule is not None:
                scale = ref[f"dw{last}"] if db_max_rule and name == f"db{last}" else r
                ratios[f"{name} (largest entry's scale)"] = err.max() / (rel * scale.to(F64).abs().max() + 1e-9)
    _judge(case, ratios)


def check_grads_f32(got: dict, ref: dict, gnorm: dict, case=""):
    """fp32 backward against float64: dfeat comes back rounded to the features' bf16 (2^-8 relative, 1e-4 of the
    frame's largest gradient for the fp32 sums under it), the weight gradients within 1e-3 relative of each channel's
    scale, the bias gradients within 2^-14 of the channel's gradient L2 norm (a thirtieth of what a bf16 gradient
    operand would leave)."""
    ratios = {}
    for name, r in ref.items():
        g, r = got[name].detach().to(F64), r.to(F64)
        err = (g - r).abs()
        if name == "dfeat":
            ratios[name] = (err / (2.0**-8 * r.abs() + 1e-4 * r.abs().flatten(1).amax(1).view(-1, 1, 1, 1) + 1e-12)).flatten(1).amax(1)
        elif name.startswith("dw"):
            ratios[name] = err.transpose(0, 1).flatten(1).amax(1) / (1e-3 * r.abs().transpose(0, 1).flatten(1).amax(1) + 1e-12)
        else:
            ratios[name] = err / (1e-3 * r.abs() + 2.0**-14 * gnorm[name].to(F64) + 1e-12)
    _judge(case, {f"fp32 {k}": v for k, v in ratios.items()})


def _operands(feats):
    return feats.dtype if feats.dtype in BARS else None


def ref_forward(head, feats):
    """float64 (logits, heatmaps) of the head on the features' operand roundings."""
    ws, bs = head_params(head)
    logits = S.head_ref_chunked(feats, ws, bs, softmax=False, operands=_operands(feats))
    return logits, torch.softmax(logits.flatten(2), -1).reshape(logits.shape)


def ref_grads(feats, ws, bs, gout, softmax, probs, operands=torch.bfloat16):
    """float64 gradients {"dfeat", "dw1", "db1", ...} and the per-channel L2 norms of the gradient each bias sums: the
    logits' for the last layer, the mid activations' for the first of two."""
    n = len(ws)
    res = S.head_grad_ref(feats, ws, bs, gout, softmax=softmax, operands=operands, want_mid_grad=n == 2)
    dfeat, dws, dbs = res[:3]
    ref = {"dfeat": dfeat, **{f"dw{i}": g for i, g in enumerate(dws, 1)}, **{f"db{i}": g for i, g in enumerate(dbs, 1)}}
    gnorm = {f"db{n}": logit_grad(gout, probs if softmax else None).pow(2).sum((0, 2, 3)).sqrt()}
    if n == 2:
        gnorm["db1"] = res[3]
    return ref, gnorm


def forward_checks(head, feats, case, splits=(None,), train=True, keypoint_bar=None):
    """Heatmaps under each softmax form in ``splits`` (None: the library's choice) and logits against float64 on the
    features' operand roundings; with ``train``, the training form's heatmaps equal the inference form's bits; with
    ``keypoint_bar``, ``check_keypoints``.  Returns the float64 heatmaps."""
    dtype = feats.dtype
    logits_ref, hm_ref = ref_forward(head, feats)
    head.final_softmax = True
    with torch.no_grad():
        for split in splits:
            with contextlib.nullcontext() if split is None else softmax_split(_lib(), split):
                out = head(feats)
            assert out.dtype == torch.float32 and out.shape == hm_ref.shape
            check_heatmaps(out, hm_ref, case if split is None else f"{case} split={split}", dtype=dtype)
        head.final_softmax = False
        check_logits(head(feats), logits_ref, case, dtype=dtype)
        head.final_softmax = True
    del logits_ref
    if train:
        out_train = head(feats.clone().requires_grad_(True))
        assert torch.equal(out_train.detach(), out), case
    if keypoint_bar is not None:
        check_keypoints(out, hm_ref, head.downsample_factor, case, keypoint_bar)
    return hm_ref


# ------------------------------------------------------------------------------------------------
# the band maxima of the 16-bit softmax and the decode that reads them
# ------------------------------------------------------------------------------------------------
def bits(t):
    return t.contiguous().view(torch.int32)


def band_max_of(hm, rows, nbands):
    """per (frame, plane, band) maximum of the non-NaN values in heatmap rows [2 j rows, 2 (j + 1) rows)"""
    b, k, h, w = hm.shape
    pad = torch.zeros((b, k, nbands * 2 * rows - h, w), device=hm.device)
    x = torch.cat([torch.nan_to_num(hm, nan=0.0), pad], dim=2)
    return x.reshape(b, k, nbands, 2 * rows * w).amax(dim=3)


def band_dims(h, w):
    """(rows, bands) of ``lpb_head_band_max_dims`` for h x w heatmaps"""
    import ctypes

    r, n = ctypes.c_int(0), ctypes.c_int(0)
    assert _lib().lpb_head_band_max_dims(h, w, ctypes.byref(r), ctypes.byref(n)) == 0
    return r.value, n.value


def assert_same_decode(hm, bm, ds, case, temperature=1000.0):
    """The decode on the band maxima ``bm`` gives ``ops.decode_forward``'s full-sweep xy, confidence and stats, bit for
    bit; returns the full sweep's."""
    from lightning_pose_b200 import ops

    full = ops.decode_forward(hm, ds, temperature)
    banded = ops.decode_forward(hm, ds, temperature, band_max=bm)
    for name, a, b in zip(("xy", "conf", "stats"), full, banded):
        assert torch.equal(bits(a), bits(b)), f"{case} ds={ds}: {name} differs in {int((bits(a) != bits(b)).sum())} elements"
    return full


def head_run(feats, weights, biases, split):
    """The 16-bit softmax head with its band maxima under softmax form ``split``, on features in either memory format
    (``ops.feature_layout``): the heatmaps equal the plain call's bits, and the maxima equal the heatmaps' own per band.
    Returns (heatmaps, ``ops.BandMax``)."""
    from lightning_pose_b200 import ops

    layout = ops.feature_layout(feats)
    with softmax_split(_lib(), split):
        hm, hints = ops._head_forward_16(feats, weights, biases, True, want_hints=True, layout=layout)
        plain = ops._head_forward_16(feats, weights, biases, True, layout=layout)
    torch.cuda.synchronize()
    assert torch.equal(bits(hm), bits(plain)), "writing the band maxima changed the heatmaps"
    rows, nbands = band_dims(hm.shape[2], hm.shape[3])
    assert (hints.rows, hints.nbands) == (rows, nbands) and hints.bits.shape == (*hm.shape[:2], nbands, 8)
    want = band_max_of(hm, rows, nbands)
    got = hints.bits.view(torch.float32).amax(dim=3)
    assert torch.equal(bits(got), bits(want)), "band maxima differ from the heatmaps' own"
    return hm, hints


def backward_checks(head, feats, softmax, hm_ref, case, seed=7, frozen=False, db_max_rule=False):
    """bf16 gradients of sum(head(feats) * gout), gout random, against float64 (``check_grads``); with ``frozen`` also
    the weight gradients of a frozen backbone's call (no feature gradient requested)."""
    head.final_softmax = softmax
    ws, bs = head_params(head)
    gout = torch.randn(hm_ref.shape, device="cuda", generator=gen(seed))
    got = grads(head, feats, gout)
    assert got["dfeat"].dtype == torch.bfloat16
    ref, gnorm = ref_grads(feats, ws, bs, gout, softmax, hm_ref)
    case = f"{case} softmax={softmax}"
    rule = softmax if db_max_rule else None
    check_grads(got, ref, gnorm, case, db_max_rule=rule)
    if frozen:
        del ref["dfeat"]
        check_grads(grads(head, feats, gout, feature_grad=False), ref, gnorm, f"{case} frozen backbone", db_max_rule=rule)
    head.final_softmax = True
