"""GPU: a NaN or inf frame stays in its own outputs (DESIGN.md K2, "Non-finite frames").

A diverged fp16 backbone or training step hands the head a frame holding NaN or inf.  In the reference (torch) that
ruins that frame's heatmaps and keypoints and nothing else.  Here persistent CTAs carry shared-memory tiles from frame
b to frame b + grid, bands and chunks have short tails, and tap blocks multiply by structural zeros: each could leak a
NaN into another frame, or into a later graph replay.  Every test plants the bad value in frame j of a batch past one
wave (2 S + 7 frames, S the SM count), j in {0, S - 1 (the last frame of a one-frame-per-CTA first wave), B - 1}, and
compares with the run where frame j holds its clean values:

- one NaN pixel, one +inf pixel, -inf at the corner (row 0, last column: next to the pads of the row layout), and an
  all-NaN frame;
- every other frame is bit-identical to the clean run; frame j is NaN wherever the float64 reference of that frame is.
"""
import pytest
import torch

import scale_oracle as S
from head_support import features, gen, head_params, make_head, softmax_split

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CL = torch.channels_last
F64 = torch.float64
BAD = ["nan", "inf", "-inf_corner", "nan_frame"]


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


def positions(b, sms):
    return {"first": 0, "wave_end": sms - 1, "last": b - 1}


def plant(x, j, bad):
    """``x`` with the bad value in frame j (x is (B, C, H, W) in any memory format; the copy keeps it)."""
    y = x.clone()
    c, h, w = x.shape[1:]
    if bad == "nan":
        y[j, c // 3, h // 2, w // 3] = float("nan")
    elif bad == "inf":
        y[j, c - 1, h - 1, 0] = float("inf")
    elif bad == "-inf_corner":
        y[j, 0, 0, w - 1] = float("-inf")
    else:
        y[j] = float("nan")
    return y


def bits(t):
    return t.detach().contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()])


def assert_others_same(a, b, j, case, name):
    keep = torch.ones(a.shape[0], dtype=torch.bool, device=a.device)
    keep[j] = False
    ba, bb = bits(a)[keep], bits(b)[keep]
    assert torch.equal(ba, bb), f"{case}: {name} of frames other than {j} differ in {int((ba != bb).sum())} elements"


def assert_nan_where(got, ref, case, name, exact=False):
    """``got`` is NaN wherever the float64 ``ref`` is (and, with ``exact``, nowhere else)."""
    gn, rn = torch.isnan(got), torch.isnan(ref)
    missing = rn & ~gn
    assert not bool(missing.any()), f"{case}: {name} finite at {int(missing.sum())} of the reference's {int(rn.sum())} NaNs"
    if exact:
        extra = gn & ~rn
        assert not bool(extra.any()), f"{case}: {name} NaN at {int(extra.sum())} entries where the reference is not"


def assert_nonfinite_within(got, ref, case, name):
    """``got`` is finite wherever the float64 ``ref`` is, and NaN only where ``ref`` is not finite."""
    rf = torch.isfinite(ref)
    wide = rf & ~torch.isfinite(got)
    assert not bool(wide.any()), f"{case}: {name} not finite at {int(wide.sum())} entries where the reference is"


# ------------------------------------------------------------------------------------------------
# head forward
# ------------------------------------------------------------------------------------------------
# route -> (C, H, W, deconv channels, feature dtype, channels-last)
ROUTES = {
    "k1a_bf16": (128, 13, 8, (17, 17), torch.bfloat16, False),
    "banded_2d_bf16": (128, 8, 5, (17, 17), torch.bfloat16, False),
    "banded_1d_bf16_nhwc": (128, 9, 8, (20,), torch.bfloat16, True),
    "k1a_fp16": (128, 13, 8, (17, 17), torch.float16, False),
    "1d_fp16_nhwc": (128, 9, 8, (20,), torch.float16, True),
    "wide_k40_bf16": (512, 8, 8, (40, 40), torch.bfloat16, False),
    "banded_2d_bf16_nhwc": (128, 13, 8, (17, 17), torch.bfloat16, True),
    "three_bf16": (512, 8, 8, (8, 8, 17), torch.bfloat16, False),
    "three_bf16_nhwc": (512, 8, 8, (8, 8, 17), torch.bfloat16, True),
    "fp32_3xtf32": (128, 6, 7, (17, 17), torch.float32, False),
    "fp32_3xtf32_nhwc": (128, 6, 7, (17,), torch.float32, True),
}


def _head_outputs(ops, head, f, softmax):
    """(heatmaps or logits, band-maxima bits or None, xy, conf) of the head's inference call"""
    head.final_softmax = softmax
    with torch.no_grad():
        if f.dtype == torch.float32:
            hm = head(f)
            bm = None
        else:
            hm, bm = ops._head_forward_16(f, *head_params(head), softmax, want_hints=True, layout=ops.feature_layout(f))
            assert torch.equal(bits(hm), bits(head(f)))
        xy, conf, _ = ops.decode_forward(hm, head.downsample_factor, 1000.0, band_max=bm)
    head.final_softmax = True
    return hm, (bm.bits if bm is not None else None), xy, conf


# the softmax form of the 16-bit routes (SOFTMAX_SPLIT, head_support.py): 0 the fused per-frame kernel, 2 split over
# (frame, group, band) with the statistics combined after; the fp32 route has one form
FWD_CASES = [(r, split) for r, v in ROUTES.items() for split in ((0, 2) if v[4] != torch.float32 else (1,))]


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("route,split", FWD_CASES)
def test_head_forward_bad_frame(ops, lib, sms, route, split, softmax):
    c, h, w, ch, dtype, nhwc = ROUTES[route]
    b = 2 * sms + 7
    head = make_head(c, ch, seed=3)
    ws, bs = head_params(head)
    clean = features(b, c, h, w, seed=4, dtype=dtype)
    if nhwc:
        clean = clean.contiguous(memory_format=CL)
    operands = dtype if dtype != torch.float32 else None
    assert dtype == torch.float32 or ops.head_16_operand(clean, list(ch), train=False)[1] == (ops.FEATURES_NHWC if nhwc else ops.FEATURES_NCHW)
    with softmax_split(lib, split):
        base = _head_outputs(ops, head, clean, softmax)
        for pos, j in positions(b, sms).items():
            for bad in BAD:
                case = f"{route} split={split} softmax={softmax} {bad} at {pos} (frame {j})"
                f = plant(clean, j, bad)
                got = _head_outputs(ops, head, f, softmax)
                for name, x, y in zip(("heatmaps", "band maxima", "xy", "conf"), base, got):
                    if x is not None:
                        assert_others_same(x, y, j, case, name)
                ref = S.head_ref(f[j : j + 1].contiguous(), ws, bs, softmax=softmax, operands=operands)[0]
                assert_nan_where(got[0][j], ref, case, "heatmaps")
                # and not finite wherever torch is not (an inf logit stays inf on the 16-bit routes, and is NaN on the
                # fp32 route: DESIGN.md K2, "Non-finite frames")
                lost = ~torch.isfinite(ref) & torch.isfinite(got[0][j])
                assert not bool(lost.any()), f"{case}: finite at {int(lost.sum())} entries where the reference is not"
                if softmax:
                    # every plane of the reference is NaN: each deconv mixes every channel, and a plane's softmax
                    # shares its NaN with the whole plane
                    assert bool(torch.isnan(ref).all()), case
                    assert bool(torch.isnan(got[2][j]).all()), f"{case}: keypoints {got[2][j]}"
                    assert bool(torch.isnan(got[3][j]).all()), f"{case}: confidences {got[3][j]}"


# ------------------------------------------------------------------------------------------------
# head backward (bf16)
# ------------------------------------------------------------------------------------------------
BWD = {"vit_1d": (384, 16, 16, (17,)), "cfg2": (2048, 12, 12, (17, 17))}


def _grads(ops, head, f, kind, softmax, gout, gkp, kp):
    head.zero_grad(set_to_none=True)
    head.final_softmax = softmax
    x = f.detach().clone().requires_grad_(True)
    if kind == "dense":
        (head(x) * gout).sum().backward()
    elif kind == "windows":
        _, xy, _ = head.forward_with_keypoints(x)
        (xy * gkp).sum().backward()
    else:
        hm = head(x)
        img = (4 * hm.shape[2], 4 * hm.shape[3])
        ops.heatmap_mse_from_keypoints(kp * torch.tensor(img[::-1], device=DEV, dtype=torch.float32), hm, img[0], img[1]).backward()
    head.final_softmax = True
    deconvs = list(head.upsampling_layers)[1:]
    out = {"dfeat": x.grad}
    for i, d in enumerate(deconvs, 1):
        out[f"dw{i}"], out[f"db{i}"] = d.weight.grad, d.bias.grad
    return out


def _softargmax_ref(hm, ds):
    """the reference's soft-argmax coordinates (B, 2K) of float64 heatmaps, differentiable (``scale_oracle._decode_planes``
    without its confidence windows, whose indices a NaN coordinate would not give)"""
    b, k, hh, ww = hm.shape
    planes = hm.reshape(b * k, hh, ww)
    field = S.upsample_op(hh, ds, hm.device) @ planes @ S.upsample_op(ww, ds, hm.device).T
    p = torch.softmax(field.flatten(1) * 1000.0, -1).reshape(field.shape)
    x = (p.sum(1) * torch.arange(field.shape[2], device=hm.device, dtype=F64)).sum(-1)
    y = (p.sum(2) * torch.arange(field.shape[1], device=hm.device, dtype=F64)).sum(-1)
    return torch.stack([x, y], -1).reshape(b, 2 * k)


def _frame_grad_ref(ops, head, f, j, kind, softmax, gout, gkp, kp):
    """float64 autograd of frame j's own term of the loss ``_grads`` differentiates: {"dfeat" (frame j), "dw1", "db1",
    ...}.  Every other frame's term is finite, so the NaN pattern of the whole batch's weight and bias gradients is that
    of frame j's term."""
    ws, bs = head_params(head)
    x = f[j : j + 1].to(F64).requires_grad_(True)
    w64 = [w.to(F64).requires_grad_(True) for w in ws]
    b64 = [b_.to(F64).requires_grad_(True) for b_ in bs]
    hm = S.head_ref(x, w64, b64, softmax=softmax)
    if kind == "dense":
        loss = (hm * gout[j : j + 1]).sum()
    elif kind == "windows":
        loss = (_softargmax_ref(hm, head.downsample_factor) * gkp[j : j + 1]).sum()
    else:
        img = (4 * hm.shape[2], 4 * hm.shape[3])
        t = ops.generate_heatmaps(kp[j : j + 1] * torch.tensor(img[::-1], device=DEV, dtype=torch.float32), img[0], img[1], hm.shape[2:])
        loss = ((hm - t.to(F64)) ** 2).sum()
    g = torch.autograd.grad(loss, [x, *w64, *b64])
    n = len(ws)
    return {"dfeat": g[0][0], **{f"dw{i}": g[i] for i in range(1, n + 1)}, **{f"db{i}": g[n + i] for i in range(1, n + 1)}}


@pytest.mark.parametrize("kind,softmax", [("dense", True), ("dense", False), ("windows", True), ("mse", True)])
@pytest.mark.parametrize("row", list(BWD))
def test_head_backward_bad_frame(ops, sms, row, kind, softmax):
    c, h, w, ch = BWD[row]
    b = 2 * sms + 7
    head = make_head(c, ch, seed=5, gain=4.0)
    clean = features(b, c, h, w, seed=6, dtype=torch.bfloat16)
    up = 4 * 2 ** (len(ch) - 1)
    gout = torch.randn(b, ch[-1], up * h, up * w, device=DEV, generator=gen(7))
    gkp = torch.randn(b, 2 * ch[-1], device=DEV, generator=gen(8))
    kp = torch.rand(b, ch[-1], 2, device=DEV, generator=gen(9))
    base = _grads(ops, head, clean, kind, softmax, gout, gkp, kp)
    for pos, j in positions(b, sms).items():
        for bad in BAD:
            case = f"{row} {kind} softmax={softmax} {bad} at {pos} (frame {j})"
            f = plant(clean, j, bad)
            got = _grads(ops, head, f, kind, softmax, gout, gkp, kp)
            assert_others_same(base["dfeat"], got["dfeat"], j, case, "dfeat")
            if not softmax:
                # a logits head is linear: frame j's dfeat and db1 do not depend on the features
                assert torch.equal(bits(got["dfeat"][j]), bits(base["dfeat"][j])), case
                assert torch.equal(bits(got["db1"]), bits(base["db1"])), case
                assert bool(torch.isfinite(got["dfeat"]).all()), case
            ref = _frame_grad_ref(ops, head, f, j, kind, softmax, gout, gkp, kp)
            for name, r in ref.items():
                g = got[name][j] if name == "dfeat" else got[name]
                if bad in ("nan", "nan_frame") or not name.startswith("dw"):
                    assert_nan_where(g.float(), r, case, name, exact=True)
                else:
                    # an inf feature or mid activation on the map's border: torch's weight gradient multiplies it by
                    # the zero gradient of the taps that fall outside the output (inf x 0 = NaN); the kernels skip
                    # those taps (DESIGN.md K2, "Non-finite frames")
                    assert_nonfinite_within(g.float(), r, case, name)


@pytest.mark.parametrize("softmax", [True, False])
def test_head_backward_nan_gradient(ops, sms, softmax):
    """A NaN in g_out of frame j: every frame's dfeat other than j is bit-identical; the NaN pattern of every gradient is
    float64 autograd's."""
    c, h, w, ch = BWD["vit_1d"]
    b = 2 * sms + 7
    head = make_head(c, ch, seed=10, gain=4.0)
    ws, bs = head_params(head)
    f = features(b, c, h, w, seed=11, dtype=torch.bfloat16)
    gout = torch.randn(b, ch[-1], 4 * h, 4 * w, device=DEV, generator=gen(12))
    base = _grads(ops, head, f, "dense", softmax, gout, None, None)
    for j in (0, sms - 1, b - 1):
        g = gout.clone()
        g[j, 3, 5, 7] = float("nan")
        got = _grads(ops, head, f, "dense", softmax, g, None, None)
        case = f"g_out NaN at frame {j} softmax={softmax}"
        assert_others_same(base["dfeat"], got["dfeat"], j, case, "dfeat")
        res = S.head_grad_ref(f, ws, bs, g, softmax=softmax)
        ref = {"dfeat": res[0], "dw1": res[1][0], "db1": res[2][0]}
        for name, r in ref.items():
            assert_nan_where(got[name].float(), r, case, name, exact=True)


# ------------------------------------------------------------------------------------------------
# crnn, regression, losses
# ------------------------------------------------------------------------------------------------
def test_crnn_bad_frame(ops):
    k, h, w, hidden, n, m = 5, 4, 6, 8, 60, 57
    g = gen(13)
    wf = torch.randn(n, k, h, w, device=DEV, generator=g)
    wb = torch.randn(n, k, h, w, device=DEV, generator=g)
    idx = torch.randint(0, n, (m, 5), device=DEV, generator=g, dtype=torch.int32)

    def params():
        return [torch.randn(k * hidden, 1, 2, 2, device=DEV, generator=g) * 0.3, torch.randn(k * hidden, device=DEV, generator=g) * 0.1,
                torch.randn(k * hidden, 1, 2, 2, device=DEV, generator=g) * 0.3, torch.randn(k, device=DEV, generator=g) * 0.1]

    hf, hb = params(), params()
    gout = torch.randn(m, k, h, w, device=DEV, generator=g)

    def run(a, bmap):
        leaves = [t.clone().requires_grad_(True) for t in [a, bmap]]
        out = ops.crnn_combine(leaves[0], leaves[1], idx, hf, hb)
        (out * gout).sum().backward()
        return out.detach(), leaves[0].grad, leaves[1].grad

    base = run(wf, wb)
    for fr in (int(idx[0, 2]), int(idx[m - 1, 0])):
        for which in ("wf", "wb"):
            a, bm = wf.clone(), wb.clone()
            (a if which == "wf" else bm)[fr, 2, 1, 3] = float("nan")
            out, dwf, dwb = run(a, bm)
            case = f"NaN in {which} of frame {fr}"
            reads = (idx == fr).any(1)
            assert bool(reads.any())
            assert torch.equal(bits(out[~reads]), bits(base[0][~reads])), case
            ref = S.crnn_combine_ref(a.to(F64), bm.to(F64), idx, [p.to(F64) for p in hf], [p.to(F64) for p in hb])
            assert_nan_where(out, ref, case, "logits", exact=True)
            assert bool(torch.isnan(out[reads]).flatten(1).any(1).all()), case
            # frames that share no window with fr
            near = torch.zeros(n, dtype=torch.bool, device=DEV)
            near[idx[reads].long().flatten()] = True
            assert torch.equal(bits(dwf[~near]), bits(base[1][~near])), case
            assert torch.equal(bits(dwb[~near]), bits(base[2][~near])), case


@pytest.mark.parametrize("dtype,nhwc", [(torch.bfloat16, False), (torch.float16, True), (torch.float32, False)])
def test_regression_head_bad_frame(ops, sms, dtype, nhwc):
    b, c, h, w, n = 2 * sms + 7, 256, 6, 5, 12
    clean = features(b, c, h, w, seed=14, dtype=dtype)
    if nhwc:
        clean = clean.contiguous(memory_format=CL)
    weight = torch.randn(n, c, device=DEV, generator=gen(15)) * 0.05
    bias = torch.randn(n, device=DEV, generator=gen(16))
    g = torch.randn(b, n, device=DEV, generator=gen(17))

    def run(f):
        x = f.clone().requires_grad_(True)
        (ops.regression_head(x, weight, bias) * g).sum().backward()
        return ops.regression_head(f, weight, bias), x.grad

    base = run(clean)
    for j in (0, sms - 1, b - 1):
        for bad in BAD:
            case = f"{dtype} {bad} at frame {j}"
            out, dfeat = run(plant(clean, j, bad))
            assert_others_same(base[0], out, j, case, "output")
            assert_others_same(base[1], dfeat, j, case, "dfeat")
            assert bool(torch.isnan(out[j]).all()) or bad == "inf" or bad == "-inf_corner", case
            assert not bool(torch.isfinite(out[j]).any()), case
            # the pooled mean's gradient does not read the features
            assert torch.equal(bits(dfeat[j]), bits(base[1][j])), case


@pytest.mark.parametrize("kind", ["mse", "kl", "js"])
@pytest.mark.parametrize("source", ["dense", "keypoints"])
def test_heatmap_loss_nan_prediction(ops, kind, source):
    b, k, oh, ow = 9, 7, 24, 20
    kp = torch.rand(b, k, 2, device=DEV, generator=gen(18)) * torch.tensor([80.0, 96.0], device=DEV)
    logits = torch.randn(b, k, oh, ow, device=DEV, generator=gen(19)) * 3
    preds = torch.softmax(logits.flatten(2), -1).reshape(logits.shape)
    targ = ops.generate_heatmaps(kp, 96, 80, (oh, ow))
    targ_ref = targ.to(F64)

    def run(p):
        x = p.clone().requires_grad_(True)
        if source == "dense":
            loss = ops.heatmap_loss(targ, x, kind)
        else:
            loss = ops.heatmap_loss_from_keypoints(kind, kp, x, 96, 80, return_count=True)[0]
        loss.backward()
        return loss.detach(), x.grad.materialize() if isinstance(x.grad, ops.MseKeypointGrad) else x.grad

    base = run(preds)
    for plane in ((0, 0), (4, 3), (b - 1, k - 1)):
        p = preds.clone()
        p[plane[0], plane[1], 5, 7] = float("nan")
        loss, grad = run(p)
        case = f"{source} {kind} NaN at {plane}"
        assert bool(torch.isnan(loss)), case
        _, ref_grad = S.heatmap_loss_ref(targ_ref, p.to(F64), kind, with_grad=True)
        ref_grad = ref_grad.reshape(p.shape)
        rn = torch.isnan(ref_grad)
        assert_nan_where(grad, ref_grad, case, "gradient", exact=True)
        assert torch.equal(bits(grad[~rn]), bits(base[1][~rn])), case


# ------------------------------------------------------------------------------------------------
# predictors
# ------------------------------------------------------------------------------------------------
def _table(head, k, feats, chunk, use_graph=True):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    n = feats.shape[0]
    bp = BatchedPredictor(head, k, n, chunk, (128, 128), use_graph=use_graph)
    bp.run(feats[i : i + chunk] for i in range(0, n, chunk))
    torch.cuda.synchronize()
    return bp.table.clone()


@pytest.mark.parametrize("kind", ["plain", "three", "context"])
def test_predictor_nan_frame(ops, kind):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    k, c, n, chunk, bad = 17, 512, 48, 8, 10
    if kind == "context":
        torch.manual_seed(3)
        head = HeatmapMHCRNNHead("resnet50", c, k).to(DEV).eval()
    else:
        head = make_head(c, (17, 17) if kind == "plain" else (8, 8, 17), seed=4).eval()
    clean = features(n, c, 4, 4, seed=20, dtype=torch.bfloat16)
    f = plant(clean, bad, "nan_frame")
    with torch.no_grad():
        base = _table(head, k, clean, chunk)
        got = _table(head, k, f, chunk)
        touched = [bad] if kind != "context" else list(range(bad - 2, bad + 3))
        keep = torch.ones(n, dtype=torch.bool, device=DEV)
        keep[touched] = False
        assert torch.equal(bits(got[keep]), bits(base[keep])), f"{kind}: rows away from frame {bad} changed"
        assert bool(torch.isnan(got[bad]).all()), got[bad]
        if kind == "context":
            # the rows next to the bad frame keep their single-frame prediction (a NaN conf_mf keeps sf)
            sf = _table(head.head_sf, k, f, chunk)
            near = [t for t in touched if t != bad]
            torch.testing.assert_close(got[near], sf[near], rtol=1e-5, atol=1e-3)
