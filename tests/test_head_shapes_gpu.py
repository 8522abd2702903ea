"""The bf16 head at every feature width its backward serves and at keypoint counts other than 17, against float64.

Several pieces of the tensor-core head depend on the shape: the class-major packing at stride HEAD_CLS = 20, the
constant-one bias channel at index c1 of the mid activations (the last class slot at c1 = 19), the padding channels of
the banded softmax, the b3a data-gradient kernel instantiated per feature width (its band height, last short band,
partial 128-channel tiles and TMA or direct-store epilogue), and the bias gradients of either head depth.  The width
table below puts one shape through each of them; the channel sweep runs 1 to 20 keypoints on two cheap shapes.  What
the table claims to cover is asserted on the CPU from the library's planner and the launch formulas restated here
(``b3a_*``), so a later routing change cannot quietly shrink the coverage.  The comparison helpers are shown to reject
plausible kernel bugs on a float64 reference (``test_comparisons_reject_plausible_kernel_bugs``)."""
import contextlib
import ctypes

import pytest
import torch

import scale_oracle as S

F64 = torch.float64

# ------------------------------------------------------------------------------------------------
# coverage: the width / route table and the launch formulas it relies on
# ------------------------------------------------------------------------------------------------
# name: (deconvs, C, H, W, channels, B, forward route, b3a bands (rows of the 2H x 2W grid), b3a epilogue)
WIDTH_TABLE = {
    "2d_c2048_4x4": (2, 2048, 4, 4, (17, 17), 4, "k1a", [8], "tma"),
    "2d_c128_48x4": (2, 128, 48, 4, (4, 4), 3, "k1a", [28, 28, 28, 12], "tma"),
    "2d_c512_8x8": (2, 512, 8, 8, (9, 9), 4, "k1a", [12, 4], "tma"),
    "2d_c768_8x12": (2, 768, 8, 12, (19, 19), 3, "k1a", [8, 8], "tma"),
    "2d_c640_12x16": (2, 640, 12, 16, (8, 17), 3, "k1a", [4] * 6, "tma"),
    "2d_c2048_32x32": (2, 2048, 32, 32, (17, 17), 2, "banded", [4] * 16, "direct"),
    "1d_c384_8x8": (1, 384, 8, 8, (20,), 4, "banded", [12, 4], "tma"),
    "1d_c768_16x24": (1, 768, 16, 24, (1,), 3, "banded", [4] * 8, "direct"),
    "1d_c384_32x32": (1, 384, 32, 32, (17,), 3, "banded", [4] * 16, "direct"),
}

# the channel sweep's two shapes: 2-deconv C = 512 at 8x8 (k1a) and 1-deconv C = 384 at 8x8 (banded)
SWEEP_TWO = [(1, 1), (2, 2), (4, 4), (17, 17), (19, 19), (19, 20), (8, 17), (17, 8)]
SWEEP_ONE = [1, 4, 17, 20]

HEAD_KC = 10  # K-chunks of 8 in the gradients' class-major K (head_prep.cuh)


def b3a_band_rows(hi1, wi1):
    """(rows per band Hh, whether Hh comes from the one-buffer formula) of b3a_band_rows (head_bwd_bf16.cu)."""
    hh = (256 // (wi1 + 1)) & ~3  # two accumulator buffers fit
    one_buffer = hh < 4
    if one_buffer:
        hh = (304 // (wi1 + 1)) & ~3
    return min(hh, hi1), one_buffer


def b3a_bands(h, w):
    """rows of each band the b3a kernel cuts the 2H x 2W grid of a frame into."""
    hh, _ = b3a_band_rows(2 * h, 2 * w)
    return [min(hh, 2 * h - r) for r in range(0, 2 * h, hh)]


def b3a_epilogue(h, w):
    """'tma' when the TMA store's staging slices fit beside the b3a stages and the d-feature tensor map encodes, else
    'direct' (lpb_head_bwd_bf16, make_dfeat_tensor_map)."""
    hh, _ = b3a_band_rows(2 * h, 2 * w)
    ncols = (hh * (2 * w + 1) + 15) & ~15
    rows_alloc = (2 * w + 2 + ncols + 7) & ~7
    smem = 2 * HEAD_KC * rows_alloc * 16 + 4 * HEAD_KC * 128 * 16 + 160
    stage = 2 * 4 * 128 * 4 * w + 128
    encodes = (h * w * 2) % 16 == 0 and (2 * w * 2) % 16 == 0 and 2 * w <= 256
    return "tma" if smem + stage <= 225 * 1024 and encodes else "direct"


def b3a_c4_tiles(c):
    """filled channels of each 128-channel tile of the C/4 shuffled channels the b3a kernel splits a frame into."""
    c4 = c // 4
    return [min(128, c4 - t) for t in range(0, c4, 128)]


def _plan(c, h, w, ch):
    from lightning_pose_b200._lib import lib

    plan = ctypes.c_int(-1)
    assert lib.lpb_head_bf16_plan(c, h, w, ch[0], ch[1] if len(ch) == 2 else 0, ctypes.byref(plan)) == 0, lib.lpb_last_error()
    return {1: "k1a", 0: "banded"}[plan.value]


@pytest.mark.parametrize("row", list(WIDTH_TABLE))
def test_width_table_routes(row):
    """Each row takes the forward route, b3a bands and epilogue the table lists, and trains on the bf16 kernels."""
    from lightning_pose_b200 import ops

    n, c, h, w, ch, b, route, bands, epi = WIDTH_TABLE[row]
    assert len(ch) == n
    assert _plan(c, h, w, ch) == route
    assert ops.head_bf16_supported((b, c, h, w), list(ch), train=True)
    assert b3a_bands(h, w) == bands
    assert b3a_epilogue(h, w) == epi


def test_width_table_coverage():
    """The table covers every width the backward serves, both b3a epilogues, both forward routes, the one-buffer band
    height, a short last b3a band, a partial second channel tile, k1a with one channel stage, and non-square maps."""
    from lightning_pose_b200._lib import lib

    n = ctypes.c_size_t(0)
    served = {w for w in range(1, 65) if lib.lpb_head_bwd_bf16_workspace_bytes(2, 512, 8, w, 17, 17, ctypes.byref(n)) == 0}
    assert served == {4, 8, 12, 16, 24, 32}
    rows = WIDTH_TABLE.values()
    assert {r[3] for r in rows} == served
    assert {r[6] for r in rows} == {"k1a", "banded"}
    assert {r[8] for r in rows} == {"tma", "direct"}
    assert any(b3a_band_rows(2 * r[2], 2 * r[3])[1] for r in rows)  # W = 32: Hh from the one-buffer formula
    assert any(len(r[7]) > 1 and r[7][-1] < r[7][0] for r in rows)
    assert any(len(b3a_c4_tiles(r[1])) > 1 and b3a_c4_tiles(r[1])[-1] < 128 for r in rows)
    assert any(r[6] == "k1a" and r[1] // 4 // 32 == 1 for r in rows)  # one 32-channel K stage
    assert any(r[2] != r[3] for r in rows)
    for n_deconv in (1, 2):  # both depths at both epilogues
        assert {r[8] for r in rows if r[0] == n_deconv} == {"tma", "direct"}


def test_sweep_covers_channel_edges():
    """The sweep runs 1 keypoint, c1 = 19 (bias channel in the last class slot), c2 = 20 and c1 = 20 (no padding channel),
    and c1 != c2 both ways; every pair is accepted by the planner and trains on the bf16 kernels."""
    from lightning_pose_b200 import ops

    assert {1, 19} <= {c1 for c1, _ in SWEEP_TWO} and 20 in {c2 for _, c2 in SWEEP_TWO} and 20 in SWEEP_ONE and 1 in SWEEP_ONE
    assert any(c1 < c2 for c1, c2 in SWEEP_TWO) and any(c1 > c2 for c1, c2 in SWEEP_TWO)
    for ch in SWEEP_TWO:
        assert _plan(512, 8, 8, ch) == "k1a" and ops.head_bf16_supported((4, 512, 8, 8), list(ch), train=True)
    for c1 in SWEEP_ONE:
        assert _plan(384, 8, 8, (c1,)) == "banded" and ops.head_bf16_supported((4, 384, 8, 8), [c1], train=True)


# ------------------------------------------------------------------------------------------------
# comparison helpers: every rule is applied per keypoint plane / output channel / frame, and returns its ratios
# (error / allowed), so that one wrong small channel cannot hide behind a large one
# ------------------------------------------------------------------------------------------------
WORST: dict = {}  # quantity -> (largest ratio seen, case)


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


def check_heatmaps(out, ref, case="", key="heatmaps"):
    """Acceptance rule of the bf16 head (test_head_bf16_real_config_shapes_forward): relative error below 3e-2 on every
    pixel, above 1e-2 on under 0.01 % of the pixels, and every keypoint plane sums to 1 within 1e-5.  The 0.01 % holds
    over the batch and, per plane, with 9 pixels to spare: a mid activation on a bf16 rounding boundary that rounds the
    other way moves the 3 x 3 output pixels it feeds, and a plane of fewer than 10^4 pixels would otherwise allow none."""
    out, ref = out.detach().to(F64), ref.to(F64)
    rel = (out - ref).abs() / (ref.abs() + 1e-7)
    over = (rel > 1e-2).to(F64)
    _judge(case, {f"{key}: relative error": rel.amax((-1, -2)) / 3e-2,
                  f"{key}: pixels over 1e-2": over.mean() / 1e-4,
                  f"{key}: pixels over 1e-2 per plane": over.sum((-1, -2)) / (1e-4 * rel[0, 0].numel() + 9),
                  f"{key}: plane sum": (out.sum((-1, -2)) - 1).abs() / 1e-5})


def check_logits(out, ref, case=""):
    """Logits head: within 1e-2 of the plane's largest magnitude plus 1e-2 relative, per (frame, keypoint) plane."""
    out, ref = out.detach().to(F64), ref.to(F64)
    allowed = 1e-2 * ref.abs().amax((-1, -2), keepdim=True) + 1e-2 * ref.abs() + 1e-12
    _judge(case, {"logits": ((out - ref).abs() / allowed).amax((-1, -2))})


def logit_grad(gout, probs=None):
    """d loss / d logits for a dense output gradient: the spatial softmax's backward when ``probs`` is given."""
    g = gout.to(F64)
    if probs is None:
        return g
    p = probs.to(F64)
    return p * (g - (p * g).sum((-1, -2), keepdim=True))


def check_grads(got: dict, ref: dict, gnorm: dict, case="", rel=1e-2, global_scale=()):
    """bf16 backward against float64 (the rule of test_head_bf16_real_config_shapes_backward, applied per channel).

    ``dfeat``: per frame, ``rel`` times the frame's largest gradient.  ``dw{i}`` [Cin, Cout, 3, 3] (layers counted from 1): per output channel,
    ``rel`` times that channel's largest weight gradient.  ``db{i}``: a bias gradient is its channel's output gradient
    summed over every pixel of every frame.  Behind a softmax that sum cancels exactly, and with a dense random gradient it
    is a sum of random signs, so the channel's own value is no scale for the error.  What sets the error is the bf16
    rounding of the gradient operand the kernels sum, at most 2^-9 of each element, whose sum over the channel is bounded
    by 4 x 2^-8 of the channel's gradient L2 norm ``gnorm[f"db{i}"][o]`` (the bound of
    test_head_with_keypoints_past_one_wave); plus ``rel`` of the channel's value, as for the other quantities.
    Quantities named in ``global_scale`` are held to ``rel`` times their largest entry instead (the rule of
    test_head_with_keypoints_past_one_wave), where the caller says why no per-channel bound is meaningful."""
    ratios = {}
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
    _judge(case, ratios)


def check_grads_f32(got: dict, ref: dict, gnorm: dict, case=""):
    """fp32 CUDA-core backward against float64: dfeat comes back rounded to the features' bf16 (2^-8 relative, 1e-4 of the
    frame's largest gradient for the fp32 sums under it), the weight
    gradients within 1e-3 relative of each channel's scale, the bias gradients within 2^-14 of the channel's gradient L2
    norm (a thirtieth of what a bf16 gradient operand would leave)."""
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


def _grad_norms(n_deconv, glogit, mid_norm=None):
    """per-channel L2 norms of the gradient each bias sums: the logits' for the last layer, the mid activations' for the
    first of two."""
    out = {f"db{n_deconv}": glogit.pow(2).sum((0, 2, 3)).sqrt()}
    if n_deconv == 2:
        out["db1"] = mid_norm
    return out


def _ref_grads(feats, ws, bs, gout, softmax, probs, bf16_operands=True):
    n = len(ws)
    res = S.head_grad_ref(feats, ws, bs, gout, softmax=softmax, bf16_operands=bf16_operands, want_mid_grad=n == 2)
    dfeat, dws, dbs = res[:3]
    ref = {"dfeat": dfeat, **{f"dw{i}": g for i, g in enumerate(dws, 1)}, **{f"db{i}": g for i, g in enumerate(dbs, 1)}}
    return ref, _grad_norms(n, logit_grad(gout, probs if softmax else None), res[3] if n == 2 else None)


def test_comparisons_reject_plausible_kernel_bugs():
    """On a float64 reference of a small two-deconv head, each plausible kernel bug applied to a copy is rejected by the
    helper the GPU tests use, and the unchanged reference is accepted."""
    torch.manual_seed(3)
    b, c, h, w, c1, c2 = 2, 128, 8, 8, 4, 4
    ws = [torch.nn.init.xavier_uniform_(torch.empty(c // 4, c1, 3, 3), gain=3.0), torch.nn.init.xavier_uniform_(torch.empty(c1, c2, 3, 3), gain=3.0)]
    bs = [torch.empty(c1).uniform_(-0.3, 0.3), torch.empty(c2).uniform_(-0.3, 0.3)]
    feats = (torch.randn(b, c, h, w) * 0.5).bfloat16()
    logits = S.head_ref_chunked(feats, ws, bs, softmax=False)
    hm = torch.softmax(logits.flatten(2), -1).reshape(logits.shape)
    gout = torch.randn(logits.shape, dtype=F64)
    ref, gnorm = _ref_grads(feats, ws, bs, gout, False, None)

    def rejects(fn, *args):
        with pytest.raises(AssertionError):
            fn(*args, case="mutated")

    check_heatmaps(hm.clone(), hm, case="reference")
    check_logits(logits.clone(), logits, case="reference")
    check_grads({k: v.clone() for k, v in ref.items()}, ref, gnorm, case="reference")
    WORST.clear()

    # a class-stride off-by-one: two adjacent keypoint channels of dw2 trade places
    bad = {k: v.clone() for k, v in ref.items()}
    bad["dw2"][:, [1, 2]] = ref["dw2"][:, [2, 1]]
    rejects(check_grads, bad, ref, gnorm)
    # the constant-one channel lost: the logits without the layer-2 bias
    rejects(check_logits, logits - bs[1].to(F64).view(1, -1, 1, 1), logits)
    # the last b3a band's rows of d features left at zero (2H x 2W grid rows 12..15 = feature rows 6, 7)
    assert b3a_bands(h, w) == [12, 4]
    bad = {k: v.clone() for k, v in ref.items()}
    bad["dfeat"][:, :, 12 // 2 :] = 0
    rejects(check_grads, bad, ref, gnorm)
    # the last keypoint plane of the heatmaps uniform (a padding channel's softmax written in its place)
    bad_hm = hm.clone()
    bad_hm[:, -1] = 1.0 / (bad_hm.shape[-1] * bad_hm.shape[-2])
    rejects(check_heatmaps, bad_hm, hm)
    # the layer-1 bias gradient never reduced
    bad = {k: v.clone() for k, v in ref.items()}
    bad["db1"].zero_()
    rejects(check_grads, bad, ref, gnorm)
    WORST.clear()


# ------------------------------------------------------------------------------------------------
# GPU: the sweep
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    """With ``-s``: the largest error / allowed ratio seen per quantity (how much headroom each rule has)."""
    WORST.clear()
    yield
    for name, (ratio, case) in sorted(WORST.items()):
        print(f"headroom {name:36s} {ratio:9.4f}  ({case})")


@contextlib.contextmanager
def softmax_unsplit(lib):
    """pin the fused per-frame softmax (LPB_TUNE_SOFTMAX_SPLIT = 0): a frame then computes the same bits at any batch"""
    saved = lib.lpb_get_tuning(7)
    try:
        assert lib.lpb_set_tuning(7, 0) == 0
        yield
    finally:
        lib.lpb_set_tuning(7, saved)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _make_head(n_deconv, c, ch, seed=13, final_softmax=True):
    """``_rand_head``-style weights (test_gpu_parity.py) for a head with deconv channels ``ch``."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    if n_deconv == 2:
        head = HeatmapHead("resnet50", c, ch[1], deconv_out_channels=ch[0], final_softmax=final_softmax)
    else:
        head = HeatmapHead("vits_dino", c, ch[0], final_softmax=final_softmax)
    deconvs = list(head.upsampling_layers)[1:]
    assert len(deconvs) == n_deconv and [d.weight.shape[1] for d in deconvs] == list(ch)
    for layer in deconvs:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
        torch.nn.init.uniform_(layer.bias, -0.3, 0.3)
    return head.cuda()


def _params(head):
    deconvs = list(head.upsampling_layers)[1:]
    return [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs]


def _feats(b, c, h, w, seed=5):
    return (torch.randn(b, c, h, w, device="cuda", generator=_gen(seed)) * 0.5).bfloat16()


def _grads(head, feats, gout):
    head.zero_grad(set_to_none=True)
    f = feats.clone().requires_grad_(True)
    (head(f) * gout).sum().backward()
    out = {"dfeat": f.grad}
    for i, d in enumerate(list(head.upsampling_layers)[1:], 1):
        out[f"dw{i}"], out[f"db{i}"] = d.weight.grad, d.bias.grad
    return out


def _forward_checks(head, feats, case):
    """softmax heatmaps and logits against float64, and the training form's bits against the inference form's;
    returns the float64 heatmaps."""
    ws, bs = _params(head)
    logits_ref = S.head_ref_chunked(feats, ws, bs, softmax=False)
    hm_ref = torch.softmax(logits_ref.flatten(2), -1).reshape(logits_ref.shape)
    head.final_softmax = True
    with torch.no_grad():
        out = head(feats)
    assert out.dtype == torch.float32 and out.shape == hm_ref.shape
    check_heatmaps(out, hm_ref, case)
    head.final_softmax = False
    with torch.no_grad():
        lg = head(feats)
    check_logits(lg, logits_ref, case)
    del lg, logits_ref
    head.final_softmax = True
    out_train = head(feats.clone().requires_grad_(True))
    assert torch.equal(out_train.detach(), out), case
    return hm_ref


def _backward_checks(head, feats, softmax, hm_ref, case, seed=7):
    head.final_softmax = softmax
    ws, bs = _params(head)
    gout = torch.randn(hm_ref.shape, device="cuda", generator=_gen(seed))
    got = _grads(head, feats, gout)
    assert got["dfeat"].dtype == torch.bfloat16
    ref, gnorm = _ref_grads(feats, ws, bs, gout, softmax, hm_ref)
    check_grads(got, ref, gnorm, f"{case} softmax={softmax}")
    head.final_softmax = True


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(WIDTH_TABLE))
def test_width_table(dev, row):
    n, c, h, w, ch, b, _, _, _ = WIDTH_TABLE[row]
    head = _make_head(n, c, ch)
    feats = _feats(b, c, h, w)
    hm_ref = _forward_checks(head, feats, row)
    for softmax in (True, False):
        _backward_checks(head, feats, softmax, hm_ref, row)


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [*SWEEP_TWO, *[(c1,) for c1 in SWEEP_ONE]], ids=lambda ch: "c" + "_".join(map(str, ch)))
def test_channel_sweep(dev, ch):
    n = len(ch)
    c = 512 if n == 2 else 384
    case = f"{n}d_c{c}_8x8 ch={ch}"
    head = _make_head(n, c, ch, seed=17)
    feats = _feats(4, c, 8, 8, seed=6)
    hm_ref = _forward_checks(head, feats, case)
    _backward_checks(head, feats, True, hm_ref, case, seed=8)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["2d_c512_8x8", "1d_c384_32x32"])
def test_batch_invariance(dev, lib, row):
    """A frame alone computes the same forward and d-feature bits as inside the batch, and permuting the frames permutes
    both exactly.  The 8 x 8 row runs at B = 2S + 7, so the persistent launches loop; it is also checked against float64
    there."""
    n, c, h, w, ch, b, _, _, _ = WIDTH_TABLE[row]
    if row == "2d_c512_8x8":
        b = 2 * torch.cuda.get_device_properties(dev).multi_processor_count + 7
    head = _make_head(n, c, ch, seed=19)
    feats = _feats(b, c, h, w, seed=9)
    up = 8 if n == 2 else 4
    gout = torch.randn(b, ch[-1], up * h, up * w, device=dev, generator=_gen(10))
    with softmax_unsplit(lib):
        with torch.no_grad():
            out = head(feats)
        got = _grads(head, feats, gout)
        for i in sorted({0, 1, b // 2, b - 1}):
            with torch.no_grad():
                assert torch.equal(head(feats[i : i + 1])[0], out[i]), (row, i)
            assert torch.equal(_grads(head, feats[i : i + 1], gout[i : i + 1])["dfeat"][0], got["dfeat"][i]), (row, i)
        perm = torch.randperm(b, generator=torch.Generator().manual_seed(1)).to(dev)
        with torch.no_grad():
            assert torch.equal(head(feats[perm]), out[perm])
        assert torch.equal(_grads(head, feats[perm], gout[perm])["dfeat"], got["dfeat"][perm])
    # and with the softmax form the batch size selects (split over (frame, band) below one wave)
    with torch.no_grad():
        out = head(feats)
        assert torch.equal(head(feats[perm]), out[perm])
    got = _grads(head, feats, gout)
    assert torch.equal(_grads(head, feats[perm], gout[perm])["dfeat"], got["dfeat"][perm])
    if row == "2d_c512_8x8":
        ws, bs = _params(head)
        logits_ref = S.head_ref_chunked(feats, ws, bs, softmax=False)
        hm_ref = torch.softmax(logits_ref.flatten(2), -1).reshape(logits_ref.shape)
        check_heatmaps(out, hm_ref, f"{row} B={b}")
        ref, gnorm = _ref_grads(feats, ws, bs, gout, True, hm_ref)
        check_grads(got, ref, gnorm, f"{row} B={b}")


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [(1, 1), (19, 19)], ids=["c1_1", "c19_19"])
def test_fused_decode(dev, ch):
    """forward_with_keypoints and its sparse-window backward at 1 and 19 keypoints: the soft-argmax gradient by float64
    autograd at the kernel's heatmaps, chained into the head's (test_head_with_keypoints_past_one_wave's rules)."""
    from lightning_pose_b200 import ops

    b, c, h, w = 4, 512, 8, 8
    case = f"fused decode ch={ch}"
    head = _make_head(2, c, ch, seed=23)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=4.0)
    feats = _feats(b, c, h, w, seed=11)
    k = ch[1]
    g_kp = torch.randn(b, 2 * k, device=dev, generator=_gen(12))
    f = feats.clone().requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f)
    (kp * g_kp).sum().backward()
    hm = hm.detach()
    with torch.no_grad():
        assert torch.equal(head(feats), hm)
    preds, _, _, conf_alt = S.decode_ref(hm, 2, 1000.0)
    assert bool(((kp.to(F64) - preds).abs() <= 2e-3 + 1e-4 * preds.abs()).all()), float((kp.to(F64) - preds).abs().max())
    assert float((cf.to(F64)[..., None] - conf_alt).abs().amin(-1).max()) <= 1e-4
    g_hm = S.decode_grad_ref(hm, 2, 1000.0, g_kp)
    ws, bs = _params(head)
    ref, gnorm = _ref_grads(feats, ws, bs, g_hm, True, hm)
    deconvs = list(head.upsampling_layers)[1:]
    got = {"dfeat": f.grad, "dw1": deconvs[0].weight.grad, "db1": deconvs[0].bias.grad, "dw2": deconvs[1].weight.grad, "db2": deconvs[1].bias.grad}
    # dw2 against its largest entry: at T = 1000 the softmax backward p (g - sum(p g)) of a peaked plane cancels all but
    # a sliver of its decode gradient g, and what is left of a small keypoint's plane (|dw2[:, o]| ~ 1e-3 beside 7e3 at
    # 19 keypoints) lies below the decode kernel's fp32 gradient error, which shows up the same through the dense decode
    # backward.  The head itself is held per channel below, against the decode gradient the kernels sum.
    check_grads(got, ref, gnorm, case, rel=2e-2, global_scale=("dw2",))
    _, _, stats = ops._decode_fwd(hm, 2, 1000.0)
    g_hm = ops._decode_bwd(hm, stats, g_kp.reshape(b, k, 2).contiguous(), 2, 1000.0)
    ref, gnorm = _ref_grads(feats, ws, bs, g_hm, True, hm)
    check_grads(got, ref, gnorm, f"{case}, kernel decode gradient", rel=2e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,ch", [((3, 512, 8, 8), (20, 20)), ((3, 512, 8, 6), (17, 17))], ids=["c20_20", "w6_train"])
def test_fp32_fallback(dev, shape, ch):
    """Heads the bf16 kernels do not train take the fp32 CUDA-core kernels: two deconvs with c1 = 20 (no room for the
    ones channel) at any call, W = 6 (forward only on the bf16 kernels) when a backward can follow.  Both match float64
    at fp32 tolerance, which the bf16 route could not."""
    from lightning_pose_b200 import ops

    b, c, h, w = shape
    assert not ops.head_bf16_supported(shape, list(ch), train=True)
    assert ops.head_bf16_supported(shape, list(ch), train=False) == (w == 6)
    case = f"fp32 fallback {shape} ch={ch}"
    head = _make_head(2, c, ch, seed=29)
    feats = _feats(b, c, h, w, seed=13)
    ws, bs = _params(head)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, bf16_operands=False)
    f = feats.clone().requires_grad_(True)
    out = head(f)
    err = (out.detach().to(F64) - hm_ref).abs()
    assert bool((err <= 1e-4 * hm_ref + 1e-9).all()), (case, float((err / (1e-4 * hm_ref + 1e-9)).max()))
    gout = torch.randn(hm_ref.shape, device=dev, generator=_gen(14))
    (out * gout).sum().backward()
    deconvs = list(head.upsampling_layers)[1:]
    got = {"dfeat": f.grad, "dw1": deconvs[0].weight.grad, "db1": deconvs[0].bias.grad, "dw2": deconvs[1].weight.grad, "db2": deconvs[1].bias.grad}
    ref, gnorm = _ref_grads(feats, ws, bs, gout, True, hm_ref, bf16_operands=False)
    check_grads_f32(got, ref, gnorm, case)
