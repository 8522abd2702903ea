"""The bf16 head's forward with more than 20 keypoints: keypoint groups on the banded kernels, against float64.

A head whose last layer has more than HEAD_CLS = 20 output channels splits them into groups of 20 (head_prep.cuh); each
group is the 80-column class-major block of a narrow head, and a work item of the banded kernel is (frame [, band],
group).  Two-deconv heads with c1 >= 20 write their mid activations group by group, in 4-channel halves of the K-chunks,
and the constant-one bias channel sits at c1 (inside a group, or past the last one).  The backward takes one group of K
per launch of the data-gradient kernels and adds the groups' fp32 partials in a fixed order, so it stays bit-reproducible;
its gradients are checked against float64 autograd with the rules of head_support.py.

The CPU tests pin the planner and the workspace queries: wide rows are accepted with the banded plan, the cap is
LPB_HEAD_MAX_CHANNELS = 80, and narrow rows give the values of the commit before keypoint groups existed."""
import ctypes

import pytest
import torch

import scale_oracle as S
from head_support import (F64, WORST, backward_checks, check_grads, check_heatmaps, features, forward_checks, fwd_layout, gen, grads,
                          head_params, make_head, ref_forward, ref_grads, report_headroom, row_layout, softmax_split)

CAP = 80  # LPB_HEAD_MAX_CHANNELS (include/lpb200.h)
ERR_INVALID, ERR_UNSUPPORTED = -1, -3

# (C, H, W, channels): the forward's wide rows.  Mirror-fish first (51 keypoints: three mirrored views x 17; ResNet-50
# features of 256 x 384 images).  (21, 21): c1 + 1 = 22, the ones channel in group 1; (40, 40): c1 + 1 = 41, the ones
# channel past both groups; (20, 21): c1 = 20 is one group with the ones channel past it; (63, 63): four groups of mid
# channels take a third K stage; (17, 51): a narrow first layer; then the cap, and one-deconv heads.
WIDE_ROWS = {
    "mirror_fish": (2048, 8, 12, (51, 51)),
    "c2048_12x12_k21": (2048, 12, 12, (21, 21)),
    "c512_8x8_k40": (512, 8, 8, (40, 40)),
    "c512_8x8_k60": (512, 8, 8, (60, 60)),
    "c512_8x8_k63": (512, 8, 8, (63, 63)),
    "c512_8x8_cap": (512, 8, 8, (CAP, CAP)),
    "c512_8x8_20_21": (512, 8, 8, (20, 21)),
    "c512_8x8_17_51": (512, 8, 8, (17, 51)),
    "1d_c384_16x16_k51": (384, 16, 16, (51,)),
    "1d_c384_24x24_k21": (384, 24, 24, (21,)),
    "1d_c384_8x8_cap": (384, 8, 8, (CAP,)),
}

# narrow rows: (C, H, W, c1, c2) -> (plan, forward workspace bytes at B = 8, backward workspace bytes at B = 8), the values
# of the library before keypoint groups
NARROW_ROWS = {
    (2048, 8, 12, 17, 17): (1, 1213184, 9584336),
    (2048, 12, 12, 17, 17): (1, 1618432, 10843856),
    (2048, 16, 16, 17, 17): (0, 2575872, 13803216),
    (384, 16, 16, 17, 0): (0, 88320, 4146624),
    (384, 24, 24, 17, 0): (0, 94720, 5846464),
    (512, 8, 8, 19, 19): (1, 686336, 9584944),
    (512, 8, 8, 19, 20): (1, 686336, 9677344),
    (384, 8, 8, 20, 0): (0, 84480, 3560448),
    (512, 8, 8, 1, 1): (1, 686336, 2342384),
}


def _lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


def _c12(ch):
    return ch[0], (ch[1] if len(ch) == 2 else 0)


def test_planner_accepts_wide_heads():
    """Every wide row takes the banded plan and is accepted by both workspace queries, so it trains and predicts on the
    tensor cores."""
    from lightning_pose_b200 import ops

    lib = _lib()
    for name, (c, h, w, ch) in WIDE_ROWS.items():
        c1, c2 = _c12(ch)
        plan, n = ctypes.c_int(-9), ctypes.c_size_t(0)
        assert lib.lpb_head_bf16_plan(c, h, w, c1, c2, ctypes.byref(plan)) == 0, (name, lib.lpb_last_error())
        assert plan.value == 0, name
        assert lib.lpb_head_bf16_workspace_bytes(8, c, h, w, c1, c2, ctypes.byref(n)) == 0
        assert n.value == fwd_layout(8, c, h, w, c1, c2).total, name
        assert lib.lpb_head_bwd_bf16_workspace_bytes(8, c, h, w, c1, c2, ctypes.byref(n)) == 0, (name, lib.lpb_last_error())
        assert ops.head_bf16_supported((8, c, h, w), list(ch), train=True), name
    # by hand, mirror-fish at B = 8: 3 groups x 16 stages of w1 (983040 B), 3 x 2 stages of w2 (c1 + 1 = 52 -> 60 group
    # channels -> 2 stages), mid 8 x 8 chunks x 1672 rows x 16 B, statistics 8 x 3 groups x 7 bands x 20 x 2 floats
    n = ctypes.c_size_t(0)
    assert lib.lpb_head_bf16_workspace_bytes(8, 2048, 8, 12, 51, 51, ctypes.byref(n)) == 0
    assert n.value == 983040 + 122880 + 1712128 + 26880 == 2844928


def test_planner_rejects_past_the_cap():
    """One channel past the cap in the last layer (or in the first of a wide two-deconv head) is UNSUPPORTED; a two-deconv
    head with c1 = 20 and c2 <= 20 stays outside the bf16 set as before (INVALID)."""
    lib = _lib()
    plan = ctypes.c_int(-9)
    for c, h, w, c1, c2 in [(512, 8, 8, CAP + 1, CAP + 1), (512, 8, 8, 17, CAP + 1), (384, 8, 8, CAP + 1, 0)]:
        assert lib.lpb_head_bf16_plan(c, h, w, c1, c2, ctypes.byref(plan)) == ERR_UNSUPPORTED, (c1, c2)
    assert lib.lpb_head_bf16_plan(512, 8, 8, CAP + 1, CAP, ctypes.byref(plan)) == ERR_UNSUPPORTED
    assert lib.lpb_head_bf16_plan(512, 8, 8, 20, 20, ctypes.byref(plan)) == ERR_INVALID
    assert lib.lpb_head_bf16_plan(2048, 12, 12, 20, 17, ctypes.byref(plan)) == ERR_INVALID


def test_narrow_rows_unchanged():
    """Heads with 20 or fewer keypoints keep their plan and both workspace sizes; the restated layout reproduces them."""
    lib = _lib()
    for (c, h, w, c1, c2), (want_plan, want_fwd, want_bwd) in NARROW_ROWS.items():
        plan, n = ctypes.c_int(-9), ctypes.c_size_t(0)
        assert lib.lpb_head_bf16_plan(c, h, w, c1, c2, ctypes.byref(plan)) == 0 and plan.value == want_plan
        assert lib.lpb_head_bf16_workspace_bytes(8, c, h, w, c1, c2, ctypes.byref(n)) == 0 and n.value == want_fwd
        assert fwd_layout(8, c, h, w, c1, c2).total == want_fwd
        assert lib.lpb_head_bwd_bf16_workspace_bytes(8, c, h, w, c1, c2, ctypes.byref(n)) == 0 and n.value == want_bwd


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(WIDE_ROWS))
def test_wide_forward(dev, row):
    """heatmaps (both softmax forms) and logits against float64; mirror-fish at B = 8"""
    c, h, w, ch = WIDE_ROWS[row]
    head = make_head(c, ch, seed=13).requires_grad_(False)
    # the batch-size choice (split below one wave of (frame, group) items), then fused
    forward_checks(head, features(8 if row == "mirror_fish" else 4, c, h, w, 5, torch.bfloat16), row, splits=(1, 0), train=False)


@pytest.mark.gpu
def test_wide_mid_activations(dev):
    """The mid activations of a wide two-deconv head hold c1 channels, the constant one at c1, and exact zeros in every
    other channel of their K-chunks (the next layer sums all of them)."""
    from lightning_pose_b200 import ops

    for c1 in (20, 40, 51, 63):
        c, h, w, c2, b = 512, 4, 4, 21, 2
        head = make_head(c, (c1, c2), seed=31).requires_grad_(False)
        feats = features(b, c, h, w, 32, torch.bfloat16)
        ws, bs = head_params(head)
        _, (xs, fws) = ops._head_forward_bf16(feats, ws, bs, True, train=True)
        _, mid_at, nst2, rows, _ = fwd_layout(b, c, h, w, c1, c2)
        hi, wi = 4 * h, 4 * w
        pp, lead, _ = row_layout(hi, wi)
        mid = fws[mid_at : mid_at + b * 4 * nst2 * rows * 16].view(torch.bfloat16).view(b, 4 * nst2, rows, 8)
        img = mid[:, :, lead : lead + hi * pp].reshape(b, 4 * nst2, hi, pp, 8)[:, :, :, :wi]  # (b, kc, y, x, 8)
        chans = img.permute(0, 1, 4, 2, 3).reshape(b, 32 * nst2, hi, wi).float()
        ref = S.head_ref_chunked(feats, ws[:1], bs[:1], softmax=False)
        err = (chans[:, :c1].to(F64) - ref).abs()
        assert bool((err <= 2.0**-7 * ref.abs() + 1e-2 * ref.abs().amax()).all()), (c1, float(err.max()))
        assert bool((chans[:, c1] == 1).all()), c1
        assert bool((chans[:, c1 + 1 :] == 0).all()), c1
        pads = torch.cat([mid[:, :, :lead].flatten(), mid[:, :, lead + hi * pp :].flatten(),
                          mid[:, :, lead : lead + hi * pp].reshape(b, 4 * nst2, hi, pp, 8)[:, :, :, wi:].flatten()])
        assert bool((pads.float() == 0).all()), c1


@pytest.mark.gpu
def test_wide_fused_decode(dev):
    """forward_with_keypoints at K = 51 without autograd: the heatmaps are the head's, the keypoints and confidences the
    float64 soft-argmax decode of them."""
    b, c, h, w, ch = 4, 512, 8, 8, (51, 51)
    head = make_head(c, ch, seed=23, gain=4.0).requires_grad_(False)
    feats = features(b, c, h, w, 11, torch.bfloat16)
    with torch.no_grad():
        hm, kp, cf = head.forward_with_keypoints(feats)
        assert torch.equal(head(feats), hm)
    _, hm_ref = ref_forward(head, feats)
    check_heatmaps(hm, hm_ref, "fused decode K=51")
    preds, _, _, conf_alt = S.decode_ref(hm, 2, 1000.0)
    assert kp.shape == (b, 2 * ch[1])
    assert bool(((kp.to(F64) - preds).abs() <= 2e-3 + 1e-4 * preds.abs()).all()), float((kp.to(F64) - preds).abs().max())
    assert float((cf.to(F64)[..., None] - conf_alt).abs().amin(-1).max()) <= 1e-4


@pytest.mark.gpu
def test_wide_past_one_wave(dev):
    """K = 51 at B = 2 S + 7: with the fused softmax a frame alone gives the batch's bits and a permuted batch permuted
    bits; the batch also matches float64, and the split form (forced) is batch-invariant too."""
    lib = _lib()
    c, h, w, ch = 512, 8, 8, (51, 51)
    b = 2 * torch.cuda.get_device_properties(dev).multi_processor_count + 7
    head = make_head(c, ch, seed=19).requires_grad_(False)
    feats = features(b, c, h, w, 9, torch.bfloat16)
    perm = torch.randperm(b, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        with softmax_split(lib, 0):
            out = head(feats)
            for i in sorted({0, 1, b // 2, b - 1}):
                assert torch.equal(head(feats[i : i + 1])[0], out[i]), i
            assert torch.equal(head(feats[perm]), out[perm])
        with softmax_split(lib, 2):
            split = head(feats)
            assert torch.equal(head(feats[perm]), split[perm])
            for i in (0, b - 1):
                assert torch.equal(head(feats[i : i + 1])[0], split[i]), i
    _, hm_ref = ref_forward(head, feats)
    check_heatmaps(out, hm_ref, f"K=51 B={b} fused")
    check_heatmaps(split, hm_ref, f"K=51 B={b} split")


@pytest.mark.gpu
def test_wide_batched_predictor_graph(dev):
    """BatchedPredictor with K = 51 on bf16 features: the table replayed from its CUDA graph equals the eager one."""
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    k, n, chunk, c, fh, fw, img = 51, 20, 8, 512, 4, 4, 128
    head = make_head(c, (k, k), seed=3).requires_grad_(False).eval()
    feats = features(n, c, fh, fw, 4, torch.bfloat16)
    bbox = torch.tensor([[3.0, 5.0, 200.0, 260.0]], device=dev).repeat(n, 1) + torch.arange(n, device=dev)[:, None]
    pad = (-n) % chunk
    f_dev = torch.cat([feats, feats[-1:].repeat(pad, 1, 1, 1)])
    b_dev = torch.cat([bbox, bbox[-1:].repeat(pad, 1)])
    tables = {}
    for use_graph in (False, True):
        bp = BatchedPredictor(head, k, n, chunk, (img, img), use_graph=use_graph)
        bp.run((f_dev[i : i + chunk], b_dev[i : i + chunk]) for i in range(0, n + pad, chunk))
        torch.cuda.synchronize()
        assert int(bp.cursor) == n + pad
        tables[use_graph] = bp.table.clone()
    assert tables[True].shape == (n, 3 * k)
    assert torch.equal(tables[True], tables[False])
    assert bool(torch.isfinite(tables[True]).all())


# ------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------
BWD_ROWS = ["mirror_fish", "c2048_12x12_k21", "c512_8x8_k40", "c512_8x8_k60", "c512_8x8_cap", "c512_8x8_17_51",
            "c512_8x8_20_21", "1d_c384_16x16_k51", "1d_c384_8x8_cap"]


@pytest.mark.gpu
@pytest.mark.parametrize("row", BWD_ROWS)
def test_wide_backward(dev, row):
    """dfeat, dW1, db1 [, dW2, db2] against float64 autograd, with and without the final softmax"""
    c, h, w, ch = WIDE_ROWS[row]
    head = make_head(c, ch, seed=17)
    feats = features(8 if row == "mirror_fish" else 4, c, h, w, 6, torch.bfloat16)
    _, hm_ref = ref_forward(head, feats)
    for softmax in (True, False):
        backward_checks(head, feats, softmax, hm_ref, row, seed=8)


@pytest.mark.gpu
def test_wide_fused_decode_backward(dev):
    """forward_with_keypoints at K = 51 and its sparse-window backward: the soft-argmax gradient by float64 autograd at
    the kernel's heatmaps, chained into the head's (the rules of test_head_shapes_gpu.py::test_fused_decode)."""
    from lightning_pose_b200 import ops

    b, c, h, w, ch = 4, 512, 8, 8, (51, 51)
    case = "fused decode K=51"
    head = make_head(c, ch, seed=23, gain=4.0)
    feats = features(b, c, h, w, 11, torch.bfloat16)
    k = ch[1]
    g_kp = torch.randn(b, 2 * k, device=dev, generator=gen(12))
    f = feats.clone().requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f)
    (kp * g_kp).sum().backward()
    hm = hm.detach()
    ws, bs = head_params(head)
    g_hm = S.decode_grad_ref(hm, 2, 1000.0, g_kp)
    ref, gnorm = ref_grads(feats, ws, bs, g_hm, True, hm)
    deconvs = list(head.upsampling_layers)[1:]
    got = {"dfeat": f.grad, "dw1": deconvs[0].weight.grad, "db1": deconvs[0].bias.grad, "dw2": deconvs[1].weight.grad, "db2": deconvs[1].bias.grad}
    check_grads(got, ref, gnorm, case, rel=2e-2, global_scale=("dw2",))
    _, _, stats = ops._decode_fwd(hm, 2, 1000.0)
    g_hm = ops._decode_bwd(hm, stats, g_kp.reshape(b, k, 2).contiguous(), 2, 1000.0)
    ref, gnorm = ref_grads(feats, ws, bs, g_hm, True, hm)
    check_grads(got, ref, gnorm, f"{case}, kernel decode gradient", rel=2e-2)


@pytest.mark.gpu
def test_wide_backward_past_one_wave(dev):
    """K = 51 at B = 2 S + 7: two backward runs are bit-identical, a frame alone gets the batch's d-feature bits, a permuted
    batch permuted bits; the gradients also match float64."""
    lib = _lib()
    c, h, w, ch = 512, 8, 8, (51, 51)
    b = 2 * torch.cuda.get_device_properties(dev).multi_processor_count + 7
    head = make_head(c, ch, seed=19)
    feats = features(b, c, h, w, 9, torch.bfloat16)
    gout = torch.randn(b, ch[-1], 8 * h, 8 * w, device=dev, generator=gen(10))
    with softmax_split(lib, 0):
        got = grads(head, feats, gout)
        again = grads(head, feats, gout)
        for name in got:
            assert torch.equal(got[name], again[name]), name
        for i in (0, b - 1):
            assert torch.equal(grads(head, feats[i : i + 1], gout[i : i + 1])["dfeat"][0], got["dfeat"][i]), i
        perm = torch.randperm(b, generator=torch.Generator().manual_seed(1)).to(dev)
        assert torch.equal(grads(head, feats[perm], gout[perm])["dfeat"], got["dfeat"][perm])
    _, hm_ref = ref_forward(head, feats)
    ws, bs = head_params(head)
    ref, gnorm = ref_grads(feats, ws, bs, gout, True, hm_ref)
    check_grads(got, ref, gnorm, f"K=51 B={b}")
