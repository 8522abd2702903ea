"""Three-deconv heads (downsample_factor 1 on a stride-32 backbone) on the 16-bit tensor-core kernels, against float64:
forward in bf16 and fp16, NCHW and channels-last, the band maxima and the decode that reads them, the gradients (dense,
decode windows, implicit keypoint targets), bit-reproducibility, batches past one wave, and the model-level routes.
The ``no_fp32_head`` fixture makes the fp32 head kernels raise: every covered shape runs on the 16-bit kernels alone.

The test heads are initialised at xavier gain 2 per layer (GAIN): three layers at the two-deconv tests' gain 3 give logits
about three times wider, so the same operand roundings move the softmax's small tail probabilities by that much more in
relative terms, and the shared bars (set for two layers) would be measuring the head's scale rather than the kernels."""
import pytest
import torch

import scale_oracle as S
from head_support import (F64, WORST, assert_same_decode, bits, check_grads, features, forward_checks, gen, grads, head_params, head_run,
                          logit_grad, make_head, ref_forward, report_headroom)

pytestmark = pytest.mark.gpu
GAIN = 2.0

SHAPES = {  # name -> (B, C, H, W)
    "c2048_12x12": (2, 2048, 12, 12),
    "c2048_8x8": (3, 2048, 8, 8),
    "c2048_4x4": (4, 2048, 4, 4),
    "c2048_16x16": (2, 2048, 16, 16),
    "c2048_8x12": (2, 2048, 8, 12),
    "c512_8x8": (3, 512, 8, 8),
}
CHANNELS = [(17, 17, 17), (8, 8, 17), (19, 19, 20), (17, 17, 5)]
CASES = [(s, ch) for s in SHAPES for ch in ((17, 17, 17),)] + [("c2048_8x8", ch) for ch in CHANNELS[1:]] + [("c512_8x8", ch) for ch in CHANNELS[1:]]


def case_id(v):
    return v if isinstance(v, str) else "c" + "_".join(map(str, v))


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


@pytest.fixture
def no_fp32_head(monkeypatch):
    """The fp32 head kernels raise when called."""
    from lightning_pose_b200 import ops

    def refuse(*args, **kwargs):
        raise AssertionError("the fp32 head kernels ran for a shape the 16-bit kernels cover")

    monkeypatch.setattr(ops, "head_forward_f32", refuse)
    monkeypatch.setattr(ops, "convt_backward_f32", refuse)
    monkeypatch.setattr(ops, "convt_forward_f32", refuse)


def ref_grads3(feats, ws, bs, gout, softmax, probs):
    """float64 gradients and, per bias, the L2 norm of the gradient it sums: the logits' (db3) and the mid activations'
    (db1: the input of layer 2, db2: the input of layer 3)."""
    w64 = [w.detach().to(F64).requires_grad_(True) for w in ws]
    b64 = [b.detach().to(F64).requires_grad_(True) for b in bs]
    dfeat = torch.empty(feats.shape, device=feats.device, dtype=F64)
    sq = [None, None]
    for i in range(feats.shape[0]):
        f = feats[i : i + 1].detach().to(F64).requires_grad_(True)
        mids: list = []
        y = S.head_ref(f, w64, b64, softmax, torch.bfloat16, mids=mids)
        (y * gout[i : i + 1].to(F64)).sum().backward()
        dfeat[i : i + 1] = f.grad
        for j in range(2):
            s = mids[j].grad.pow(2).sum((0, 2, 3))
            sq[j] = s if sq[j] is None else sq[j] + s
    ref = {"dfeat": dfeat, **{f"dw{i}": w.grad for i, w in enumerate(w64, 1)}, **{f"db{i}": b.grad for i, b in enumerate(b64, 1)}}
    gnorm = {"db1": sq[0].sqrt(), "db2": sq[1].sqrt(), "db3": logit_grad(gout, probs if softmax else None).pow(2).sum((0, 2, 3)).sqrt()}
    return ref, gnorm


def layout_of(feats, nhwc):
    return feats.contiguous(memory_format=torch.channels_last) if nhwc else feats


@pytest.mark.parametrize("name,ch", CASES, ids=[f"{s}-{case_id(c)}" for s, c in CASES])
@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_forward(no_fp32_head, name, ch, nhwc):
    b, c, h, w = SHAPES[name]
    head = make_head(c, ch, seed=13, gain=GAIN)
    assert head.downsample_factor == 1
    for dtype in (torch.bfloat16, torch.float16):
        feats = layout_of(features(b, c, h, w, 5, dtype), nhwc)
        case = f"{name} ch={ch} {dtype} {'nhwc' if nhwc else 'nchw'}"
        hm_ref = forward_checks(head, feats, case, splits=(None, 0, 2), train=dtype == torch.bfloat16, keypoint_bar=0.5)
        assert hm_ref.shape == (b, ch[-1], 16 * h, 16 * w)
        ws, bs = head_params(head)
        for split in (0, 2):
            hm, hints = head_run(feats, ws, bs, split)
            if 16 * w <= 192:
                assert_same_decode(hm, hints, 1, case)
            else:  # the decode's shared-memory tile takes 192 x 192 planes, not 256 x 256 ones: it refuses them
                from lightning_pose_b200._lib import LpbError
                from lightning_pose_b200 import ops

                with pytest.raises(LpbError, match="error -3"):
                    ops.decode_forward(hm, 1, 1000.0, band_max=hints)


@pytest.mark.parametrize("name,ch", CASES, ids=[f"{s}-{case_id(c)}" for s, c in CASES])
def test_backward(no_fp32_head, name, ch):
    b, c, h, w = SHAPES[name]
    head = make_head(c, ch, seed=21, gain=GAIN)
    feats = features(b, c, h, w, 6, torch.bfloat16)
    _, hm_ref = ref_forward(head, feats)
    gout = torch.randn(hm_ref.shape, device="cuda", generator=gen(7))
    ws, bs = head_params(head)
    for softmax in (True, False):
        head.final_softmax = softmax
        got = grads(head, feats, gout)
        assert got["dfeat"].dtype == torch.bfloat16 and set(got) == {"dfeat", "dw1", "db1", "dw2", "db2", "dw3", "db3"}
        ref, gnorm = ref_grads3(feats, ws, bs, gout, softmax, hm_ref)
        case = f"{name} ch={ch} softmax={softmax}"
        check_grads(got, ref, gnorm, case)
        again = grads(head, feats, gout)
        for k in got:
            assert torch.equal(bits(got[k]), bits(again[k])), f"{case}: {k} differs between two identical backward calls"
        del ref["dfeat"]
        check_grads(grads(head, feats, gout, feature_grad=False), ref, gnorm, f"{case} frozen backbone")
    head.final_softmax = True


def test_backward_channels_last(no_fp32_head):
    b, c, h, w = SHAPES["c2048_8x8"]
    head = make_head(c, (17, 17, 17), seed=22, gain=GAIN)
    feats = features(b, c, h, w, 8, torch.bfloat16)
    gout = torch.randn(b, 17, 16 * h, 16 * w, device="cuda", generator=gen(9))
    nchw = grads(head, feats, gout)
    nhwc = grads(head, layout_of(feats, True), gout)
    assert nhwc["dfeat"].is_contiguous(memory_format=torch.channels_last)
    for k in nchw:
        assert torch.equal(bits(nchw[k].contiguous()), bits(nhwc[k].contiguous())), k


def test_decode_windows(no_fp32_head):
    """forward_with_keypoints and its sparse-window backward: the soft-argmax gradient by float64 autograd at the kernel's
    heatmaps, chained into the head's (test_head_shapes_gpu.py::test_fused_decode's rules)."""
    from lightning_pose_b200 import ops

    b, c, h, w = 3, 512, 8, 8
    ch = (17, 17, 17)
    head = make_head(c, ch, seed=23, gain=GAIN)
    feats = features(b, c, h, w, 11, torch.bfloat16)
    g_kp = torch.randn(b, 2 * ch[-1], device="cuda", generator=gen(12))
    f = feats.clone().requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f)
    (kp * g_kp).sum().backward()
    hm = hm.detach()
    with torch.no_grad():
        assert torch.equal(head(feats), hm)
    preds, _, _, _ = S.decode_ref(hm, 1, 1000.0)
    assert bool(((kp.to(F64) - preds).abs() <= 2e-3 + 1e-4 * preds.abs()).all()), float((kp.to(F64) - preds).abs().max())
    deconvs = list(head.upsampling_layers)[1:]
    got = {"dfeat": f.grad, **{f"dw{i}": d.weight.grad for i, d in enumerate(deconvs, 1)}, **{f"db{i}": d.bias.grad for i, d in enumerate(deconvs, 1)}}
    _, _, stats = ops._decode_fwd(hm, 1, 1000.0)
    g_hm = ops._decode_bwd(hm, stats, g_kp.reshape(b, ch[-1], 2).contiguous(), 1, 1000.0)
    ws, bs = head_params(head)
    ref, gnorm = ref_grads3(feats, ws, bs, g_hm, True, hm)
    check_grads(got, ref, gnorm, "decode windows, kernel decode gradient", rel=2e-2)


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_implicit_keypoint_targets(no_fp32_head, nhwc):
    """The keypoint-target MSE's gradient stays implicit into the three-deconv backward, with the same bits as the same
    backward fed the materialised gradient; with the decode windows as well."""
    from lightning_pose_b200 import ops

    b, c, h, w, k = 4, 2048, 8, 8, 17
    head = make_head(c, (17, 17, k), seed=3, gain=GAIN)
    f = layout_of(features(b, c, h, w, seed=4, dtype=torch.bfloat16), nhwc).requires_grad_(True)
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    g = torch.Generator().manual_seed(5)
    img = 2.0 * 16 * h  # the heatmap (16H x 16W) is half the image at downsample factor 1
    kp = (torch.rand(b, k, 2, generator=g) * img).cuda()
    vis = torch.randint(0, 3, (b, k), generator=g, dtype=torch.int32).cuda()
    for with_decode in (False, True):
        if with_decode:
            hm, kpp, _ = head.forward_with_keypoints(f)
        else:
            hm = head(f)
        loss = ops.heatmap_mse_from_keypoints(kp, hm, img, img, visibility=vis)
        (gl,) = torch.autograd.grad(loss, hm, retain_graph=True)
        assert isinstance(gl, ops.MseKeypointGrad)
        outs = [hm] + ([kpp] if with_decode else [])
        g_kp = [torch.randn(kpp.shape, device="cuda", generator=gen(6))] if with_decode else []
        implicit = torch.autograd.grad(outs, [f] + params, [gl] + g_kp, retain_graph=True)
        assert gl.dense is None, "the head backward materialised the gradient"
        dense = torch.autograd.grad(outs, [f] + params, [gl.materialize().clone()] + g_kp, retain_graph=True)
        for i, (x, y) in enumerate(zip(implicit, dense)):
            assert torch.equal(bits(x.contiguous()), bits(y.contiguous())), (with_decode, i)


def test_past_one_wave(no_fp32_head):
    """B = 2 SMs + 7 frames: every persistent launch (k1a, the banded layers with the fused softmax, b2d, the weight
    gradients, b3a) loops past one wave; forward and gradients against float64, and a frame alone gives the batch's bits."""
    from head_support import softmax_split, _lib

    b = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    c, h, w, ch = 512, 4, 4, (17, 17, 17)
    head = make_head(c, ch, seed=31, gain=GAIN)
    feats = features(b, c, h, w, 12, torch.bfloat16)
    hm_ref = forward_checks(head, feats, f"B={b}", keypoint_bar=0.5)
    gout = torch.randn(hm_ref.shape, device="cuda", generator=gen(13))
    ws, bs = head_params(head)
    got = grads(head, feats, gout)
    ref, gnorm = ref_grads3(feats, ws, bs, gout, True, hm_ref)
    check_grads(got, ref, gnorm, f"B={b}")
    with softmax_split(_lib(), 0), torch.no_grad():
        out = head(feats)
        for i in (0, b // 2, b - 1):
            assert torch.equal(head(feats[i : i + 1])[0], out[i]), i


def test_tracker_step_from_keypoint_targets(no_fp32_head):
    """A HeatmapTracker with downsample_factor 1 trains a labeled step from keypoint targets on the 16-bit kernels: the
    heatmaps are half the image, and the head's gradients equal those of its backward fed the dense target gradient."""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker

    class Conv(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 512, 32, stride=32)

        def forward(self, x):
            return self.conv(x).bfloat16()

    b, k, img = 4, 17, 256
    torch.manual_seed(41)
    t = HeatmapTracker(k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None), backbone=Conv(), downsample_factor=1,
                       num_fc_input_features=512).cuda()
    assert len(list(t.head.upsampling_layers)) == 4
    for layer in list(t.head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=GAIN)
    g = torch.Generator().manual_seed(42)
    kp = torch.rand(b, k, 2, generator=g) * img
    batch = {"images": torch.randn(b, 3, img, img, generator=g).cuda(), "bbox": torch.tensor([[0.0, 0.0, img, img]]).repeat(b, 1).cuda(),
             "keypoints": kp.reshape(b, -1).cuda(), "visibility": torch.full((b, k), 2, dtype=torch.int32).cuda()}
    loss = t.evaluate_labeled(batch, "train", 1.0)
    loss.backward()
    assert torch.isfinite(loss)
    for p in t.head.parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0


def test_batched_predictor_graph_equals_eager(no_fp32_head):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    k, n, chunk, c, img = 17, 20, 8, 512, 256
    head = make_head(c, (17, 17, k), seed=43, gain=GAIN).eval()
    feats = features(n + (-n) % chunk, c, 8, 8, 14, torch.bfloat16)
    bbox = (torch.tensor([[3.0, 5.0, 200.0, 260.0]], device="cuda").repeat(feats.shape[0], 1)
            + torch.arange(feats.shape[0], device="cuda")[:, None])
    tables = []
    for use_graph in (True, False):
        bp = BatchedPredictor(head, k, n, chunk, (img, img), use_graph=use_graph)
        bp.run((feats[i : i + chunk], bbox[i : i + chunk]) for i in range(0, feats.shape[0], chunk))
        torch.cuda.synchronize()
        tables.append(bp.table.clone())
    assert torch.equal(bits(tables[0]), bits(tables[1]))
