"""The heatmap head on channels-last features (``torch.channels_last``, a transformer's tokens viewed as a feature map):
read in place, d features written in place, against the NCHW call on the same logical tensor and the float64 references."""
import numpy as np
import pytest
import torch

import channels_last_oracle as O
import head_support as HS
from lightning_pose_b200 import ops
from lightning_pose_b200.models.backbones import tokens_to_feature_map

pytestmark = pytest.mark.gpu
CL = torch.channels_last
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


@pytest.fixture(scope="module", autouse=True)
def _headroom():
    yield
    HS.report_headroom()


def _pair(b, c, h, w, seed, dtype):
    x = HS.features(b, c, h, w, seed, dtype)
    xc = x.contiguous(memory_format=CL)
    assert ops.feature_layout(xc) == ops.FEATURES_NHWC and ops.feature_layout(x) == ops.FEATURES_NCHW
    return x, xc


def test_shuffle_kernel_writes_the_oracles_bytes():
    """The saved operand of a training forward is the row layout: byte-identical between the layouts and to the numpy
    packing of the same features."""
    head = HS.make_head(128, [5], 1)
    ws, bs = HS.head_params(head)
    x, xc = _pair(3, 128, 4, 8, 2, BF16)
    (_, (xs_a, _)) = ops._head_forward_16(x, ws, bs, True, train=True)
    (_, (xs_b, _)) = ops._head_forward_16(xc, ws, bs, True, train=True, layout=ops.FEATURES_NHWC)
    assert torch.equal(xs_a, xs_b)
    want = O.pack_rows_nhwc(xc.permute(0, 2, 3, 1).contiguous().view(torch.int16).cpu().numpy().view(np.uint16))
    assert xs_b.cpu().numpy().tobytes() == want.tobytes()


# the NCHW call of these shapes takes the banded kernels too, so everything downstream of the shuffle is the same code on
# the same bytes; the data gradient's channels-last store rounds the same fp32 sums
SAME_KERNELS = [("vit16", 6, 384, 16, 16, [17]), ("vit24", 4, 384, 24, 24, [17]), ("16x24", 3, 256, 16, 24, [17, 17]),
                ("wide51", 3, 2048, 8, 12, [51, 51]), ("wide-one", 3, 384, 16, 16, [45])]


@pytest.mark.parametrize("case,b,c,h,w,channels", SAME_KERNELS, ids=[s[0] for s in SAME_KERNELS])
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "fp16"])
def test_same_bits_where_the_kernels_coincide(case, b, c, h, w, channels, dtype):
    head = HS.make_head(c, channels, 3)
    x, xc = _pair(b, c, h, w, 4, dtype)
    with torch.no_grad():
        out = head(x)
        assert torch.equal(head(xc), out), case
    if dtype != BF16:
        return
    assert torch.equal(head(xc.clone().requires_grad_(True)).detach(), out)
    for softmax in (True, False):
        head.final_softmax = softmax
        gout = torch.randn(out.shape, device="cuda", generator=HS.gen(5))
        a, g = HS.grads(head, x, gout), HS.grads(head, xc, gout)
        assert g["dfeat"].is_contiguous(memory_format=CL) and not g["dfeat"].is_contiguous()
        for k in a:
            assert torch.equal(a[k], g[k].contiguous()), (case, softmax, k)


K1A = [("resnet12", 6, 2048, 12, 12), ("resnet16", 4, 2048, 16, 16), ("r18-8x12", 5, 512, 8, 12)]


@pytest.mark.parametrize("case,b,c,h,w", K1A, ids=[s[0] for s in K1A])
def test_whole_frame_shapes_against_float64(case, b, c, h, w):
    """NCHW features of these shapes take the whole-frame kernel, channels-last ones the banded kernels: both are held to
    the float64 reference, and their decoded keypoints to each other."""
    head = HS.make_head(c, [17, 17], 6)
    x, xc = _pair(b, c, h, w, 7, BF16)
    hm_ref = HS.forward_checks(head, xc, f"channels-last {case}", keypoint_bar=0.05)
    for softmax in (True, False):
        HS.backward_checks(head, xc, softmax, hm_ref, f"channels-last {case}", frozen=softmax)
    with torch.no_grad():
        HS.check_keypoints(head(xc), head(x).to(HS.F64), head.downsample_factor, f"{case} layouts", 0.05)


F32_CASES = [("one", 3, 384, 8, 8, [17]), ("two", 2, 512, 6, 8, [17, 17]), ("three", 2, 256, 4, 6, [9, 9, 9]), ("cin-50", 2, 200, 6, 4, [7, 5])]


@pytest.mark.parametrize("case,b,c,h,w,channels", F32_CASES, ids=[s[0] for s in F32_CASES])
def test_fp32_route_same_bits(case, b, c, h, w, channels):
    head = HS.make_head(c, channels, 8)
    x, xc = _pair(b, c, h, w, 9, F32)
    with torch.no_grad():
        out = head(x)
        assert torch.equal(head(xc), out)
    gout = torch.randn(out.shape, device="cuda", generator=HS.gen(10))
    a, g = HS.grads(head, x, gout), HS.grads(head, xc, gout)
    assert g["dfeat"].is_contiguous(memory_format=CL)
    # the weight gradient is summed with float atomics in both layouts: its order varies from run to run
    for k in a:
        if k.startswith("dw") or k.startswith("db"):
            torch.testing.assert_close(g[k], a[k], rtol=1e-4, atol=1e-6 + 1e-5 * float(a[k].abs().max()))
        else:
            assert torch.equal(a[k], g[k].contiguous()), (case, k)


def test_token_gradient_and_strides():
    head = HS.make_head(384, [17], 11)
    tokens = HS.features(4, 384, 16, 16, 12, BF16).permute(0, 2, 3, 1).reshape(4, 256, 384).contiguous()
    leaf = tokens.clone().requires_grad_(True)
    fm = tokens_to_feature_map(leaf * 1.0, (16, 16))  # a non-leaf token tensor
    gout = torch.randn(4, 17, 64, 64, device="cuda", generator=HS.gen(13))
    (head(fm) * gout).sum().backward()
    nchw = HS.grads(head, fm.detach().contiguous(), gout)["dfeat"]
    assert leaf.grad.is_contiguous() and torch.equal(leaf.grad, nchw.permute(0, 2, 3, 1).reshape(4, 256, 384))
    # a tensor that is both formats is NCHW; slices that are neither are copied; a misaligned view raises
    x, xc = _pair(4, 384, 16, 16, 14, BF16)
    with torch.no_grad():
        want = head(x)
        assert torch.equal(head(xc[:, :, :, :]), want) and torch.equal(head(xc[1:3]), want[1:3])
        assert torch.equal(head(torch.cat([xc, xc], 1)[:, :384]), want)
        ws, bs = HS.head_params(head)
        odd = torch.empty(4 * 16 * 16 * 384 + 1, device="cuda", dtype=BF16)[1:].view(4, 16, 16, 384).permute(0, 3, 1, 2)
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            ops._head_forward_16(odd, ws, bs, True, layout=ops.FEATURES_NHWC)


def test_multiview_transformer_feeds_the_head_its_tokens():
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    class Embed(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Conv2d(3, 384, 16, 16)

        def forward(self, im):
            return self.proj(im).flatten(2).transpose(1, 2).to(BF16)

    def build():
        torch.manual_seed(0)
        enc = torch.nn.Linear(384, 384).to(BF16)
        factory = LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None)
        return HeatmapTrackerMultiviewTransformer(5, 2, Embed(), enc, 384, loss_factory=factory).cuda()

    a, b = build(), build()
    vit = b.forward_vit
    b.forward_vit = lambda im, channels_last=False: vit(im).contiguous()  # the NCHW copy, as before the view existed
    g = HS.gen(15)
    batch = {"images": torch.randn(3, 2, 3, 256, 256, device="cuda", generator=g),
             "keypoints": torch.rand(3, 20, device="cuda", generator=g) * 256,
             "heatmaps": torch.rand(3, 10, 64, 64, device="cuda", generator=g),
             "bbox": torch.tensor([[0.0, 0.0, 256.0, 256.0] * 2] * 3, device="cuda"), "is_multiview": True}
    la, lb = a.training_step(dict(batch), 0)["loss"], b.training_step(dict(batch), 0)["loss"]
    assert torch.equal(la, lb)
    la.backward()
    lb.backward()
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        assert p.grad is not None and torch.equal(p.grad, q.grad), n
    ka, kb = a.predict_step(dict(batch), 0), b.predict_step(dict(batch), 0)
    assert torch.equal(ka[0], kb[0]) and torch.equal(ka[1], kb[1])


def test_no_feature_sized_copy(tmp_path):
    """Forward and backward on channels-last features launch no copy kernel over a feature-sized tensor."""
    from torch.profiler import ProfilerActivity, profile

    head = HS.make_head(384, [17], 16)
    _, xc = _pair(8, 384, 16, 16, 17, BF16)
    xc.requires_grad_(True)
    gout = torch.randn(8, 17, 64, 64, device="cuda", generator=HS.gen(18))
    (head(xc) * gout).sum().backward()  # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        (head(xc) * gout).sum().backward()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(tmp_path / "channels_last_trace.json"))
    names = [e.name for e in prof.events()]
    assert any("rows_shuffle_nhwc_kernel" in n for n in names) and any("b3a_dgrad_kernel" in n for n in names)
    assert not any("rows_shuffle_kernel" in n for n in names)
    for e in prof.events():
        if e.name in ("aten::copy_", "aten::contiguous", "aten::clone") and e.input_shapes:
            assert list(e.input_shapes[0]) != list(xc.shape), (e.name, e.input_shapes)
