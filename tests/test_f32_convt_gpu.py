"""The fp32 head's tensor-core convolutions (3xTF32, head_f32.cu) against float64 on the device: each layer on its own
across keypoint counts, input channels and map sizes (odd sizes, widths above 256), whole heads on fp32 features at
keypoint counts past the old 28-channel limit, and a batch of several waves, which must also be batch-independent."""
import pytest
import torch
import torch.nn.functional as F

import scale_oracle as S
from head_support import F64, WORST, check_grads_f32, features, gen, head_params, make_head, ref_grads, report_headroom
COUT = [1, 8, 17, 20, 21, 28, 29, 51, 64, 81, 128]
CIN = [1, 3, 17, 51, 512]
SIZES = [(1, 1), (3, 5), (6, 8), (16, 24), (48, 48), (4, 300)]
# every (Cout, Cin) pair at one small map; every map size with a spread of channel pairs
CASES = [(co, ci, (6, 8), sh) for co in COUT for ci in CIN for sh in (False, True)]
CASES += [(co, ci, hw, sh) for hw in SIZES if hw != (6, 8) for (co, ci) in [(1, 1), (17, 512), (29, 17), (51, 51), (128, 3)]
          for sh in (False, True) if not sh or (hw[0] % 2 == 0 and hw[1] % 2 == 0)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


def _layer_ref(x, w, bias, shuffle):
    xi = F.pixel_shuffle(x, 2) if shuffle else x
    return F.conv_transpose2d(xi, w, bias, stride=2, padding=1, output_padding=1)


@pytest.mark.gpu
@pytest.mark.parametrize("cout,cin,hw,shuffle", CASES, ids=[f"o{c[0]}_c{c[1]}_{c[2][0]}x{c[2][1]}_{'ps' if c[3] else 'plain'}" for c in CASES])
def test_layer_against_float64(dev, cout, cin, hw, shuffle):
    from lightning_pose_b200 import ops

    hi, wi = hw
    b = 2
    x = torch.randn((b, 4 * cin, hi // 2, wi // 2) if shuffle else (b, cin, hi, wi), device=dev, generator=gen(cout * 131 + cin))
    w = torch.randn(cin, cout, 3, 3, device=dev, generator=gen(3)) / (cin * 2.25) ** 0.5
    bias = torch.randn(cout, device=dev, generator=gen(4))
    case = f"Cout={cout} Cin={cin} {hi}x{wi} shuffle={shuffle}"

    out = ops.convt_forward_f32(x, w, bias, shuffle)
    x64, w64, b64 = x.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True), bias.to(F64).requires_grad_(True)
    ref = _layer_ref(x64, w64, b64, shuffle)
    assert out.shape == ref.shape, case
    scale = ref.detach().abs().amax((0, 2, 3)).view(1, -1, 1, 1)
    ratio = float(((out.to(F64) - ref.detach()).abs() / (1e-5 * scale + 1e-30)).max())
    assert ratio < 1.0, (case, "forward", ratio)

    g = torch.randn(ref.shape, device=dev, generator=gen(5))
    dx, dw, db = ops.convt_backward_f32(x, g, w, shuffle)
    (ref * g.to(F64)).sum().backward()
    fscale = x64.grad.abs().flatten(1).amax(1).view(-1, *([1] * (x.dim() - 1)))
    ratio = float(((dx.to(F64) - x64.grad).abs() / (1e-5 * fscale + 1e-30)).max())
    assert ratio < 1.0, (case, "d input", ratio)
    check_grads_f32({"dw1": dw, "db1": db}, {"dw1": w64.grad, "db1": b64.grad}, {"db1": g.to(F64).pow(2).sum((0, 2, 3)).sqrt()}, case)


HEADS = {
    "mirror_fish_51": ((4, 2048, 8, 12), (51, 51)),
    "c512_29": ((3, 512, 8, 8), (29, 29)),
    "one_deconv_81": ((3, 384, 8, 8), (81,)),
    "odd_map_17": ((3, 512, 5, 7), (17, 17)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HEADS))
def test_head_fp32_features_train(dev, name):
    """forward_with_keypoints on fp32 features, backward from a dense heatmap gradient plus a keypoint gradient."""
    from lightning_pose_b200 import ops

    (b, c, h, w), ch = HEADS[name]
    head = make_head(c, ch, seed=31)
    deconvs, (ws, bs) = list(head.upsampling_layers)[1:], head_params(head)
    feats = features(b, c, h, w, 9, torch.float32)
    f = feats.clone().requires_grad_(True)
    hm, kp, _ = head.forward_with_keypoints(f)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, operands=None)
    err = (hm.detach().to(F64) - hm_ref).abs()
    assert bool((err <= 1e-4 * hm_ref + 1e-9).all()), (name, float((err / (1e-4 * hm_ref + 1e-9)).max()))

    g_dense = torch.randn(hm.shape, device=dev, generator=gen(10))
    g_kp = torch.randn(kp.shape, device=dev, generator=gen(11))
    ((hm * g_dense).sum() + (kp * g_kp).sum()).backward()
    k = hm.shape[1]
    _, _, stats = ops._decode_fwd(hm.detach(), 2, 1000.0)
    g_hm = g_dense + ops._decode_bwd(hm.detach(), stats, g_kp.reshape(b, k, 2).contiguous(), 2, 1000.0)
    ref, gnorm = ref_grads(feats, ws, bs, g_hm, True, hm_ref, operands=None)
    fscale = ref["dfeat"].abs().flatten(1).amax(1).view(-1, 1, 1, 1)
    ratio = float(((f.grad.to(F64) - ref["dfeat"]).abs() / (1e-4 * fscale + 1e-30)).max())
    assert ratio < 1.0, (name, "d features", ratio)
    got = {}
    for i, d in enumerate(deconvs, 1):
        got[f"dw{i}"], got[f"db{i}"] = d.weight.grad, d.bias.grad
    check_grads_f32(got, {kk: v for kk, v in ref.items() if kk != "dfeat"}, gnorm, name)


@pytest.mark.gpu
def test_head_fp32_several_waves_batch_independent(dev):
    """128 frames of a ResNet-50 head (forward: 640 CTAs, data gradients more) against float64, and each frame's
    heatmaps and d features bit-identical to the same frame run alone: neither has a cross-frame sum."""
    b, c, h, w = 128, 2048, 12, 12
    head = make_head(c, (17, 17), seed=41)
    deconvs, (ws, bs) = list(head.upsampling_layers)[1:], head_params(head)
    feats = features(b, c, h, w, 12, torch.float32)
    f = feats.clone().requires_grad_(True)
    hm = head(f)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, operands=None)
    err = (hm.detach().to(F64) - hm_ref).abs()
    assert bool((err <= 1e-4 * hm_ref + 1e-9).all()), float((err / (1e-4 * hm_ref + 1e-9)).max())
    gout = torch.randn(hm.shape, device=dev, generator=gen(13))
    (hm * gout).sum().backward()
    ref, gnorm = ref_grads(feats, ws, bs, gout, True, hm_ref, operands=None)
    fscale = ref["dfeat"].abs().flatten(1).amax(1).view(-1, 1, 1, 1)
    ratio = float(((f.grad.to(F64) - ref["dfeat"]).abs() / (1e-4 * fscale + 1e-30)).max())
    assert ratio < 1.0, ("d features", ratio)
    check_grads_f32({"dw1": deconvs[0].weight.grad, "db1": deconvs[0].bias.grad, "dw2": deconvs[1].weight.grad, "db2": deconvs[1].bias.grad},
                    {kk: v for kk, v in ref.items() if kk != "dfeat"}, gnorm, "128 frames")
    for i in (0, 77, b - 1):
        fi = feats[i : i + 1].clone().requires_grad_(True)
        hi = head(fi)
        assert torch.equal(hi.detach(), hm.detach()[i : i + 1]), i
        (hi * gout[i : i + 1]).sum().backward()
        assert torch.equal(fi.grad, f.grad[i : i + 1]), i
