"""GPU: the head's forward on fp16 features (``lpb_head_fwd_f16``), the inference route of ``precision="fp16"``.

Under ``torch.autocast(float16)`` the reference's backbone hands the head fp16 features and every ConvTranspose2d runs on
fp16 operands.  The fp16 forward is the bf16 forward's kernels instantiated on fp16 operands: the weights (and the bias
that rides on the constant-one channel) rounded to fp16 on the device, fp16 mid activations, fp32 accumulators and fp32
heatmaps.

Oracle A is float64 on exactly those roundings (``scale_oracle.head_ref`` with fp16 operands).  Its bars are the bf16
head's (1e-2 relative, at most 0.01 % of the pixels up to 3e-2) scaled by the unit-roundoff ratio 2^-11 / 2^-8 = 1/8 and
rounded up: 2e-3 relative, at most 0.01 % of the pixels up to 5e-3 (``head_support.BARS``).  The pixels allowed past 2e-3 are those fed by a mid activation that sits on an
fp16 rounding boundary and rounds the other way than in the oracle (fp32 summation order).  Oracle B is the reference's own
HeatmapHead and soft-argmax under autocast(float16), held to the reference's 1 px bar for swapping the compute behind a
forward."""
import ctypes

import pytest
import torch

import scale_oracle as S
from head_support import WORST, check_heatmaps, features, forward_checks, fwd_layout, head_params, make_head, report_headroom, softmax_split

F16 = torch.float16
pytestmark = pytest.mark.gpu

# (C, H, W, channels): fast path (cfg 2), banded two-deconv (cfg 5), one-deconv (cfgs 3 and 4), wide heads
ROWS = {
    "cfg2_c2048_12x12": (2048, 12, 12, (17, 17)),
    "cfg5_c2048_16x16": (2048, 16, 16, (17, 17)),
    "cfg3_1d_c384_16x16": (384, 16, 16, (17,)),
    "cfg4_1d_c384_24x24": (384, 24, 24, (17,)),
    "mirror_fish_c2048_8x12_k51": (2048, 8, 12, (51, 51)),
    "1d_c384_16x16_k51": (384, 16, 16, (51,)),
}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


def _lib():
    from lightning_pose_b200._lib import lib

    return lib


@pytest.mark.parametrize("row", list(ROWS))
def test_f16_forward_vs_oracle_a(dev, row):
    """Heatmaps (fused and split softmax), logits and decoded keypoints against oracle A."""
    c, h, w, ch = ROWS[row]
    head = make_head(c, ch, seed=13).requires_grad_(False).eval()
    forward_checks(head, features(8, c, h, w, 5, F16), row, splits=(1, 0, 2), train=False, keypoint_bar=0.1)


def test_f16_forward_past_one_wave(dev):
    """cfg 2 at B = 2 S + 7 (the persistent kernels run past one wave): oracle A, and with the fused softmax forced (a
    lone frame would otherwise take the split form) a frame alone gives the batch's bits."""
    c, h, w, ch = ROWS["cfg2_c2048_12x12"]
    b = 2 * torch.cuda.get_device_properties(dev).multi_processor_count + 7
    head = make_head(c, ch, seed=19).requires_grad_(False).eval()
    feats = features(b, c, h, w, 9, F16)
    ws, bs = head_params(head)
    with torch.no_grad(), softmax_split(_lib(), 0):
        out = head(feats)
        for i in (0, b // 2, b - 1):
            assert torch.equal(head(feats[i : i + 1])[0], out[i]), i
    check_heatmaps(out, S.head_ref_chunked(feats, ws, bs, True, operands=F16), f"cfg2 B={b}", dtype=F16)


def _pack_ref(w, bias, nst, ngroups):
    """The forward operand pack restated (head_bf16.cu head_prep_kernel): [group][stage][shift][kchunk][80][8] fp32 values."""
    cin, cout = w.shape[0], w.shape[1]
    out = torch.zeros(ngroups, nst, 4, 4, 80, 8, dtype=torch.float32, device=w.device)
    for grp in range(ngroups):
        for cls in range(4):
            py, px = cls >> 1, cls & 1
            for sh in range(4):
                dm, dn = sh >> 1, sh & 1
                if (py == 0 and dm == 1) or (px == 0 and dn == 1):
                    continue
                ky = 1 if py == 0 else (0 if dm else 2)
                kx = 1 if px == 0 else (0 if dn else 2)
                for ol in range(20):
                    o = 20 * grp + ol
                    if o >= cout:
                        continue
                    col = w[:, o, ky, kx]  # (cin,)
                    full = torch.zeros(nst * 32, device=w.device)
                    full[:cin] = col
                    out[grp, :, sh, :, cls * 20 + ol, :] = full.reshape(nst, 4, 8)
        if bias is not None:
            for ol in range(20):
                o = 20 * grp + ol
                if o < cout:
                    st, kc, e = cin // 32, (cin % 32) // 8, cin % 8
                    for cls in range(4):
                        out[grp, st, 0, kc, cls * 20 + ol, e] = bias[o]
    return out


def test_f16_packs_equal_torch_half(dev):
    """The packed w1 / w2 in the forward workspace are torch's .half() of the fp32 weights bit for bit: subnormal weights
    (xavier gain 0.01 puts many below 2^-14) and the second layer's bias included."""
    from lightning_pose_b200 import ops

    lib = _lib()
    b, c, h, w, c1, c2 = 2, 512, 8, 8, 17, 17
    head = make_head(c, (c1, c2), seed=3, gain=0.01).requires_grad_(False).eval()
    ws, bs = head_params(head)
    with torch.no_grad():
        ws[0][0, 0, 0, 0] = 3e-8        # fp16 subnormal
        ws[0][1, 0, 1, 1] = -6.0e-5     # just below the smallest normal
        ws[1][2, 3, 1, 1] = 1e-7
        bs[1].copy_(torch.linspace(-1e-6, 70000.0, c2))  # subnormals, normals and an overflow to inf
    assert bool((ws[0].abs() < 6.1e-5).any())
    feats = features(b, c, h, w, 5, F16)
    n = ctypes.c_size_t(0)
    assert lib.lpb_head_bf16_workspace_bytes(b, c, h, w, c1, c2, ctypes.byref(n)) == 0
    ws_buf = torch.zeros(n.value, dtype=torch.uint8, device=dev)
    out = torch.empty(b, c2, 8 * h, 8 * w, device=dev)
    rc = lib.lpb_head_fwd_f16(ctypes.c_void_p(feats.data_ptr()), b, c, h, w, ctypes.c_void_p(ws[0].data_ptr()), ctypes.c_void_p(bs[0].data_ptr()), c1,
                              ctypes.c_void_p(ws[1].data_ptr()), ctypes.c_void_p(bs[1].data_ptr()), c2, 0, ctypes.c_void_p(out.data_ptr()), None,
                              ctypes.c_void_p(ws_buf.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, lib.lpb_last_error()
    torch.cuda.synchronize()
    w1_at, w2_at = 0, fwd_layout(b, c, h, w, c1, c2).w2_at
    stage = 4 * 4 * 80 * 16
    nst1, nst2 = c // 128, 1
    got1 = ws_buf[w1_at : w1_at + nst1 * stage].view(torch.int16)
    got2 = ws_buf[w2_at : w2_at + nst2 * stage].view(torch.int16)
    want1 = _pack_ref(ws[0], None, nst1, 1).half().view(torch.int16).flatten()
    want2 = _pack_ref(ws[1], bs[1], nst2, 1).half().view(torch.int16).flatten()
    assert torch.equal(got1, want1)
    assert torch.equal(got2, want2)
    assert bool(torch.isinf(want2.view(torch.float16).float()).any())  # the overflowing bias is inf in both
    # the same heads through ops: the bf16 route packs bf16 of the same weights (the element type is all that differs)
    _, (_, fws) = ops._head_forward_bf16(feats.bfloat16(), ws, bs, False, train=True)
    assert torch.equal(fws[w1_at : w1_at + nst1 * stage].view(torch.int16), _pack_ref(ws[0], None, nst1, 1).bfloat16().view(torch.int16).flatten())


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages() if e.device_time_total > 0]


def test_f16_routing(dev):
    """No gradient: fp16 features run the tensor-core kernels' fp16 instantiations (k1a on cfg 2, the banded kernel on
    cfg 5).  With requires_grad they keep the fp32 route, bit-identical to head_forward_f32 on .float() features, and the
    backward runs."""
    from lightning_pose_b200 import ops

    for row, first in (("cfg2_c2048_12x12", "k1a_shuffle_convt_kernel<__half"), ("cfg5_c2048_16x16", "convt_rows_kernel<__half")):
        c, h, w, ch = ROWS[row]
        head = make_head(c, ch, seed=13).requires_grad_(False).eval()
        feats = features(4, c, h, w, 5, F16)
        with torch.no_grad():
            names = _kernel_names(lambda: head.forward_with_keypoints(feats))
        assert any(first in k for k in names), (row, names)
        assert any("convt_rows_kernel<__half" in k for k in names), (row, names)
        assert not any("__nv_bfloat16" in k or "convt3x3" in k for k in names), (row, names)
    c, h, w, ch = ROWS["cfg2_c2048_12x12"]
    head = make_head(c, ch, seed=13).eval()
    feats = features(4, c, h, w, 5, F16).requires_grad_(True)
    ws = [d.weight for d in list(head.upsampling_layers)[1:]]
    bs = [d.bias for d in list(head.upsampling_layers)[1:]]
    out = head(feats)
    ref = ops.head_forward_f32(feats.detach().float(), [x.detach() for x in ws], [x.detach() for x in bs], True)
    assert torch.equal(out.detach(), ref)
    out.pow(2).sum().backward()
    assert feats.grad is not None and feats.grad.dtype == torch.float16 and bool(torch.isfinite(feats.grad).all())
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in ws + bs)


def test_f16_graph_replay_equals_eager(dev):
    """A captured CUDA graph of fp16 head + decode replays the eager bits."""
    c, h, w, ch = ROWS["cfg5_c2048_16x16"]
    head = make_head(c, ch, seed=7).requires_grad_(False).eval()
    feats = features(16, c, h, w, 8, F16)
    static = feats.clone()
    with torch.no_grad():
        eager = head.forward_with_keypoints(feats)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            head.forward_with_keypoints(static)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs = head.forward_with_keypoints(static)
        static.copy_(features(16, c, h, w, 99, F16))
        g.replay()
        static.copy_(feats)
        g.replay()
        torch.cuda.synchronize()
    for a, e in zip(outs, eager):
        assert torch.equal(a, e)


def test_f16_context_head_vs_oracle_a(dev):
    """HeatmapMHCRNNHead.forward_sequence on fp16 features: the single-frame heatmaps are oracle A's, and the context
    heatmaps are the fp32 context combine of oracle A's W_f / W_b logits."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    torch.manual_seed(21)
    c, h, w, k, t = 2048, 8, 8, 17, 9
    head = HeatmapMHCRNNHead("resnet50", c, k).cuda().eval().requires_grad_(False)
    for m in head.modules():
        if isinstance(m, torch.nn.ConvTranspose2d) and m.weight.shape[-1] == 3:
            torch.nn.init.xavier_uniform_(m.weight, gain=3.0)
            torch.nn.init.uniform_(m.bias, -0.3, 0.3)
    feats = features(t, c, h, w, 22, F16)
    with torch.no_grad():
        hm_sf, hm_mf = head.forward_sequence(feats)
    ws, bs = head_params(head.head_sf)
    check_heatmaps(hm_sf, S.head_ref_chunked(feats[2 : t - 2], ws, bs, True, operands=F16), "context head_sf", dtype=F16)
    mf = head.head_mf
    maps = []
    for last in (mf.W_f, mf.W_b):
        layers = ([mf.W_pre] if mf.upsampling_factor == 2 else []) + [last]
        maps.append(S.head_ref_chunked(feats, [m.weight for m in layers], [m.bias for m in layers], False, operands=F16).float())
    idx = (torch.arange(t - 4, device=dev)[:, None] + torch.arange(5, device=dev)[None, :]).to(torch.int32)
    hf = (mf.H_f[0].weight, mf.H_f[0].bias, mf.H_f[1].weight, mf.H_f[1].bias)
    hb = (mf.H_b[0].weight, mf.H_b[0].bias, mf.H_b[1].weight, mf.H_b[1].bias)
    with torch.no_grad():
        ref = ops.plane_softmax(ops.crnn_combine(maps[0], maps[1], idx, hf, hb))
    check_heatmaps(hm_mf, ref, "context head_mf", dtype=F16)


def test_f16_vs_reference_under_autocast(dev):
    """Oracle B: the reference's own HeatmapHead layers under torch.autocast("cuda", float16) on the same fp16 features
    and weights, then the reference's spatial softmax and run_subpixelmaxima in fp32 (as autocast runs the softmax; the
    kornia functions they call are restated with CPU constants, so they run on the CPU).  Keypoints agree within 1 px on
    confident keypoints (the reference's bar for swapping the compute behind forward); the largest difference is
    printed."""
    from oracle import ref_loader as R

    if not R.reference_available():
        pytest.skip("the reference's staged copy (oracle/_ref, made by build()) is absent")
    R.install()
    ref_mod = R.load("lightning_pose.models.heads.heatmap")
    c, h, w, ch = ROWS["cfg2_c2048_12x12"]
    head = make_head(c, ch, seed=29, gain=4.0).requires_grad_(False).eval()
    ref_head = ref_mod.HeatmapHead("resnet50", c, ch[1], deconv_out_channels=ch[0]).cuda().eval()
    ref_head.load_state_dict(head.state_dict())
    feats = features(16, c, h, w, 30, F16)
    with torch.no_grad():
        hm, kp, cf = head.forward_with_keypoints(feats)
        with torch.autocast("cuda", dtype=torch.float16):
            logits_r = ref_head.upsampling_layers(feats)
        assert logits_r.dtype == torch.float16
        hm_r = ref_mod.spatial_softmax2d(logits_r.float().cpu(), temperature=torch.tensor([1.0]))
        kp_r, cf_r = ref_mod.run_subpixelmaxima(hm_r, ref_head.downsample_factor, ref_head.temperature)
    kp, cf = kp.cpu(), cf.cpu()
    d = (kp.float() - kp_r.float()).abs().reshape(-1, ch[1], 2).amax(-1)
    conf = cf_r.float() > 0.5
    worst = float(d[conf].max()) if bool(conf.any()) else 0.0
    print(f"oracle B (reference under autocast fp16): max keypoint difference {worst:.4f} px over {int(conf.sum())} confident keypoints")
    assert bool(conf.any())
    assert worst < 1.0
