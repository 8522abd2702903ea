"""Launches at the edges of the shared-memory launch rule (``set_dynamic_smem``, lpb_common.cuh): every launch with
dynamic shared memory sets its kernel's limit to the bytes it requests, and CUDA refuses that only when the kernel's
static plus dynamic memory passes the device's opt-in limit.

- Exactly 48 KiB of dynamic memory on kernels that also have static memory: the fp32 plane softmax on 12,288-pixel
  planes (what a 384 x 512 image gives a ResNet-50 head), and the unsupervised losses' forward.
- Between 200 KB (a former hand-written cap) and the device limit: the plane softmax forward and backward and
  ``upsample2x``.
- Past the device limit: LPB_ERR_UNSUPPORTED (-3) naming the entry, and the stream stays usable."""
import pytest
import torch

import scale_oracle as S
from head_support import F64, check_grads_f32, features, gen, head_params, make_head, ref_grads

pytestmark = pytest.mark.gpu

KIB = 1024
UNSUPPORTED = -3


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from lightning_pose_b200 import ops

    return ops


@pytest.fixture(scope="module")
def smem_limit():
    """The device's opt-in shared memory per block (static plus dynamic), bytes."""
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# the dynamic shared memory of each entry, restated from its launch
def softmax_fwd_bytes(hw):
    return hw * 4  # lpb_plane_softmax_f32: the plane


def softmax_bwd_bytes(hw):
    return 2 * hw * 4  # lpb_plane_softmax_bwd: the plane and its gradient


def upsample2x_bytes(h, w):
    pitch = (4 + w + 3 + 3) & ~3  # dec_pitch(w, 3) (decode.cu)
    return (h + 6) * pitch * 4


def unsup_fwd_bytes(t, n_sel, views, n_comp):
    """lpb_unsup_losses_fwd with one multi-view PCA loss: pca_scratch_floats (losses.cu) plus 4 floats."""
    rows = t * n_sel
    return (rows * 2 * views + rows * n_comp + 2 * t + 4) * 4


def softmax_ref(x):
    return torch.softmax(x.to(F64).flatten(2), -1).reshape(x.shape)


def check_softmax(out, x):
    ref = softmax_ref(x)
    err = (out.to(F64) - ref).abs()
    assert bool((err <= 1e-4 * ref + 1e-12).all()), float((err / (1e-4 * ref + 1e-12)).max())
    assert bool(((out.to(F64).sum((-1, -2)) - 1).abs() < 1e-5).all())


def check_softmax_bwd(out, p, g):
    """p (g - <p, g>) per plane; the error bound scales with what the kernel sums: p (|g| + <p, |g|>)."""
    p64, g64 = p.to(F64), g.to(F64)
    ref = p64 * (g64 - (p64 * g64).sum((-1, -2), keepdim=True))
    allowed = 1e-4 * p64 * (g64.abs() + (p64 * g64.abs()).sum((-1, -2), keepdim=True)) + 1e-15
    ratio = float(((out.to(F64) - ref).abs() / allowed).max())
    assert ratio < 1.0, ratio


def check_upsample2x(out, x):
    h, w = x.shape[-2:]
    uh, uw = S.upsample_op(h, 1, x.device), S.upsample_op(w, 1, x.device)
    ref = torch.einsum("ia,bkac,jc->bkij", uh, x.to(F64), uw)
    err = float((out.to(F64) - ref).abs().max())
    assert err <= 2e-6 * float(ref.abs().max()), err


def first_size_over(nbytes, limit, size_of):
    """The smallest n with size_of(n) above nbytes; it must still fit the device (static memory is at most 1 KB)."""
    n = 1
    while size_of(n) <= nbytes:
        n += 1
    assert size_of(n) <= limit - KIB, (n, size_of(n), limit)
    return n


# ------------------------------------------------------------------------------------------------
# exactly 48 KiB of dynamic memory beside static memory
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(96, 128), (64, 192)])
def test_plane_softmax_at_48_kib(ops, h, w):
    assert softmax_fwd_bytes(h * w) == 48 * KIB
    x = torch.randn(3, 5, h, w, device="cuda", generator=gen(1)) * 3
    out = ops.plane_softmax_(x.clone())
    check_softmax(out, x)


def test_fp32_head_at_96x128(ops):
    """A ResNet-50 head on fp32 features (B, 2048, 12, 16): two deconvs to 96 x 128 heatmaps, whose final softmax and its
    backward take 48 and 96 KiB of dynamic shared memory.  Forward, then backward from a dense heatmap gradient, against
    float64 at the fp32 rules."""
    b, c, h, w = 2, 2048, 12, 16
    head = make_head(c, (17, 17), seed=51)
    deconvs, (ws, bs) = list(head.upsampling_layers)[1:], head_params(head)
    feats = features(b, c, h, w, 52, torch.float32)
    f = feats.clone().requires_grad_(True)
    hm = head(f)
    assert hm.shape == (b, 17, 96, 128)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, operands=None)
    err = (hm.detach().to(F64) - hm_ref).abs()
    assert bool((err <= 1e-4 * hm_ref + 1e-9).all()), float((err / (1e-4 * hm_ref + 1e-9)).max())

    gout = torch.randn(hm.shape, device="cuda", generator=gen(53))
    (hm * gout).sum().backward()
    ref, gnorm = ref_grads(feats, ws, bs, gout, True, hm_ref, operands=None)
    fscale = ref["dfeat"].abs().flatten(1).amax(1).view(-1, 1, 1, 1)
    ratio = float(((f.grad.to(F64) - ref["dfeat"]).abs() / (1e-4 * fscale + 1e-30)).max())
    assert ratio < 1.0, ("d features", ratio)
    got = {}
    for i, d in enumerate(deconvs, 1):
        got[f"dw{i}"], got[f"db{i}"] = d.weight.grad, d.bias.grad
    check_grads_f32(got, {k: v for k, v in ref.items() if k != "dfeat"}, gnorm, "fp32 head 96x128")


def test_unsup_losses_at_48_kib(ops):
    """Multi-view PCA of 9 keypoints in 3 views, 3 components: the T whose forward scratch is exactly 48 KiB, against
    float64 forward and backward (the backward takes more, and opts in as before)."""
    n_sel, views, n_comp, n_clips = 9, 3, 3, 2
    t = next(t for t in range(1, 1000) if unsup_fwd_bytes(t, n_sel, views, n_comp) >= 48 * KIB)
    assert unsup_fwd_bytes(t, n_sel, views, n_comp) == 48 * KIB, t
    kk = views * n_sel
    g = gen(71)
    mcm = torch.arange(kk).reshape(views, n_sel)
    mean = torch.randn(2 * views, device="cuda", generator=g) * 50 + 150
    kept = torch.linalg.qr(torch.randn(2 * views, n_comp, device="cuda", generator=g))[0].T.contiguous()
    pts = torch.randn(n_clips, t, n_sel, n_comp, device="cuda", generator=g) * 40 @ kept + mean
    pts = pts + torch.randn(n_clips, t, n_sel, 2 * views, device="cuda", generator=g) * 3.0
    kp = pts.reshape(n_clips, t, n_sel, views, 2).permute(0, 1, 3, 2, 4).reshape(n_clips, t, 2 * kk).contiguous()
    conf = torch.rand(n_clips, t, kk, device="cuda", generator=g)
    mv = ops.PcaParams(mcm.reshape(-1).numpy().astype("int32"), n_sel, views, None, mean.cpu().numpy(), kept.cpu().numpy(), 2.0, "cuda")
    eps, thr = 4.0, 0.1
    wts = torch.rand(n_clips, 3, device="cuda", generator=g) + 0.5
    x = kp.clone().requires_grad_(True)
    out = ops.unsup_losses(x, conf, temporal_eps=eps, prob_threshold=thr, pca_multiview=mv)
    (out[:, :3] * wts).sum().backward()
    xr = kp.to(F64).requires_grad_(True)
    zero = torch.zeros((), dtype=F64, device="cuda")
    ref = torch.stack([torch.stack([S.temporal_loss_ref(xr[i], conf[i], eps, thr), zero,
                                    S.pca_multiview_ref(xr[i], mcm.tolist(), mv.mean, mv.kept, 2.0)]) for i in range(n_clips)])
    (ref * wts.to(F64)).sum().backward()
    err = (out[:, :3].detach().to(F64) - ref.detach()).abs()
    assert bool((err <= 1e-5 + 1e-4 * ref.detach().abs()).all()), err
    gerr = (x.grad.to(F64) - xr.grad).abs()
    assert bool((gerr <= 1e-6 * float(xr.grad.abs().max()) + 1e-3 * xr.grad.abs()).all()), float(gerr.max())


# ------------------------------------------------------------------------------------------------
# between the former 200 KB cap and the device limit
# ------------------------------------------------------------------------------------------------
def test_plane_softmax_above_200_kb(ops, smem_limit):
    hw = first_size_over(200 * KIB, smem_limit, softmax_fwd_bytes)
    x = torch.randn(2, 3, 1, hw, device="cuda", generator=gen(81)) * 3
    check_softmax(ops.plane_softmax_(x.clone()), x)


def test_plane_softmax_backward_above_200_kb(ops, smem_limit):
    hw = first_size_over(200 * KIB, smem_limit, softmax_bwd_bytes)
    p = softmax_ref(torch.randn(2, 3, 1, hw, device="cuda", generator=gen(82)) * 3).float()
    g = torch.randn(p.shape, device="cuda", generator=gen(83))
    check_softmax_bwd(ops.plane_softmax_backward(p, g), p, g)


def test_upsample2x_above_200_kb(ops, smem_limit):
    n = first_size_over(200 * KIB, smem_limit, lambda n: upsample2x_bytes(n, n))
    x = torch.rand(1, 2, n, n, device="cuda", generator=gen(84))
    check_upsample2x(ops.upsample2x(x), x)


# ------------------------------------------------------------------------------------------------
# past the device limit
# ------------------------------------------------------------------------------------------------
def test_refused_past_the_device_limit(ops, smem_limit):
    """Each entry refuses a plane past the limit with LPB_ERR_UNSUPPORTED and its name, queues nothing, and the next call
    on the same stream runs."""
    from lightning_pose_b200._lib import LpbError

    hw = first_size_over(smem_limit, 1 << 30, softmax_fwd_bytes)
    with pytest.raises(LpbError, match=f"error {UNSUPPORTED}: plane_softmax_f32: needs {softmax_fwd_bytes(hw)} B"):
        ops.plane_softmax_(torch.zeros(1, 1, 1, hw, device="cuda"))
    x = torch.randn(2, 2, 8, 12, device="cuda", generator=gen(91))
    check_softmax(ops.plane_softmax_(x.clone()), x)

    hw = first_size_over(smem_limit, 1 << 30, softmax_bwd_bytes)
    p = torch.full((1, 1, 1, hw), 1.0 / hw, device="cuda")
    with pytest.raises(LpbError, match=f"error {UNSUPPORTED}: plane_softmax_bwd: needs {softmax_bwd_bytes(hw)} B"):
        ops.plane_softmax_backward(p, p)
    p = softmax_ref(x).float()
    check_softmax_bwd(ops.plane_softmax_backward(p, x), p, x)

    n = first_size_over(smem_limit, 1 << 30, lambda n: upsample2x_bytes(n, n))
    with pytest.raises(LpbError, match=f"error {UNSUPPORTED}: upsample2x: needs {upsample2x_bytes(n, n)} B"):
        ops.upsample2x(torch.zeros(1, 1, n, n, device="cuda"))
    check_upsample2x(ops.upsample2x(x), x)
    torch.cuda.synchronize()
