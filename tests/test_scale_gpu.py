"""The persistent kernels past one wave: production batch sizes against the float64 references of tests/scale_oracle.py.

Most of the hot path runs as persistent launches whose grid is capped at the SM count S (or S x residency); each CTA
loops over frames, (frame, tile-group) pairs, planes or queued plane parts, and its barrier phases, ring slots and
shared-memory buffers carry over from one item to the next.  Every test below picks its batch from the grid formula of
the launch it exercises (restated in the ``*_launches`` helpers) and asserts that some CTA gets two or more items, so a
later change to a launch's item count cannot quietly drop the test back to one item per CTA.  S is read from the
device (H100 SXM: 132, PCIe: 114)."""
import contextlib
import ctypes

import pytest
import torch

import scale_oracle as S

pytestmark = pytest.mark.gpu

F64 = torch.float64
K = 17


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


@pytest.fixture(scope="module")
def lib(lpb):
    from lightning_pose_b200._lib import lib

    return lib


@pytest.fixture(scope="module")
def props(dev):
    return torch.cuda.get_device_properties(dev)


@pytest.fixture(scope="module")
def sms(props):
    return props.multi_processor_count


def items_per_cta(items: int, grid: int) -> int:
    """Largest number of work items one CTA of a persistent launch (CTA i takes items i, i + grid, ...) loops over."""
    return -(-items // max(1, grid))


def assert_some_cta_loops(launches, at_least=2):
    """``launches``: (name, items, grid) of the launches a call makes; at least one must give a CTA ``at_least`` items."""
    assert any(items_per_cta(n, g) >= at_least for _, n, g in launches), launches


@contextlib.contextmanager
def tuning(lib, settings: dict):
    saved = {k: lib.lpb_get_tuning(k) for k in settings}
    try:
        for k, v in settings.items():
            assert lib.lpb_set_tuning(k, v) == 0
        yield
    finally:
        for k, v in saved.items():
            lib.lpb_set_tuning(k, v)


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def close(a, b, atol, rtol):
    a, b = a.detach().to(F64), b.detach().to(F64)
    err = (a - b).abs()
    bad = ~(err <= atol + rtol * b.abs()) & ~(torch.isnan(a) & torch.isnan(b))
    assert not bool(bad.any()), f"{int(bad.sum())} of {b.numel()} differ; worst {float(err[bad].max())} (atol {atol}, rtol {rtol})"


# ------------------------------------------------------------------------------------------------
# a / b: the bf16 tensor-core head
# ------------------------------------------------------------------------------------------------
# BASELINE configs 2 (ResNet-50 384^2: k1a + banded softmax), 3 (ViT-S 256^2: one deconv, banded) and 5 (ResNet-50 512^2:
# banded mid + banded softmax)
HEAD_CFGS = {"cfg2": ("resnet50", 2048, 12, 12), "cfg3": ("vits_dino", 384, 16, 16), "cfg5": ("resnet50", 2048, 16, 16)}
B_KINDS = {"S-1": lambda s: s - 1, "S": lambda s: s, "S+1": lambda s: s + 1, "2S+7": lambda s: 2 * s + 7}


def _head_fwd_launches(cfg, b, s, split_key):
    """(name, items, grid) of the persistent launches of lpb_head_fwd_bf16 (head_bf16.cu:931-932,
    head_rows_bf16.cu:437-470)."""
    arch, _, h, w = HEAD_CFGS[cfg]

    def banded(hi, wi, mode):
        r = min(256 // (wi + 1), hi)  # image rows per band: CR_TILES * 128 / (Wi + 1)
        nbands = -(-hi // r)
        if mode == "softmax" and not (split_key == 2 or (split_key == 1 and b < s)):
            return ("banded, fused two-pass softmax (one frame per item)", b, min(b, s))
        return (f"banded {mode} (one (frame, band) per item)", b * nbands, min(b * nbands, s))

    if cfg == "cfg2":
        ntg = -(-(-(-(2 * h * (2 * w + 1)) // 128)) // 2)  # (frame, group of two 128-row M-tiles) items
        return [("k1a", b * ntg, min(b * ntg, s)), banded(4 * h, 4 * w, "softmax")]
    if cfg == "cfg3":
        return [banded(2 * h, 2 * w, "softmax")]
    return [banded(2 * h, 2 * w, "mid"), banded(4 * h, 4 * w, "softmax")]


def _head_bwd_launches(cfg, b, s):
    """(name, items, grid) of the frame loops of lpb_head_bwd_bf16 (head_bwd_bf16.cu:1049-1051, :1091-1096)."""
    _, c, _, _ = HEAD_CFGS[cfg]
    ntile1 = -(-(c // 4) // 128)
    slots = max(1, min(s // ntile1, b))
    out = [("b3a dgrad (frames per slot)", b, slots)]
    if cfg != "cfg3":
        out.append(("b2d dgrad", b, min(b, 2 * s, 264)))  # B2D_MAX_CTAS
    return out


def _rand_head(arch, cin, gain=3.0, seed=13, final_softmax=True):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(seed)
    head = HeatmapHead(arch, cin, K, final_softmax=final_softmax)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=gain)
        torch.nn.init.uniform_(layer.bias, -0.3, 0.3)
    return head


def _head_params(head):
    deconvs = list(head.upsampling_layers)[1:]
    return [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs]


def _feats(cfg, b, dev, seed=5, scale=0.5):
    _, c, h, w = HEAD_CFGS[cfg]
    return (torch.randn(b, c, h, w, device=dev, generator=_gen(seed)) * scale).bfloat16()


def _check_heatmaps(out, ref_hm):
    """Acceptance rule of the bf16 head (test_head_bf16_real_config_shapes_forward): relative error below 3e-2 everywhere,
    above 1e-2 on at most 0.01 % of the pixels (a mid activation on a bf16 rounding boundary may round the other way);
    every plane sums to 1."""
    rel = ((out.to(F64) - ref_hm).abs() / (ref_hm.abs() + 1e-7)).flatten()
    assert float(rel.max()) < 3e-2 and float((rel > 1e-2).to(F64).mean()) < 1e-4, (float(rel.max()), float((rel > 1e-2).to(F64).mean()))
    sums = out.sum((2, 3))
    assert float((sums - 1).abs().max()) <= 1e-5


@pytest.mark.parametrize("bkind", list(B_KINDS))
@pytest.mark.parametrize("cfg", list(HEAD_CFGS))
def test_head_forward_past_one_wave(lpb, lib, dev, sms, cfg, bkind):
    arch, c, h, w = HEAD_CFGS[cfg]
    b = B_KINDS[bkind](sms)
    two = arch == "resnet50"
    launches = _head_fwd_launches(cfg, b, sms, lib.lpb_get_tuning(7))
    if cfg == "cfg3" and bkind == "S":  # the boundary itself: one launch, exactly one frame per CTA
        assert [items_per_cta(n, g) for _, n, g in launches] == [1]
    else:
        assert_some_cta_loops(launches)
    plan = ctypes.c_int(-1)
    assert lib.lpb_head_bf16_plan(c, h, w, K, K if two else 0, ctypes.byref(plan)) == 0
    assert plan.value == (1 if cfg == "cfg2" else 0)  # which kernels the launches above describe
    head = _rand_head(arch, c).to(dev)
    feats = _feats(cfg, 2 * sms + 7, dev)[:b]
    ws, bs = _head_params(head)
    logits_ref = S.head_ref_chunked(feats, ws, bs, softmax=False)
    hm_ref = torch.softmax(logits_ref.flatten(2), -1).reshape(logits_ref.shape)
    with torch.no_grad():
        out = head(feats)
    assert out.dtype == torch.float32 and out.shape == hm_ref.shape
    _check_heatmaps(out, hm_ref)
    del hm_ref
    head.final_softmax = False
    with torch.no_grad():
        lg = head(feats)
    close(lg, logits_ref, atol=1e-2 * float(logits_ref.abs().max()), rtol=1e-2)
    del lg, logits_ref
    # the training route (saved operand copy, inter-layer activations kept) computes the same bits
    head.final_softmax = True
    out_train = head(feats.clone().requires_grad_(True))
    assert torch.equal(out_train.detach(), out)
    del out_train
    if bkind != "2S+7":
        return
    # a permutation moves every frame to another CTA and another loop iteration: the outputs permute exactly
    perm = torch.randperm(b, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        assert torch.equal(head(feats[perm]), out[perm])
    # with the fused softmax pinned (key 7 = 0: no split at any batch), a frame computes the same bits in a batch of one
    with tuning(lib, {7: 0}):
        with torch.no_grad():
            big = head(feats)
            assert torch.equal(big, out)  # at B >= S the default never splits either
            for i in (0, sms - 1, sms, sms + 1, b - 1):
                assert torch.equal(head(feats[i : i + 1])[0], big[i]), i


def _grads(head, feats, gout):
    head.zero_grad(set_to_none=True)
    f = feats.clone().requires_grad_(True)
    (head(f) * gout).sum().backward()
    return [f.grad.clone()] + [p.grad.clone() for p in head.parameters()]


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_head_backward_past_one_wave(lpb, dev, sms, cfg):
    arch, c, h, w = HEAD_CFGS[cfg]
    b = 2 * sms + 7
    assert_some_cta_loops(_head_bwd_launches(cfg, b, sms))
    head = _rand_head(arch, c, seed=31).to(dev)
    feats = _feats(cfg, b, dev, seed=6)
    up = 8 if arch == "resnet50" else 4
    gout = torch.randn(b, K, up * h, up * w, device=dev, generator=_gen(7))
    run1 = _grads(head, feats, gout)
    run2 = _grads(head, feats, gout)
    for x, y in zip(run1, run2):  # fixed-order sums: bit-reproducible at this batch
        assert torch.equal(x, y)
    assert run1[0].dtype == torch.bfloat16
    perm = torch.randperm(b, generator=torch.Generator().manual_seed(2)).to(dev)
    assert torch.equal(_grads(head, feats[perm], gout[perm])[0], run1[0][perm])
    ws, bs = _head_params(head)
    dfeat, dws, dbs = S.head_grad_ref(feats, ws, bs, gout, softmax=True)
    deconvs = list(head.upsampling_layers)[1:]
    got = {"dfeat": run1[0]}
    for i, d in enumerate(deconvs):
        got[f"dw{i}"], got[f"db{i}"] = d.weight.grad, d.bias.grad
    ref = {"dfeat": dfeat, **{f"dw{i}": g for i, g in enumerate(dws)}, **{f"db{i}": g for i, g in enumerate(dbs)}}
    wscale = float(dws[-1].abs().max())
    for name in ref:
        err, scale = float((got[name].to(F64) - ref[name]).abs().max()), float(ref[name].abs().max())
        if name.startswith("db"):  # cancelling sums (exactly 0 behind a softmax): rounding noise, bounded by the dw scale
            scale = max(scale, wscale)
        assert err <= 1e-2 * scale + 1e-9, (name, err, scale)


def test_head_with_keypoints_past_one_wave(lpb, dev, sms):
    """forward_with_keypoints at config 2, B = 2S + 7, with three frames of all-zero features: their 51 diffuse planes
    overflow the 32 x 32 decode windows into the dense backward route."""
    arch, c, h, w = HEAD_CFGS["cfg2"]
    b = 2 * sms + 7
    head = _rand_head(arch, c, gain=4.0, seed=31).to(dev)
    feats = _feats("cfg2", b, dev, seed=8)
    flat_frames = [5, sms, b - 3]
    feats[flat_frames] = 0
    g_kp = torch.randn(b, 2 * K, device=dev, generator=_gen(9))
    f = feats.clone().requires_grad_(True)
    hm, kp, cf = head.forward_with_keypoints(f)
    (kp * g_kp).sum().backward()
    hm = hm.detach()
    # the windows of these heatmaps: every plane of the flat frames overflows (dense queue route)
    _, _, stats = lpb._decode_fwd(hm, 2, 1000.0)
    _, meta, _ = lpb.decode_backward_windows(hm, stats, g_kp.reshape(b, K, 2).contiguous(), 2, 1000.0)
    flags = meta[:, 2].reshape(b, K)
    assert bool((flags[flat_frames] == 2).all()) and int((flags == 2).sum()) >= 3 * K
    preds, _, _, conf_alt = S.decode_ref(hm, 2, 1000.0)
    close(kp, preds, atol=2e-3, rtol=1e-4)
    cerr = (cf.to(F64)[..., None] - conf_alt).abs().amin(-1)
    assert float(cerr.max()) <= 1e-4, float(cerr.max())
    # the fused backward against float64 autograd: the soft-argmax gradient taken at the kernel's heatmaps, then the head
    g_hm = S.decode_grad_ref(hm, 2, 1000.0, g_kp)
    ws, bs = _head_params(head)
    dfeat, dws, dbs, mid_norm = S.head_grad_ref(feats, ws, bs, g_hm, softmax=True, want_mid_grad=True)
    d1, d2 = list(head.upsampling_layers)[1:]
    # db1 only sees the image border and is left as rounding noise of the bf16 gradient operand, 2^-8 ||d mid||_2 per
    # channel (test_head_with_keypoints_fused_backward_vs_oracle); db2 is exactly 0: bounded by the dw2 scale
    err = (d1.bias.grad.to(F64) - dbs[0]).abs()
    assert bool((err <= 2e-2 * dbs[0].abs().max() + 4.0 * 2.0**-8 * mid_norm).all()), (err, mid_norm)
    for name, got, ref, scale in [("dfeat", f.grad, dfeat, None), ("dw1", d1.weight.grad, dws[0], None), ("dw2", d2.weight.grad, dws[1], None),
                                  ("db2", d2.bias.grad, dbs[1], float(dws[1].abs().max()))]:
        scale = float(ref.abs().max()) if scale is None else scale
        e = float((got.to(F64) - ref).abs().max())
        assert e <= 2e-2 * scale + 1e-9, (name, e, scale)


# ------------------------------------------------------------------------------------------------
# c / d: the soft-argmax decode
# ------------------------------------------------------------------------------------------------
DECODE_SIZES = {"64_ds2": (64, 2), "96_ds2": (96, 2), "96_ds3": (96, 3), "128_ds2": (128, 2), "90_ds2": (90, 2)}  # 90: w % 4 != 0
MIXES = ["peaked", "one_diffuse", "half_S_diffuse", "over_resident_diffuse", "all_diffuse"]


def _resident_bound(props, sms):
    """decode_fwd_kernel has 256 threads: at most max_threads_per_SM / 256 resident CTAs per SM (decode.cu:1160)."""
    return sms * (props.max_threads_per_multi_processor // 256)


def _smem_planes(props, hw):
    """Whole hw x hw fp32 planes that fit in one CTA's shared memory beside four 32 x 33 windows, at most 8."""
    tiles_b = (4 * 32 * 33 * 4 + 127) & ~127
    return min(8, (props.shared_memory_per_block_optin - tiles_b - 256) // (hw * hw * 4))


def _n_planes(props, sms, hw):
    """(2 _smem_planes + 1) planes per SM, and more planes than the CTA kernel has resident CTAs."""
    n = max((2 * _smem_planes(props, hw) + 1) * sms, _resident_bound(props, sms) + 2 * sms) + 5
    return -(-n // K) * K


def _n_diffuse(mix, n, props, sms):
    return {"peaked": 0, "one_diffuse": 1, "half_S_diffuse": sms // 2, "over_resident_diffuse": _resident_bound(props, sms) + sms // 2,
            "all_diffuse": n}[mix]


def _decode_inputs(n, hw, n_diffuse, seed):
    """(B, 17, hw, hw) heatmaps: peaked planes (random centres, sigma 1.6, 5 % logit noise) with ``n_diffuse`` planes at
    random positions replaced by diffuse ones (logit noise 0.01, the bench's untrained regime); and the diffuse mask."""
    b = -(-n // K)
    g = _gen(seed)
    dev = torch.device("cuda")
    cy = torch.rand(b * K, 1, 1, device=dev, generator=g) * (hw - 1)
    cx = torch.rand(b * K, 1, 1, device=dev, generator=g) * (hw - 1)
    yy = torch.arange(hw, device=dev).view(1, hw, 1).float()
    xx = torch.arange(hw, device=dev).view(1, 1, hw).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * 1.6**2) + 0.05 * torch.randn(b * K, hw, hw, device=dev, generator=g)
    diffuse = torch.zeros(b * K, dtype=torch.bool, device=dev)
    diffuse[torch.randperm(b * K, device=dev, generator=g)[: min(n_diffuse, b * K)]] = True
    logits[diffuse] = 0.01 * torch.randn(int(diffuse.sum()), hw, hw, device=dev, generator=g)
    hm = torch.softmax(logits.reshape(b * K, -1), -1).reshape(b, K, hw, hw).contiguous()
    return hm, diffuse


def _decode_route(lpb, hm, ds, route):
    """"queue": the warp kernel, its leftovers queued for the CTA kernel.  "unaligned": the same planes 4 bytes into their
    storage, so that the warp kernel reads them with scalar loads and the CTA kernel stages queued planes with plain
    loads (as for any plane with w % 4 != 0)."""
    return lpb._decode_fwd(hm if route == "queue" else _misaligned(hm), ds, 1000.0)


def _decode_fwd_launches(n, q, resident_bound, sms):
    """(name, items, grid) of the persistent decode launch (decode.cu launch_decode_fwd), q = planes the warp kernel
    leaves for the CTA kernel.  The CTA kernel's grid is min(n, resident) <= min(n, resident_bound): the item counts per
    CTA derived here are lower bounds."""
    np_ = min(16, max(1, sms // q))  # queued plane split over NP CTAs (decode.cu:273; grid >= S)
    return [("CTA kernel, queued plane parts", q * np_, min(q * np_, resident_bound))]


def _check_decode(xy, conf, ref, diffuse, where=None):
    """preds within 1e-4 (peaked) / 5e-4 (diffuse) + 1e-4 relative, as test_decode_vs_oracle_shapes / golden regimes;
    confidence within 2e-6 (+1e-4 relative) of the window at trunc() of the reference coordinates -- or of the window on
    the other side of an integer that a coordinate lies within 1e-3 px of (trunc rule)."""
    preds, _, _, conf_alt = ref
    n = diffuse.numel()
    xy, conf = xy.reshape(n, 2).to(F64), conf.reshape(n).to(F64)
    pr, alt = preds.reshape(n, 2), conf_alt.reshape(n, 9)
    keep = torch.ones(n, dtype=torch.bool, device=xy.device) if where is None else where
    tol = torch.where(diffuse, 5e-4, 1e-4)[:, None] + 1e-4 * pr.abs()
    bad = ((xy - pr).abs() > tol).any(-1) & keep
    assert not bool(bad.any()), f"{int(bad.sum())} planes off, worst {float(((xy - pr).abs() - tol).amax(-1)[bad].max())} px past tolerance"
    cerr = ((conf[:, None] - alt).abs() - (2e-6 + 1e-4 * alt.abs())).amin(-1)
    bad = (cerr > 0) & keep
    assert not bool(bad.any()), f"{int(bad.sum())} confidences off, worst {float(cerr[bad].max())} past tolerance"


SIZE_MIX = [(s, m) for s in DECODE_SIZES for m in MIXES] + [("bench_96_ds2", "half_S_diffuse"), ("bench_96_ds2", "all_diffuse")]
DECODE_ROUTES = ["queue", "unaligned"]


@pytest.mark.parametrize("route", DECODE_ROUTES)
@pytest.mark.parametrize("size,mix", SIZE_MIX)
def test_decode_forward_past_one_wave(lpb, props, sms, size, mix, route):
    hw, ds = DECODE_SIZES.get(size, (96, 2))
    n = 768 * K if size.startswith("bench") else _n_planes(props, sms, hw)
    nd = _n_diffuse(mix, n, props, sms)
    hm, diffuse = _decode_inputs(n, hw, nd, seed=hw + ds)
    n = diffuse.numel()
    res = _resident_bound(props, sms)
    q = int(diffuse.sum())  # planes the warp kernel leaves for the queue
    if mix == "half_S_diffuse":
        assert min(16, sms // q) >= 2  # each queued plane is split over NP > 1 CTAs
    if mix in ("over_resident_diffuse", "all_diffuse"):  # the other mixes give a CTA at most one queued plane part
        assert q > res  # NP = 1 and several queued planes per CTA
        assert_some_cta_loops(_decode_fwd_launches(n, q, res, sms))
    ref = S.decode_ref(hm, ds, 1000.0)
    out = _decode_route(lpb, hm, ds, route)
    _check_decode(out[0], out[1], ref, diffuse)
    # the default route again: queue mode (atomic work counters, merges of split planes) is bit-reproducible, and the
    # scalar loads of the unaligned route read the same values in the same 4-column groups as the 16-byte ones
    for x, y in zip(out, lpb._decode_fwd(hm, ds, 1000.0)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("route", DECODE_ROUTES)
@pytest.mark.parametrize("size", list(DECODE_SIZES))
def test_decode_forward_nan_planes(lpb, props, sms, size, route):
    """A few NaN planes among peaked ones (the "peaked" input of test_decode_forward_past_one_wave): their keypoints are
    NaN, and every other plane is bit-identical to the run with the NaN planes replaced by their peaked originals.
    (A single NaN pixel away from a peak is not propagated: the peaked-plane route never reads it; DESIGN.md K2.)"""
    hw, ds = DECODE_SIZES[size]
    n = _n_planes(props, sms, hw)
    base, _ = _decode_inputs(n, hw, 0, seed=hw + ds)
    flat = base.reshape(-1, hw, hw)
    m = flat.shape[0]
    nan_planes = [3, m // 2, m - 1]
    bad = flat.clone()
    bad[nan_planes] = float("nan")
    bad = bad.reshape(base.shape)
    others = torch.ones(m, dtype=torch.bool, device=base.device)
    others[nan_planes] = False
    xy0, c0, _ = _decode_route(lpb, base, ds, route)
    xy1, c1, _ = _decode_route(lpb, bad, ds, route)
    xy0, xy1 = xy0.reshape(m, 2), xy1.reshape(m, 2)
    assert bool(torch.isnan(xy1[nan_planes]).all()), xy1[nan_planes]
    assert torch.equal(xy1[others], xy0[others]) and torch.equal(c1.reshape(m)[others], c0.reshape(m)[others])


def _rebuild_windows(win, meta, ov, h, w):
    """Dense gradient planes from lpb_decode_bwd_windows' output (as test_decode_backward_windows_match_dense): flag 1 ->
    the 32 x 32 window at (r0, c0), flag 2 -> the overflow plane, flag 0 -> zero; nothing of a window may fall outside."""
    n = meta.shape[0]
    m = meta.long()
    pad = torch.zeros(n, h + 64, w + 64, device=win.device)
    pl = (m[:, 2] == 1).nonzero()[:, 0]
    assert bool(((m[pl, 0] >= -32) & (m[pl, 0] <= h) & (m[pl, 1] >= -32) & (m[pl, 1] <= w)).all())
    ar = torch.arange(32, device=win.device)
    rows = (m[pl, 0] + 32)[:, None, None] + ar[None, :, None]
    cols = (m[pl, 1] + 32)[:, None, None] + ar[None, None, :]
    pad[pl[:, None, None], rows, cols] = win[pl]
    inner = pad[:, 32 : 32 + h, 32 : 32 + w].clone()
    pad[:, 32 : 32 + h, 32 : 32 + w] = 0.0
    assert float(pad.abs().max()) == 0.0
    two = m[:, 2] == 2
    inner[two] = ov.reshape(n, h, w)[two]
    return inner, m[:, 2]


def _check_plane_grads(got, ref):
    """2e-3 of each plane's max |ref| (test_decode_backward_vs_autograd)."""
    n = ref.shape[0] * ref.shape[1]
    got, ref = got.reshape(n, -1).to(F64), ref.reshape(n, -1)
    err = (got - ref).abs().amax(-1)
    lim = 2e-3 * ref.abs().amax(-1) + 1e-12
    bad = err > lim
    assert not bool(bad.any()), f"{int(bad.sum())} planes off, worst ratio {float((err / lim).max())}"


@pytest.mark.parametrize("mix", MIXES[1:])
@pytest.mark.parametrize("size", list(DECODE_SIZES))
def test_decode_backward_past_one_wave(lpb, props, sms, size, mix):
    hw, ds = DECODE_SIZES[size]
    n = _n_planes(props, sms, hw)
    hm, diffuse = _decode_inputs(n, hw, _n_diffuse(mix, n, props, sms), seed=hw + ds + 1)
    b = hm.shape[0]
    _, _, stats = lpb._decode_fwd(hm, ds, 1000.0)
    gxy = torch.randn(b, K, 2, device=hm.device, generator=_gen(ds))
    ref = S.decode_grad_ref(hm, ds, 1000.0, gxy)
    _check_plane_grads(lpb._decode_bwd(hm, stats, gxy, ds, 1000.0), ref)
    win, meta, ov = lpb.decode_backward_windows(hm, stats, gxy, ds, 1000.0)
    rebuilt, flags = _rebuild_windows(win, meta, ov, hw, hw)
    assert bool((flags[diffuse] == 2).all())  # diffuse planes overflow their window into the dense queue route
    q = int((flags == 2).sum())
    if mix in ("over_resident_diffuse", "all_diffuse"):  # dense backward in queue mode: grid min(n, 2S) (decode.cu:1193-1194)
        assert_some_cta_loops([("dense backward, queued planes", q, min(b * K, 2 * sms))])
    _check_plane_grads(rebuilt.reshape(ref.shape), ref)


# ------------------------------------------------------------------------------------------------
# e: losses and the CRNN combine
# ------------------------------------------------------------------------------------------------
def _peaked_planes(b, k, h, w, seed, sigma=1.6):
    g = _gen(seed)
    dev = torch.device("cuda")
    cy = torch.rand(b, k, 1, 1, device=dev, generator=g) * (h - 1)
    cx = torch.rand(b, k, 1, 1, device=dev, generator=g) * (w - 1)
    yy = torch.arange(h, device=dev).view(1, 1, h, 1).float()
    xx = torch.arange(w, device=dev).view(1, 1, 1, w).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sigma**2) + 0.05 * torch.randn(b, k, h, w, device=dev, generator=g)
    return torch.softmax(logits.reshape(b, k, -1), -1).reshape(b, k, h, w)


def _misaligned(x):
    """A contiguous copy of x starting 4 bytes into its storage (fails the kernels' 16-byte alignment check)."""
    buf = torch.empty(x.numel() + 1, device=x.device, dtype=x.dtype)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


@pytest.mark.parametrize("layout", ["bench_768x17_96x96", "odd_30x41", "misaligned_96x96"])
@pytest.mark.parametrize("kind", ["mse", "kl", "js"])
def test_heatmap_losses_at_scale(lpb, dev, kind, layout):
    """HeatmapMSE/KL/JS forward + backward with about 10 % all-zero targets; the odd plane (hw % 4 != 0) and the
    misaligned views take the scalar loop of heatmap_loss_plane_kernel (losses.cu:61-67), the bench batch the float4 one."""
    b, h, w = {"bench_768x17_96x96": (768, 96, 96), "odd_30x41": (64, 30, 41), "misaligned_96x96": (32, 96, 96)}[layout]
    targ = _peaked_planes(b, K, h, w, seed=11)
    targ[torch.rand(b, K, device=dev, generator=_gen(12)) < 0.1] = 0.0
    pred = _peaked_planes(b, K, h, w, seed=13, sigma=2.5)
    if layout.startswith("misaligned"):
        targ, pred = _misaligned(targ), _misaligned(pred)
    v_ref, g_ref = S.heatmap_loss_ref(targ, pred, kind, with_grad=True)
    p = pred.detach().requires_grad_(True)
    v = lpb.heatmap_loss(targ, p, kind)
    close(v, v_ref, atol=1e-7, rtol=1e-4)
    (1.7 * v).backward()
    close(p.grad, 1.7 * g_ref, atol=1e-6 * float(g_ref.abs().max()), rtol=1e-3)


def test_heatmap_mse_from_keypoints_at_scale(lpb, dev):
    """Fused targets + MSE on 256 labeled frames: visibility 0 / 1 / 2, keypoints outside the frame and NaN."""
    b, img, oh = 256, 384, 96
    g = _gen(14)
    kp = torch.rand(b, K, 2, device=dev, generator=g) * img
    sel = torch.rand(b, K, device=dev, generator=g)
    kp[sel < 0.05] = -12.0                            # left of / above the frame
    kp[(sel >= 0.05) & (sel < 0.1), 0] = img + 9.0    # right of the frame
    kp[(sel >= 0.1) & (sel < 0.12)] = float("nan")
    vis = torch.randint(0, 3, (b, K), device=dev, generator=g)
    pred = _peaked_planes(b, K, oh, oh, seed=15, sigma=2.0)
    targ = S.gaussian_targets_ref(kp, img, img, (oh, oh), visibility=vis)
    v_ref, g_ref = S.heatmap_loss_ref(targ, pred, "mse", with_grad=True)
    p = pred.detach().requires_grad_(True)
    v = lpb.heatmap_mse_from_keypoints(kp, p, img, img, visibility=vis)
    close(v, v_ref, atol=1e-7, rtol=1e-4)
    (1.3 * v).backward()
    close(p.grad, 1.3 * g_ref, atol=1e-6 * float(g_ref.abs().max()), rtol=1e-3)


def _pca_scratch_floats(n_sel, n_views, n_comp, t, bwd):
    """losses.cu:662-669."""
    d = 2 * n_views if n_views > 0 else 2 * n_sel
    rows = t * n_sel if n_views > 0 else t
    f = rows * d + rows * n_comp + 2 * t
    return f + (rows * d + rows * n_comp if bwd else 0)


def _unsup_check(lpb, kp, conf, eps, thr, sv, mv, sv_ref, mv_ref):
    n_clips = kp.shape[0]
    wts = torch.rand(n_clips, 3, device=kp.device, generator=_gen(16)) + 0.5
    x = kp.clone().requires_grad_(True)
    out = lpb.unsup_losses(x, conf, temporal_eps=eps, prob_threshold=thr, pca_singleview=sv, pca_multiview=mv)
    (out[:, :3] * wts).sum().backward()
    xr = kp.to(F64).requires_grad_(True)
    refs = []
    for i in range(n_clips):
        row = [S.temporal_loss_ref(xr[i], conf[i], eps, thr),
               sv_ref(xr[i]) if sv is not None else torch.zeros((), dtype=F64, device=kp.device),
               mv_ref(xr[i]) if mv is not None else torch.zeros((), dtype=F64, device=kp.device)]
        refs.append(torch.stack(row))
    ref = torch.stack(refs)
    (ref * wts.to(F64)).sum().backward()
    close(out[:, :3], ref, atol=1e-5, rtol=1e-4)
    close(x.grad, xr.grad, atol=1e-6 * float(xr.grad.abs().max()), rtol=1e-3)


def test_unsup_losses_bench_clips(lpb, dev, golden):
    """The bench's 16 clips x 32 frames: temporal + single-view PCA (median centring) + multi-view PCA per clip."""
    gl = golden("losses")
    base = torch.from_numpy(gl["pca_in_kp"]).to(dev)
    kp = base[None] + 3.0 * torch.randn(16, *base.shape, device=dev, generator=_gen(17))
    conf = torch.rand(16, base.shape[0], K, device=dev, generator=_gen(18))
    cols, mcm = gl["pca_sv_cols"], gl["pca_mv_mcm"]
    sv = lpb.PcaParams(cols.astype("int32"), len(cols), 0, "median", gl["pca_sv_mean"], gl["pca_sv_kept"], 2.5, dev)
    mv = lpb.PcaParams(mcm.reshape(-1).astype("int32"), mcm.shape[1], mcm.shape[0], None, gl["pca_mv_mean"], gl["pca_mv_kept"], 0.7, dev)
    sv_ref = lambda x: S.pca_singleview_ref(x, cols.tolist(), "median", sv.mean, sv.kept, 2.5)
    mv_ref = lambda x: S.pca_multiview_ref(x, mcm.tolist(), mv.mean, mv.kept, 0.7)
    _unsup_check(lpb, kp, conf, 3.0, 0.2, sv, mv, sv_ref, mv_ref)


def test_unsup_losses_large_shared_memory_route(lpb, dev):
    """Multi-view PCA, 4 views x 17 keypoints, 3 components, T = 80: the clip needs more than the default 48 KB of shared
    memory in both directions (losses.cu:753-755, :779-781) and stays under the 200 KB limit."""
    views, t, nc, n_clips = 4, 80, 3, 3
    kk = views * K
    fwd = (_pca_scratch_floats(K, views, nc, t, False) + 4) * 4
    bwd = (_pca_scratch_floats(K, views, nc, t, True) + t * kk * 2 + 4) * 4
    assert 48 * 1024 < fwd <= 200 * 1024 and 48 * 1024 < bwd <= 200 * 1024, (fwd, bwd)
    g = _gen(19)
    mcm = torch.arange(kk).reshape(views, K)
    mean = torch.randn(2 * views, device=dev, generator=g) * 50 + 150
    kept = torch.linalg.qr(torch.randn(2 * views, nc, device=dev, generator=g))[0].T.contiguous()
    # keypoints near the PCA subspace plus noise: some reprojection errors below epsilon, most above
    coef = torch.randn(n_clips, t, K, nc, device=dev, generator=g) * 40
    pts = coef @ kept + mean + torch.randn(n_clips, t, K, 2 * views, device=dev, generator=g) * 3.0
    kp = pts.reshape(n_clips, t, K, views, 2).permute(0, 1, 3, 2, 4).reshape(n_clips, t, 2 * kk).contiguous()
    conf = torch.rand(n_clips, t, kk, device=dev, generator=g)
    mv = lpb.PcaParams(mcm.reshape(-1).numpy().astype("int32"), K, views, None, mean.cpu().numpy(), kept.cpu().numpy(), 2.0, dev)
    mv_ref = lambda x: S.pca_multiview_ref(x, mcm.tolist(), mv.mean, mv.kept, 2.0)
    _unsup_check(lpb, kp, conf, 4.0, 0.1, None, mv, None, mv_ref)


def test_crnn_combine_grid_split(lpb, dev):
    """M * K >= 65536 windows exceed grid.y of one launch and are split (ops.py:475-477): the forward equals the
    single-launch runs on the sub-ranges bit for bit and every gradient their sum (to the rounding of the backward's
    atomic accumulation); both equal the float64 recurrence on all windows."""
    n, h, w, hidden, m = 64, 4, 6, 16, 5000
    per = 65535 // K
    assert m * K >= 65536 and per * K < 65536 and -(-m // per) == 2  # two launches
    g = _gen(20)
    wf = torch.randn(n, K, h, w, device=dev, generator=g)
    wb = torch.randn(n, K, h, w, device=dev, generator=g)
    idx = torch.randint(0, n, (m, 5), device=dev, generator=g, dtype=torch.int32)

    def params():
        return [torch.randn(K * hidden, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(K * hidden, device=dev, generator=g) * 0.1,
                torch.randn(K * hidden, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(K, device=dev, generator=g) * 0.1]

    hf, hb = params(), params()
    gout = torch.randn(m, K, h, w, device=dev, generator=g)

    def run(sl):
        leaves = [t.clone().requires_grad_(True) for t in [wf, wb, *hf, *hb]]
        out = lpb.crnn_combine(leaves[0], leaves[1], idx[sl], leaves[2:6], leaves[6:10])
        (out * gout[sl]).sum().backward()
        return out.detach(), [t.grad for t in leaves]

    out, grads = run(slice(0, m))
    out_a, grads_a = run(slice(0, per))
    out_b, grads_b = run(slice(per, m))
    assert torch.equal(out, torch.cat([out_a, out_b]))
    for x, a, b in zip(grads, grads_a, grads_b):
        close(x, a + b, atol=1e-6 * float((a + b).abs().max()), rtol=1e-5)
    leaves = [t.to(F64).requires_grad_(True) for t in [wf, wb, *hf, *hb]]
    ref = S.crnn_combine_ref(leaves[0], leaves[1], idx, leaves[2:6], leaves[6:10])
    close(out, ref, atol=1e-5 * float(ref.detach().abs().max()), rtol=1e-5)
    (ref * gout.to(F64)).sum().backward()
    for x, r in zip(grads, leaves):
        close(x, r.grad, atol=2e-6 * float(r.grad.abs().max()), rtol=2e-3)
