"""The soft-argmax decode (csrc/decode.cu) where its routes split, against the float64 references of tests/scale_oracle.py.

The forward warp kernel bounds the field by lip * max|h|, keeps the coarse pixels with |h| >= theta = (mlb - DEC_CUT / T)
/ lip, and evaluates their hull plus an R-tap halo (the box) in a 32 x 32 window; a plane whose box has more than
DECW_WIN - 2R - 2 rows or columns, a NaN plane and T <= 0 are queued for the CTA kernel, which evaluates the whole plane.
The backward window kernel takes the forward's box; a box of more than DEC_WIN - 2R rows or columns overflows into the
dense backward.  Every case below observes the route a plane took -- the forward's queue in a workspace the test owns,
the backward's ``meta[:, 2]`` -- checks it against a float64 restatement of those rules (``predict_forward``), and
compares keypoints, confidences and both backward entries with ``decode_ref`` / ``decode_grad_ref``.

Bars (``check_planes``): keypoints 1e-4 px (peaked) / 5e-4 px (diffuse: the largest float64 pixel probability below
1 %) + 1e-4 relative, confidence 2e-6 + 1e-4 relative of the window at trunc() of the reference coordinates or across an
integer within 1e-3 px -- ``_check_decode``'s rules -- each widened by what a field error of 8 fp32 ulps can move the
float64 answer (zero where one pixel holds the mass; it matters for raw planes whose mass splits between far-apart
pixels of equal field).  Backward: every plane within 2e-3 of its largest |reference| element
(``_check_plane_grads``'s bar) plus the gradient that the kernel's keypoint error and that field error explain, on the
dense entry and on the windows re-assembled.  With ``pytest -s`` the worst error / bound ratio of each case family is
printed at the end of the module, with the wall time and the peak device memory.
"""
import ctypes
import time

import pytest
import torch

import scale_oracle as S
from test_scale_gpu import _check_decode, _rebuild_windows

pytestmark = pytest.mark.gpu

F64 = torch.float64
DEC_CUT = 40.0
WIN = 32  # DECW_WIN and DEC_WIN
UNSUPPORTED = -3
TEMPS = [1000.0, 100.0, 10.0, 1.0]
DSS = [1, 2, 3]
WORST: dict = {}  # case family -> (worst backward error / bound, case)


def fwd_limit(ds):
    """Most rows / columns of a box the forward warp kernel evaluates (DECW_WIN - 2R - 2)."""
    return WIN - 2 * (ds + 2) - 2


def bwd_limit(ds):
    """Most rows / columns of a box the backward window kernel takes (DEC_WIN - 2R)."""
    return WIN - 2 * (ds + 2)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from lightning_pose_b200 import ops

    return ops


@pytest.fixture(scope="module")
def lib(ops):
    from lightning_pose_b200._lib import lib

    return lib


@pytest.fixture(scope="module", autouse=True)
def _report(dev):
    WORST.clear()
    torch.empty(1, device=dev)  # the allocator exists before its peak is reset
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    yield
    for name, (ratio, case) in sorted(WORST.items()):
        print(f"decode edges: backward {name:28s} worst error / bound {ratio:.4f}  ({case})")
    print(f"decode edges: wall {time.perf_counter() - t0:.1f} s, peak allocated {torch.cuda.max_memory_allocated(dev) / 2**20:.0f} MiB")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------
# the entries, with buffers the test owns
# ------------------------------------------------------------------------------------------------
def decode_fwd(ops, lib, hm, ds, T):
    """lpb_decode_fwd on (B, K, h, w) planes with this test's workspace: (xy, conf, stats, queued (n,) bool).  The
    workspace starts with {queue count, queued plane ids ...} (launch_decode_fwd)."""
    from lightning_pose_b200._lib import check

    b, k, h, w = hm.shape
    n = b * k
    xy = torch.empty((b, k, 2), device=hm.device)
    conf = torch.empty((b, k), device=hm.device)
    stats = torch.empty((b, k, 8), device=hm.device)
    nbytes = ctypes.c_size_t(0)
    check(lib.lpb_decode_fwd_workspace_bytes(n, ctypes.byref(nbytes)))
    ws = torch.full((nbytes.value // 4,), -7, dtype=torch.int32, device=hm.device)
    check(lib.lpb_decode_fwd(ops._ptr(hm), n, h, w, ds, T, ops._ptr(xy), ops._ptr(conf), ops._ptr(stats), ops._ptr(ws), ops._stream()))
    count = int(ws[0])
    ids = ws[1 : 1 + count].long()
    queued = torch.zeros(n, dtype=torch.bool, device=hm.device)
    queued[ids] = True
    assert int(queued.sum()) == count, "a plane was queued twice"
    return xy, conf, stats, queued


# ------------------------------------------------------------------------------------------------
# the forward's route, restated in float64
# ------------------------------------------------------------------------------------------------
def field64(planes, ds):
    """(n, h, w) float64 -> the upsampled field (n, h 2^ds, w 2^ds)."""
    _, h, w = planes.shape
    return S.upsample_op(h, ds, planes.device) @ planes @ S.upsample_op(w, ds, planes.device).T


def lip(n, ds, dev):
    return float(S.upsample_op(n, ds, dev).abs().sum(1).max())


def predict_forward(hm, ds, T, cut=DEC_CUT):
    """decode_plane_warp's decisions for the fp32 planes hm (B, K, h, w), in float64: a dict of (n,) tensors
    ``queued``, ``box`` (n, 4) = (A0, A1, B0, B1), ``near`` (a pixel within 1e-5 relative of theta: fp32 rounding may
    decide the candidate set), ``diffuse`` (the largest softmax probability below 1 %) and ``theta``; and the float64
    field ``field`` and softmax ``p`` (n, h 2^ds, w 2^ds)."""
    b, k, h, w = hm.shape
    n, f, r = b * k, 1 << ds, ds + 2
    x = hm.reshape(n, h, w).to(F64)
    a = x.abs()
    fld = field64(x, ds)
    logits = (fld * T).reshape(n, -1)
    diffuse = (logits.amax(1) - torch.logsumexp(logits, 1)).exp() < 1e-2
    nan = torch.isnan(a).flatten(1).any(1)
    best = torch.nan_to_num(a, nan=-1.0).reshape(n, -1).argmax(1)  # the first arg max, as the kernel's tie-break
    ba, bb = best // w, best % w
    ar = torch.arange(n, device=hm.device)
    # exact field on the arg max's F x F block, one pixel per lane: at ds 3 the warp's 32 lanes take its first 4 rows
    mlb = fld.reshape(n, h, f, w, f)[ar, ba, : min(f, 32 // f), bb, :].amax((1, 2))
    theta = ((mlb - cut / T) / (lip(h, ds, hm.device) * lip(w, ds, hm.device))) if T > 0 else torch.zeros_like(mlb)
    cand = a >= theta[:, None, None]
    rows, cols = cand.any(2), cand.any(1)
    ia, ib = torch.arange(h, device=hm.device), torch.arange(w, device=hm.device)
    amin = torch.where(rows, ia, h).amin(1)
    amax = torch.where(rows, ia, -1).amax(1)
    bmin = torch.where(cols, ib, w).amin(1) // 4 * 4  # the hull sweep's 4-column groups
    bmax = (torch.where(cols, ib, -1).amax(1) // 4 * 4 + 3).clamp(max=w - 1)
    box = torch.stack([(amin - r).clamp(min=0), (amax + r).clamp(max=h - 1), (bmin - r).clamp(min=0), (bmax + r).clamp(max=w - 1)], 1)
    nrows, ncols = box[:, 1] - box[:, 0] + 1, box[:, 3] - box[:, 2] + 1
    queued = nan | (T <= 0) | (amax < 0) | (nrows > fwd_limit(ds)) | (ncols > fwd_limit(ds))
    near = ((a - theta[:, None, None]).abs() <= 1e-5 * theta.abs()[:, None, None]).flatten(1).any(1) & ~nan & (T > 0)
    p = torch.softmax(logits, 1).reshape(fld.shape)
    return {"queued": queued, "box": box, "near": near, "diffuse": diffuse, "theta": theta, "field": fld, "p": p}


# ------------------------------------------------------------------------------------------------
# one call of every entry on a batch of planes, against float64
# ------------------------------------------------------------------------------------------------
def check_planes(ops, lib, hm, ds, T, gxy, family, case):
    """Forward and both backward entries on hm (B, K, h, w) at temperature T.  Returns (queued, predicted, flags)."""
    b, k, h, w = hm.shape
    n = b * k
    xy, conf, stats, queued = decode_fwd(ops, lib, hm, ds, T)
    pred = predict_forward(hm, ds, T)
    sure = ~pred["near"]
    wrong = (queued != pred["queued"]) & sure
    assert not bool(wrong.any()), (case, "forward route", wrong.nonzero()[:, 0].tolist(), queued[wrong].tolist())
    # a plane the warp kernel took reports the box it evaluated: the predicted one
    took = ~queued & sure
    got_box = stats.reshape(n, 8)[:, 4:].round().long()
    bad = (got_box != pred["box"]).any(1) & took
    assert not bool(bad.any()), (case, "forward box", got_box[bad][:4].tolist(), pred["box"][bad][:4].tolist())
    # a queued plane's box is the whole plane
    full = torch.tensor([0, h - 1, 0, w - 1], device=hm.device)
    assert bool((got_box[queued & ~torch.isnan(stats.reshape(n, 8)[:, 4])] == full).all()), (case, "queued box")
    ref = S.decode_ref(hm, ds, T)
    pre = ref[2].reshape(n, 2)
    assert torch.equal(torch.isnan(xy.reshape(n, 2)), torch.isnan(pre)), (case, "NaN keypoints")
    # keypoints: _check_decode's bars, widened by what a field error of 2^-21 max|field| (8 fp32 ulps) can move them:
    # |d xhat| <= |T| df sum p |j - xhat|.  Zero for a plane whose mass sits on one pixel; it matters only where the
    # mass splits between far-apart pixels of almost equal field (the raw planes)
    fld, p = pred["field"], pred["p"]
    df = 2.0**-21 * fld.abs().flatten(1).amax(1)
    jj = torch.arange(fld.shape[2], device=hm.device, dtype=F64)
    ii = torch.arange(fld.shape[1], device=hm.device, dtype=F64)
    spread = torch.stack([(p.sum(1) * (jj - pre[:, :1]).abs()).sum(1), (p.sum(2) * (ii - pre[:, 1:]).abs()).sum(1)], 1)
    cond = abs(T) * df[:, None] * spread
    tol = torch.where(pred["diffuse"], 5e-4, 1e-4)[:, None] + 1e-4 * ref[0].reshape(n, 2).abs() + cond
    kerr = (xy.reshape(n, 2).to(F64) - ref[0].reshape(n, 2)).abs()
    bad = (kerr > tol).any(1)
    assert not bool(bad.any()), (case, "keypoints", bad.nonzero()[:, 0].tolist(), float((kerr - tol).amax(1).max()))
    # confidence: the trunc rule of _check_decode, widened by |T| df (|d conf| <= |T| df sum p |1[window] - conf|)
    alt = ref[3].reshape(n, 9)
    cerr = ((conf.reshape(n, 1).to(F64) - alt).abs() - (2e-6 + 1e-4 * alt.abs()) - abs(T) * df[:, None]).amin(1)
    assert not bool((cerr > 0).any()), (case, "confidence", (cerr > 0).nonzero()[:, 0].tolist(), float(cerr.max()))

    # backward: the dense entry and the windows, on the forward's stats
    g_ref = S.decode_grad_ref(hm, ds, T, gxy).reshape(n, -1)
    dense = ops._decode_bwd(hm, stats, gxy, ds, T)
    win, meta, ov = ops.decode_backward_windows(hm, stats, gxy, ds, T)
    rebuilt, flags = _rebuild_windows(win, meta, ov, h, w)
    nrows, ncols = got_box[:, 1] - got_box[:, 0] + 1, got_box[:, 3] - got_box[:, 2] + 1
    zero = (gxy.reshape(n, 2) == 0).all(1)
    want = torch.where(zero, 0, torch.where((nrows > bwd_limit(ds)) | (ncols > bwd_limit(ds)), 2, 1))
    assert torch.equal(flags, want), (case, "backward route", flags.tolist(), want.tolist())
    # 2e-3 of the plane's max |reference|, plus the gradient its inputs' rounding explains: G = T p ((j - xhat) gx +
    # (i - yhat) gy) moves by T p dx gx for a keypoint error dx (the kernel's stats against float64, + 2^-21 |xhat|) and
    # by T df |G| for a field error df.  Where one pixel holds all the mass the reference gradient is itself of the
    # order of T 2^-24 |xhat|, and only these terms are meaningful.
    uh, uw = S.upsample_op(h, ds, hm.device).abs(), S.upsample_op(w, ds, hm.device).abs()
    st = stats.reshape(n, 8)[:, 2:4].to(F64)
    dx = (st - pre).abs().nan_to_num(0.0) + 2.0**-21 * pre.abs()
    g64 = gxy.reshape(n, 2).to(F64)
    gfield = T * p * ((jj - pre[:, :1, None]) * g64[:, :1, None] + (ii[:, None] - pre[:, 1:, None]) * g64[:, 1:, None])
    lim = (2e-3 * g_ref.abs().amax(1) + 1e-12
           + abs(T) * (dx * g64.abs()).sum(1) * (uh.T @ p @ uw).flatten(1).amax(1)
           + abs(T) * df * (uh.T @ gfield.abs() @ uw).flatten(1).amax(1))
    ratio = 0.0
    for name, got in (("dense", dense), ("windows", rebuilt)):
        err = (got.reshape(n, -1).to(F64) - g_ref).abs().amax(1)
        bad = ~(err <= lim)
        assert not bool(bad.any()), (case, name, f"{int(bad.sum())} planes off, worst ratio {float((err / lim).nan_to_num(1e30).max())}")
        ratio = max(ratio, float((err / lim).max()))
    if ratio >= WORST.get(family, (-1.0, ""))[0]:
        WORST[family] = (ratio, case)
    return queued, pred, flags


def random_gxy(n, seed, dev, zero_every=0):
    g = torch.randn(n, 2, device=dev, generator=gen(seed))
    if zero_every:
        g[::zero_every] = 0.0
    return g


# ------------------------------------------------------------------------------------------------
# 1. window-fit sweep
# ------------------------------------------------------------------------------------------------
def sweep_planes(ds, h, w, axis, ds_range, amp, dev):
    """One plane per separation d: two single-pixel peaks of height amp, d coarse pixels apart along ``axis``; the
    first at row R (rows: the box starts at row 0, unclipped) or column 4 (columns: the hull starts on a 4-column group), the other coordinate mid-plane."""
    r = ds + 2
    hm = torch.zeros(len(ds_range), h, w, device=dev)
    for i, d in enumerate(ds_range):
        if axis == "rows":
            hm[i, r, w // 2] = hm[i, r + d, w // 2] = amp
        else:
            hm[i, h // 2, 4] = hm[i, h // 2, 4 + d] = amp
    return hm[None]


@pytest.mark.parametrize("T", TEMPS)
@pytest.mark.parametrize("axis", ["rows", "cols"])
@pytest.mark.parametrize("ds", DSS)
def test_window_fit_sweep(ops, lib, dev, ds, axis, T):
    """Two equal single-pixel peaks d coarse pixels apart, height 1000 / T (the same T * h at every T), swept across the
    forward's limit (box of DECW_WIN - 2R - 2 rows / columns: the first separation that queues is 30 - 4R along rows).
    On a plane of DEC_WIN - 2R pixels a side, a queued plane's box -- the whole plane -- still fits the backward window:
    the forward queues but the backward window fits.  On a 48 x 40 plane the queued planes overflow the backward window
    too.  The reverse (forward window, backward overflow) cannot occur: the forward's box is at most DECW_WIN - 2R - 2.
    Closest existing tests: test_scale_gpu.py::test_decode_forward_past_one_wave (single peaks, far from any limit) and
    test_gpu_parity.py::test_decode_backward_windows_match_dense."""
    d_first = fwd_limit(ds) - 2 * (ds + 2)  # rows: d + 1 + 2R > DECW_WIN - 2R - 2
    d_range = list(range(d_first - 5, d_first + 2))
    for side, (h, w) in (("bwd-fit plane", (bwd_limit(ds), bwd_limit(ds))), ("48x40 plane", (48, 40))):
        hm = sweep_planes(ds, h, w, axis, d_range, 1000.0 / T, dev)
        case = f"ds{ds} {axis} T={T:g} {side}"
        queued, pred, flags = check_planes(ops, lib, hm, ds, T, random_gxy(len(d_range), ds, dev), "1 window-fit sweep", case)
        q = queued.tolist()
        # both routes occur, and the route flips once, between adjacent separations
        assert q == sorted(q) and not q[0] and q[-1], (case, dict(zip(d_range, q)))
        flip = d_range[q.index(True)]
        if axis == "rows":
            assert flip == d_first, (case, flip, d_first)
        f = flags.tolist()
        if side == "bwd-fit plane":
            assert f == [1] * len(d_range), (case, f)  # queued planes keep the backward window
        else:
            assert f == [2 if x else 1 for x in q], (case, f)
            assert f.index(2) == q.index(True)  # the backward's route flips at the same separation
        print(f"{case}: forward queues from d = {flip}, backward flags {dict(zip(d_range, f))}")


# ------------------------------------------------------------------------------------------------
# 2. pruning-cut sweep
# ------------------------------------------------------------------------------------------------
GAPS = [DEC_CUT - 0.5, DEC_CUT + 0.5, 20.0, 5.0]  # T (mlb - bump field): just inside / outside the cut, and well inside
OFFSETS = [(-9, 0), (9, 0), (0, -9), (0, 9), (-20, 0), (20, 0), (0, -20), (0, 20)]


def bump_planes(ds, T, dev, h=64, w=64):
    """A single-pixel main peak of height 1000 / T mid-plane and one bump (single pixel or a Gaussian of sigma 2) at
    each offset, scaled so that the bump's largest float64 field value is mlb - gap / T; and the gaps."""
    amp = 1000.0 / T
    cy, cx = h // 2, w // 2
    main = torch.zeros(h, w, device=dev, dtype=F64)
    main[cy, cx] = amp
    mlb = float(field64(main[None], ds).max())
    yy = torch.arange(h, device=dev, dtype=F64)[:, None]
    xx = torch.arange(w, device=dev, dtype=F64)[None, :]
    planes, cases = [], []
    for shape in ("pixel", "gauss"):
        for dy, dx in OFFSETS:
            if shape == "pixel":
                unit = torch.zeros(h, w, device=dev, dtype=F64)
                unit[cy + dy, cx + dx] = 1.0
            else:
                unit = torch.exp(-((yy - cy - dy) ** 2 + (xx - cx - dx) ** 2) / 8.0)
            fu, fm = field64(unit[None], ds)[0], field64(main[None], ds)[0]
            at = fu.argmax()
            for gap in GAPS:
                target = mlb - gap / T
                planes.append(main + unit * (target - fm.flatten()[at]) / fu.flatten()[at])
                cases.append((shape, dy, dx, gap))
    return torch.stack(planes)[None].float(), cases, mlb


@pytest.mark.parametrize("T", TEMPS)
@pytest.mark.parametrize("ds", DSS)
def test_pruning_cut_sweep(ops, lib, dev, ds, T):
    """A main peak and one bump whose largest field value is DEC_CUT / T +- 0.5 / T below the field maximum (just inside
    and just outside the cut), or 20 / T and 5 / T below it (mass the keypoint must see), 9 and 20 coarse pixels away
    on each side of the peak along rows and columns, as a single pixel (|h| far above theta: the bump is a candidate
    and widens the hull) and as a Gaussian of sigma 2 (field close to h: a candidate by a margin of about lip, the bound
    the forward's theta rests on).  Far bumps queue the plane, near ones keep the window.
    Closest existing test: test_gpu_parity.py::test_decode_multimodal_random_fields (random spiky planes, T = 1000)."""
    hm, cases, _ = bump_planes(ds, T, dev)
    queued, pred, _ = check_planes(ops, lib, hm, ds, T, random_gxy(len(cases), 10 + ds, dev), "2 pruning cut", f"ds{ds} T={T:g}")
    q = queued.tolist()
    assert any(q) and not all(q), q  # both routes occur within the sweep
    far = [i for i, c in enumerate(cases) if max(abs(c[1]), abs(c[2])) == 20 and c[3] < DEC_CUT]
    assert all(q[i] for i in far)  # a bump inside the cut, 20 pixels away, widens the hull past the window


# ------------------------------------------------------------------------------------------------
# 3. clipped boxes: peaks within R of the borders and corners, and planes of at most 2R + 1 pixels a side
# ------------------------------------------------------------------------------------------------
CLIP_SHAPES = [(48, 64), (64, 48), (30, 41), (1, 9), (9, 1), (3, 5), (7, 7)]


def border_positions(n, r):
    if n <= 2 * r + 2:
        return list(range(n))
    return sorted({0, 1, r - 1, r, n - 1 - r, n - r, n - 2, n - 1, n // 2})


def clipped_planes(ds, h, w, T, dev):
    """Planes of two kinds at every (row, column) within R of a border or mid-plane: a single pixel of height 1000 / T,
    and a plane softmax of a Gaussian of sigma 1.6 (the broad peak of a trained head; diffuse at low T)."""
    r = ds + 2
    pos = [(y, x) for y in border_positions(h, r) for x in border_positions(w, r)]
    yy = torch.arange(h, device=dev, dtype=torch.float32)[:, None]
    xx = torch.arange(w, device=dev, dtype=torch.float32)[None, :]
    planes = []
    for y, x in pos:
        p = torch.zeros(h, w, device=dev)
        p[y, x] = 1000.0 / T
        planes.append(p)
        planes.append(torch.softmax((-((yy - y) ** 2 + (xx - x) ** 2) / (2 * 1.6**2)).flatten(), 0).reshape(h, w))
    return torch.stack(planes)[None].contiguous()


@pytest.mark.parametrize("T", TEMPS)
@pytest.mark.parametrize("shape", CLIP_SHAPES, ids=[f"{h}x{w}" for h, w in CLIP_SHAPES])
@pytest.mark.parametrize("ds", DSS)
def test_clipped_boxes(ops, lib, dev, ds, shape, T):
    """Peaks within R of each border and corner of non-square planes, where the box is clipped and the 5 x 5 confidence
    window steps outside the plane; and planes no taller or wider than 2R + 1, where every row or column is a border row
    of the upsampling tables.  Closest existing tests: test_gpu_parity.py::test_decode_vs_oracle_shapes (random Gaussian
    targets on 30 x 41, 5 x 7 and 8 x 8, forward only) and ::test_decode_backward_windows_match_dense (one corner peak,
    48 x 40, compared with the dense kernel)."""
    h, w = shape
    hm = clipped_planes(ds, h, w, T, dev)
    n = hm.shape[1]
    queued, _, _ = check_planes(ops, lib, hm, ds, T, random_gxy(n, 20 + ds, dev, zero_every=7), "3 clipped boxes", f"ds{ds} {h}x{w} T={T:g}")
    if T == 1000.0 and h * w > 9:
        assert not bool(queued.all())  # the window route serves border peaks


# ------------------------------------------------------------------------------------------------
# 4. temperature
# ------------------------------------------------------------------------------------------------
def softmax_planes(h, w, n, sigma, seed, dev):
    """Plane softmaxes of Gaussians of the given sigma at random centres, a quarter of them within 2 pixels of a border."""
    g = gen(seed)
    cy = torch.rand(n, 1, 1, device=dev, generator=g) * (h - 1)
    cx = torch.rand(n, 1, 1, device=dev, generator=g) * (w - 1)
    cy[: n // 4] = cy[: n // 4] % 2.0
    cx[n // 8 : n // 4] = (w - 1) - cx[n // 8 : n // 4] % 2.0
    yy = torch.arange(h, device=dev).view(1, h, 1).float()
    xx = torch.arange(w, device=dev).view(1, 1, w).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sigma**2)
    return torch.softmax(logits.reshape(n, -1), -1).reshape(1, n, h, w).contiguous()


@pytest.mark.parametrize("T", TEMPS + [0.0])
@pytest.mark.parametrize("ds", DSS)
def test_softmax_planes_across_temperature(ops, lib, dev, ds, T):
    """Plane softmaxes of Gaussians of sigma 1.0 and 1.6 on 48 x 64 planes (T * mlb from about 140 at T = 1000 to 0.1 at
    T = 1: below DEC_CUT the forward's theta is negative and every plane queues), and the window-fit sweep's planes of
    height 1, at every temperature; and T = 0 (a uniform softmax: the plane's centre, zero gradient), which queues every
    plane in the forward; the backward then runs on the whole-plane box.  T < 0 is refused (test_negative_temperature).
    Closest existing test: test_gpu_parity.py::test_decode_reference_known_answers (T = 1000, 100, 10 on golden planes)."""
    hm = torch.cat([softmax_planes(48, 64, 24, 1.0, 30 + ds, dev), softmax_planes(48, 64, 24, 1.6, 40 + ds, dev)], 1)
    queued, _, _ = check_planes(ops, lib, hm, ds, T, random_gxy(48, 50 + ds, dev), "4 temperature", f"ds{ds} T={T:g} softmax")
    if T <= 0:
        assert bool(queued.all())
    d = fwd_limit(ds) - 2 * (ds + 2)
    sweep = sweep_planes(ds, 48, 40, "rows", [d - 1, d], 1.0, dev)
    queued, _, _ = check_planes(ops, lib, sweep, ds, T, random_gxy(2, 60 + ds, dev), "4 temperature", f"ds{ds} T={T:g} sweep")
    if T <= 0:
        assert bool(queued.all())


# ------------------------------------------------------------------------------------------------
# 5. raw planes
# ------------------------------------------------------------------------------------------------
def raw_planes(dev, h=40, w=48):
    g = gen(77)
    out = []
    p = torch.zeros(h, w, device=dev)  # the arg max of |h| is a negative pixel far from the positive peak
    p[10, 12], p[30, 40] = -2.0, 1.0
    out.append(p)
    p = torch.zeros(h, w, device=dev)  # ... two pixels from it
    p[20, 20], p[20, 22] = -3.0, 1.0
    out.append(p)
    p = torch.zeros(h, w, device=dev)  # ... a negative ring around a positive peak
    p[15:20, 15:20] = -4.0
    p[17, 17] = 2.5
    out.append(p)
    out.append(torch.full((h, w), -100.0, device=dev))  # a negative constant: the field is largest at the border
    out[-1][20, 24] = -95.0
    out.append(torch.randn(h, w, device=dev, generator=g) * 10.0)  # large-magnitude noise of both signs
    out.append(torch.randn(h, w, device=dev, generator=g) * 0.01 - 5.0)  # a negative, almost flat plane
    p = torch.randn(h, w, device=dev, generator=g) * 0.01  # a positive peak beside a larger negative one
    p[5, 5], p[5, 9] = 3.0, -6.0
    out.append(p)
    return torch.stack(out)[None].contiguous()


@pytest.mark.parametrize("T", [1000.0, 1.0])
@pytest.mark.parametrize("ds", DSS)
def test_raw_planes(ops, lib, dev, ds, T):
    """Planes that are not softmaxes: negative values, large magnitudes, and an arg max of |h| at a negative pixel, which
    puts mlb far below the positive peak's field.  Whichever route the plane takes, it must decode as float64 does.
    Closest existing test: test_gpu_parity.py::test_decode_golden_regimes[raw] (one golden raw regime, forward only)."""
    hm = raw_planes(dev)
    queued, pred, flags = check_planes(ops, lib, hm, ds, T, random_gxy(hm.shape[1], 70 + ds, dev), "5 raw planes", f"ds{ds} T={T:g}")
    print(f"raw planes ds{ds} T={T:g}: queued {queued.tolist()}, backward flags {flags.tolist()}")


# ------------------------------------------------------------------------------------------------
# 6. size limits
# ------------------------------------------------------------------------------------------------
WIDEST = {1: 256, 2: 256, 3: 128}  # w <= 256 and w << ds <= 1024


def fwd_smem(h, w, ds):
    """launch_decode_fwd's dynamic shared memory: the zero-padded plane tile and DEC_FWD_SCRATCH floats, + 16 B."""
    r = ds + 2
    pitch = (((r + 3) & ~3) + w + r + 3) & ~3  # dec_pitch
    return ((h + 2 * r) * pitch + 880) * 4 + 16


def bwd_smem(h, w, ds):
    """launch_decode_bwd's: the tile and its gradient tile, 8 warps x 64 floats of row buffers, + 16 B."""
    r = ds + 2
    pitch = (((r + 3) & ~3) + w + r + 3) & ~3
    return (2 * (h + 2 * r) * pitch + 8 * 64) * 4 + 16


def first_refused(w, ds, smem_of, limit):
    h = 1
    while smem_of(h, w, ds) <= limit:
        h += 1
    return h


def limit_planes(h, w, dev, seed):
    """A peaked plane (the warp kernel's) and a diffuse one (queued: the CTA kernel stages the whole plane)."""
    g = gen(seed)
    peaked = torch.zeros(h, w, device=dev)
    peaked[h // 2, w // 3] = 1.0
    diffuse = torch.softmax(torch.randn(h * w, device=dev, generator=g) * 0.01, 0).reshape(h, w)
    return torch.stack([peaked, diffuse])[None].contiguous()


@pytest.mark.parametrize("ds", DSS)
def test_size_limits(ops, lib, dev, ds):
    """At the widest accepted width, the tallest plane each kernel's shared memory serves runs and matches float64, and
    the next height is refused with LPB_ERR_UNSUPPORTED naming the entry and the bytes, with every output untouched.
    The backward stages the plane and its gradient, twice the forward's tile, so the forward serves heights the
    backward refuses: at w = 256, h 104..210 (ds 1) and 102..208 (ds 2); at w = 128, h 190..387 (ds 3), on a device
    with 227 KB of opt-in shared memory (H100).  The largest heatmaps of the supported models, 128 x 128 at ds 2, need
    150,032 B in the backward.  Closest existing test: test_launch_limits_gpu.py::test_refused_past_the_device_limit
    (the plane softmax and upsample2x, not the decode)."""
    from lightning_pose_b200._lib import LpbError, check

    limit = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin  # the decode kernels have no static shared memory
    w = WIDEST[ds]
    hf, hb = first_refused(w, ds, fwd_smem, limit), first_refused(w, ds, bwd_smem, limit)
    print(f"size limits ds{ds} w={w}: forward refuses h >= {hf}, backward h >= {hb}")
    assert hb < hf
    if limit == 232448:  # H100: the heights DESIGN.md K2 / K2b records
        assert (hf, hb) == {1: (211, 104), 2: (209, 102), 3: (388, 190)}[ds]

    # the tallest plane the forward serves, and the tallest the backward serves, against float64
    hm = limit_planes(hf - 1, w, dev, 90 + ds)
    xy, conf, stats, queued = decode_fwd(ops, lib, hm, ds, 1000.0)
    assert queued.tolist() == [False, True]
    _check_decode(xy, conf, S.decode_ref(hm, ds, 1000.0), torch.tensor([False, True], device=dev))
    del hm
    check_planes(ops, lib, limit_planes(hb - 1, w, dev, 95 + ds), ds, 1000.0, random_gxy(2, 96 + ds, dev), "6 size limits", f"ds{ds} h={hb - 1}")

    # refused: the forward at hf, both backward entries at hb (whose forward runs); nothing is written
    def sentinel(*shape, dtype=torch.float32):
        return torch.full(shape, 7, dtype=dtype, device=dev)

    nb = ctypes.c_size_t(0)
    check(lib.lpb_decode_fwd_workspace_bytes(2, ctypes.byref(nb)))
    big = torch.zeros(1, 2, hf, w, device=dev)
    xy, conf, stats, ws = sentinel(2, 2), sentinel(2), sentinel(2, 8), sentinel(nb.value // 4, dtype=torch.int32)
    rc = lib.lpb_decode_fwd(ops._ptr(big), 2, hf, w, ds, 1000.0, ops._ptr(xy), ops._ptr(conf), ops._ptr(stats), ops._ptr(ws), ops._stream())
    msg = lib.lpb_last_error().decode()
    torch.cuda.synchronize()
    assert rc == UNSUPPORTED and msg.startswith(f"decode_fwd: needs {fwd_smem(hf, w, ds)} B"), (rc, msg)
    assert all(bool((t == 7).all()) for t in (xy, conf, stats, ws))

    hm = limit_planes(hb, w, dev, 97 + ds)
    _, _, stats, _ = decode_fwd(ops, lib, hm, ds, 1000.0)
    gxy = random_gxy(2, 98 + ds, dev)
    with pytest.raises(LpbError, match=f"error {UNSUPPORTED}: decode_bwd: needs {bwd_smem(hb, w, ds)} B"):
        ops._decode_bwd(hm, stats, gxy, ds, 1000.0)
    win, meta, ov, qu = sentinel(2, 32, 32), sentinel(2, 4, dtype=torch.int32), sentinel(2, hb, w), sentinel(3, dtype=torch.int32)
    rc = lib.lpb_decode_bwd_windows(ops._ptr(hm), ops._ptr(stats), ops._ptr(gxy), 2, hb, w, ds, 1000.0, ops._ptr(win), ops._ptr(meta),
                                    ops._ptr(ov), ops._ptr(qu), ops._stream())
    msg = lib.lpb_last_error().decode()
    torch.cuda.synchronize()
    assert rc == UNSUPPORTED and msg.startswith(f"decode_bwd: needs {bwd_smem(hb, w, ds)} B"), (rc, msg)
    assert all(bool((t == 7).all()) for t in (win, meta, ov, qu))

    # the stream still runs the next call
    small = limit_planes(20, 24, dev, 99)
    check_planes(ops, lib, small, ds, 1000.0, random_gxy(2, 100 + ds, dev), "6 size limits", f"ds{ds} after refusals")


@pytest.mark.parametrize("ds", DSS)
def test_negative_temperature(ops, lib, dev, ds):
    """T < 0 (and NaN) is refused by the forward and both backward entries with LPB_ERR_INVALID and a readable message,
    before anything is queued: the online softmax of the CTA kernel starts from a running maximum that assumes T >= 0,
    and before the check T = -1 gave NaN gradients on every plane of test_softmax_planes_across_temperature's input.
    Closest existing test: none takes T <= 0."""
    hm = softmax_planes(24, 20, 2, 1.0, 110 + ds, dev)
    _, _, stats, _ = decode_fwd(ops, lib, hm, ds, 1000.0)
    gxy = random_gxy(2, 111 + ds, dev)
    nb = ctypes.c_size_t(0)
    assert lib.lpb_decode_fwd_workspace_bytes(2, ctypes.byref(nb)) == 0
    for T in (-1.0, -1e-30, float("nan")):
        out = [torch.full(sh, 7.0, device=dev) for sh in ((2, 2), (2,), (2, 8), (2, 24, 20), (2, 32, 32), (2, 24, 20))]
        ints = [torch.full((nb.value // 4,), 7, dtype=torch.int32, device=dev), torch.full((2, 4), 7, dtype=torch.int32, device=dev),
                torch.full((3,), 7, dtype=torch.int32, device=dev)]
        xy, conf, st, g, win, ov = out
        ws, meta, qu = ints
        calls = {
            "decode_fwd": lambda: lib.lpb_decode_fwd(ops._ptr(hm), 2, 24, 20, ds, T, ops._ptr(xy), ops._ptr(conf), ops._ptr(st), ops._ptr(ws), ops._stream()),
            "decode_bwd": lambda: lib.lpb_decode_bwd(ops._ptr(hm), ops._ptr(stats), ops._ptr(gxy), 2, 24, 20, ds, T, ops._ptr(g), ops._stream()),
            "decode_bwd_windows": lambda: lib.lpb_decode_bwd_windows(ops._ptr(hm), ops._ptr(stats), ops._ptr(gxy), 2, 24, 20, ds, T, ops._ptr(win),
                                                                     ops._ptr(meta), ops._ptr(ov), ops._ptr(qu), ops._stream()),
        }
        for name, call in calls.items():
            rc = call()
            msg = lib.lpb_last_error().decode()
            assert rc == -1 and msg.startswith(f"{name}: temperature") and "must be >= 0" in msg, (name, T, rc, msg)
        torch.cuda.synchronize()
        assert all(bool((t == 7).all()) for t in out + ints), T
