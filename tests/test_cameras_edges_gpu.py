"""GPU: the calibrated multi-view geometry (csrc/cameras.cu) at its edges against float64.

Every entry is run through ``ops`` on the cases of ``tests/cameras_oracle.py`` (each distortion coefficient alone, the
conditioning sweep and the fly calibration, far and infinite triangulated points, points on and behind a camera's
principal plane, NaN data, degenerate boxes) and compared, forward and gradient for a seeded upstream gradient, with
float64 autograd through the restatements on the same fp32 inputs, under ``cameras_oracle.bar_failures``: a few fp32
ulps of each point's magnitude forward, 1e-5 relative + 1e-6 of the tensor's max for gradients, plus 4x the measured
input sensitivity where the case is ill-conditioned.  Also: V from 2 to 64, K 1 to 51, B = 0, a launch of more than
2^20 threads, the keypoint on the baseline (a double lambda_min), and the pairwise-projection loss past 100k entries in
its one CTA.  Every case also runs twice and must give the same bits."""
import numpy as np
import pytest
import torch

import cameras_oracle as O

pytestmark = pytest.mark.gpu

CASES = O.edge_cases(np.load(O.GOLDEN_PATH))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


def gpu_outputs(ops, c: O.EdgeCase, dev):
    """the kernels' forward and gradient of every op of the case (keys as cameras_oracle.case_outputs), fp32 numpy"""
    x = {k: None if t is None else t.float().to(dev) for k, t in c.x.items()}
    K, E, D, bb = x["K"], x["E"], x["dist"], x["bbox"]
    kw = dict(bbox=bb, model_size=c.model_size if bb is not None else None)
    out = {}
    for op in c.ops:
        inp = x["points3d" if op == "proj" else "pairs3d" if op == "pmean" else "points"].clone().requires_grad_(True)
        if op == "tri":
            y = ops.triangulate_pairs(inp, K, E, D)
        elif op == "proj":
            y = ops.project_points(inp, K, E, D, **kw)
        elif op == "pmean":
            y = ops.project_points(inp, K, E, D, mean_over_pairs=True, **kw)
        elif op == "reproj":
            y = ops.project_points(ops.triangulate_pairs(inp, K, E, D), K, E, D, mean_over_pairs=True, **kw)
        else:
            y = ops.frame_to_model(inp, bb, *c.model_size)
        (g,) = torch.autograd.grad(y, inp, c.g[op].float().to(dev))
        out[op], out[op + "_grad"] = y.detach().cpu().numpy(), g.cpu().numpy()
    return out


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def run_twice(ops, c, dev):
    got, again = gpu_outputs(ops, c, dev), gpu_outputs(ops, c, dev)
    for k in got:
        assert same_bits(got[k], again[k]), f"{c.name}/{k}: two runs differ"
    return got


@pytest.mark.parametrize("name", list(CASES))
def test_case_within_the_float64_bars(lpb, dev, name):
    c = CASES[name]
    got = run_twice(lpb, c, dev)
    ref = O.case_outputs(c)
    if c.sign_free:  # V = 2: one pair per keypoint; the sign the kernel's rounding-level v3 chose, per point
        s = np.where((got["tri"] * ref["tri"]).sum(-1, keepdims=True) < 0, -1.0, 1.0)
        ref["tri"], ref["tri_grad"] = ref["tri"] * s, ref["tri_grad"] * s
    fails = O.bar_failures(c, got, ref, O.case_sensitivity(c))
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("k", [1, 17, 51])
@pytest.mark.parametrize("v", [2, 3, 5, 8, 17, 64])
def test_view_and_keypoint_counts(lpb, dev, v, k):
    c = O.shape_case(v, k, b=1 if v == 64 else 2)
    got = run_twice(lpb, c, dev)
    fails = O.bar_failures(c, got, O.case_outputs(c))
    assert not fails, "\n".join(fails)


def test_triangulation_past_2_pow_20_threads(lpb, dev):
    """B x pairs x K = 11 x 2016 x 51 threads in the forward: the int64 thread index and output offsets"""
    c = O.shape_case(64, 51, b=11)
    c.ops = ("tri",)
    assert 11 * 2016 * 51 > 1 << 20
    got = run_twice(lpb, c, dev)
    fails = O.bar_failures(c, got, O.case_outputs(c))
    assert not fails, "\n".join(fails)


def test_empty_batch(lpb, dev):
    """B = 0 through every entry: empty results (the loss 0 with a count of 0) and empty gradients, nothing read"""
    K, E, D = torch.zeros(0, 3, 3, 3, device=dev), torch.zeros(0, 3, 3, 4, device=dev), torch.zeros(0, 3, 5, device=dev)
    bb = torch.zeros(0, 12, device=dev)
    pts = torch.zeros(0, 3, 4, 2, device=dev, requires_grad=True)
    assert lpb.triangulate_pairs(pts, K, E, D).shape == (0, 3, 4, 3)
    for f in (lambda: lpb.triangulate_pairs(pts, K, E, D),
              lambda: lpb.project_points(lpb.triangulate_pairs(pts, K, E, D), K, E, D, mean_over_pairs=True, bbox=bb, model_size=(64, 64)),
              lambda: lpb.frame_to_model(pts, bb, 64, 64)):
        y = f()
        (g,) = torch.autograd.grad(y, pts, torch.ones_like(y))
        assert g.shape == pts.shape
    p3 = torch.zeros(0, 4, 3, device=dev, requires_grad=True)
    y = lpb.project_points(p3, K, E, D)
    assert y.shape == (0, 3, 4, 2) and torch.autograd.grad(y, p3, torch.ones_like(y))[0].shape == p3.shape
    pred = torch.zeros(0, 3, 4, 3, device=dev, requires_grad=True)
    loss, n = lpb.pairwise_projections_loss(torch.zeros(0, 4, 3, device=dev), pred, return_count=True)
    assert float(loss) == 0.0 and float(n) == 0.0
    assert torch.autograd.grad(loss, pred)[0].shape == pred.shape


def test_keypoint_on_the_baseline(lpb, dev):
    """Keypoint 0 sits at both epipoles: the DLT matrix has rank 2, lambda_min is double and the SVD's gradient is
    infinite, so there is no float64 answer to compare with.  The point returned must lie on both rays (reproject to
    both input pixels within the forward bar) and the gradient must be finite; keypoint 1 is ordinary."""
    c = O.baseline_keypoint_case()
    got = run_twice(lpb, c, dev)
    assert np.isfinite(got["tri"]).all() and np.isfinite(got["tri_grad"]).all()
    X = torch.from_numpy(got["tri"][:, 0]).double()
    rep = O.project_points_ref(X, c.x["K"], c.x["E"], c.x["dist"]).numpy()  # (1, 2 views, 2 keypoints, 2)
    px = c.x["points"].numpy()
    err = np.abs(rep[:, :, 0] - px[:, :, 0])
    assert (err <= 5e-7 * np.abs(px[:, :, 0]).max(-1, keepdims=True)).all(), (rep[:, :, 0], px[:, :, 0])
    ref = O.case_outputs(c)
    np.testing.assert_allclose(got["tri"][:, :, 1], ref["tri"][:, :, 1], rtol=0, atol=5e-7 * np.abs(ref["tri"][:, :, 1]).max())
    np.testing.assert_allclose(got["tri_grad"][:, :, 1], ref["tri_grad"][:, :, 1], rtol=1e-5, atol=1e-6 * np.abs(ref["tri_grad"][:, :, 1]).max())


def _loss_inputs(kind):
    gen = torch.Generator().manual_seed({"large": 90, "all_nan": 91, "zero_distance": 92}[kind])
    b, p, k = (40, 66, 51) if kind == "large" else (4, 6, 17)
    targ = torch.randn(b, k, 3, generator=gen) * 0.3
    pred = targ[:, None] + torch.randn(b, p, k, 3, generator=gen) * 0.05
    if kind == "large":
        targ[0, 2] = float("nan")
        pred.view(-1, 3)[torch.randperm(b * p * k, generator=gen)[: b * p * k // 100], torch.randint(0, 3, (b * p * k // 100,), generator=gen)] = float("nan")
    elif kind == "all_nan":
        pred[:] = float("nan")
    else:
        pred[:, :, ::2] = targ[:, None, ::2]
    return targ, pred


@pytest.mark.parametrize("kind", ["large", "all_nan", "zero_distance"])
def test_pairwise_projections_loss(lpb, dev, kind):
    """one CTA over all entries, up to 40 x 66 x 51 = 134,640: the loss (a few fp32 ulps), the kept count (exact) and
    the gradient (zero for dropped entries and exact-zero distances) against float64"""
    targ, pred = _loss_inputs(kind)
    assert kind != "large" or pred[..., 0].numel() > 100_000
    gup = 0.7
    runs = []
    for _ in range(2):
        p = pred.to(dev).requires_grad_(True)
        loss, n = lpb.pairwise_projections_loss(targ.to(dev), p, return_count=True)
        (g,) = torch.autograd.grad(loss, p, torch.tensor(gup, device=dev))
        runs.append((loss.detach().cpu().numpy().reshape(1), g.cpu().numpy(), float(n)))
    assert all(same_bits(a, b) for a, b in zip(runs[0][:2], runs[1][:2]))
    got_loss, got_g, got_n = runs[0]
    p64 = pred.double().requires_grad_(True)
    ref, ref_n = O.pairwise_projections_loss_ref(targ.double(), p64)
    (ref_g,) = torch.autograd.grad(ref, p64, torch.tensor(gup, dtype=torch.float64))
    ref, ref_g = float(ref), ref_g.numpy()
    assert got_n == int(ref_n)
    assert abs(float(got_loss[0]) - ref) <= 5e-7 * abs(ref), (float(got_loss[0]), ref)
    assert np.isfinite(got_g).all()
    np.testing.assert_allclose(got_g, ref_g, rtol=1e-5, atol=1e-6 * np.abs(ref_g).max())
    dropped = np.isnan(pred.numpy() - targ[:, None].numpy()).any(-1)
    assert (got_g[dropped] == 0).all()
    if kind == "zero_distance":
        assert (got_g[:, :, ::2] == 0).all()
