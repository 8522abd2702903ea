"""CPU: pin the float64 restatement of the Gaussian-target rule (``targets_oracle.py``) to the golden vectors of the
reference's own code and to ``oracle.lp_oracle``, and show that the edge batch and the acceptance rules of
``test_targets_edges_gpu.py`` reject plausible wrong rules."""
import numpy as np
import pytest
import torch

import targets_oracle as TO
from oracle import lp_oracle as O

T = torch.from_numpy
F64 = torch.float64
CONFIGS, SIGMAS = TO.CONFIGS, TO.SIGMAS


def test_restatement_matches_golden(golden):
    g = golden("targets")
    kp, vis = T(g["in_keypoints"]), T(g["in_visibility"])
    close = lambda a, b: np.testing.assert_allclose(a.numpy(), b, atol=1e-7, rtol=1e-5)  # noqa: E731
    close(TO.target_planes(kp, 48, 64, 12, 16)[0], g["out_vis_none"])
    close(TO.target_planes(kp, 48, 64, 12, 16, visibility=vis)[0], g["out_vis"])
    close(TO.target_planes(kp, 48, 64, 24, 32, sigma=2.0)[0], g["out_sigma2_ds1"])
    close(TO.window_sum(T(g["eval_in_heatmaps"]), T(g["eval_in_locs"]), TO.window_radius()), g["eval_out"])


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("sigma", SIGMAS)
def test_restatement_matches_cpu_oracle_on_the_edge_batch(cfg, sigma):
    h, w, oh, ow = cfg
    kp, vis = TO.edge_batch(h, w, oh, ow)
    for v in (None, vis):
        ours, mode = TO.target_planes(kp, h, w, oh, ow, sigma, v)
        TO.check_planes(O.gaussian_targets(kp, h, w, (oh, ow), sigma, v), ours, f"{cfg} sigma {sigma}")
        pat = TO.plane_pattern(ours)
        assert torch.equal(pat == TO.ZERO, mode == TO.ZERO) and torch.equal(pat == TO.UNIFORM, mode == TO.UNIFORM)


def test_edge_batch_lands_on_the_bounds():
    """Every config's edge rows scale to exactly -1 and size + 1 in fp32, with the nearest products on either side."""
    for h, w, oh, ow in CONFIGS:
        x, y = TO.grid_coords(TO.edge_rows(h, w, oh, ow), h, w, oh, ow)
        for v, hi in ((x, ow + 1), (y, oh + 1)):
            for bound in (-1.0, float(hi)):
                assert bool((v == bound).any())
                # the nearest fp32 product on either side: the bound's neighbour, or the one after it when no fp32
                # image coordinate times the scale rounds to the neighbour (ratios that are not powers of two)
                for d in (np.inf, -np.inf):
                    n1 = np.nextafter(np.float32(bound), np.float32(d))
                    n2 = np.nextafter(n1, np.float32(d))
                    near = (v == float(n1)) | (v == float(n2))
                    assert bool(near.any()), (h, w, oh, ow, bound, d)
                    if h in (384, 256):  # power-of-two ratios: every neighbour is a product
                        assert bool((v == float(n1)).any())
        assert bool(torch.isnan(x).any()) and bool(torch.isinf(x).any()) and bool(torch.isinf(y).any())


def test_patterns_of_the_edge_batch():
    """What the rule decides on the edge batch: on a bound is inside, one product outside is bad; a NaN y alone is not
    bad (its plane is NaN); visibility 3 and -1 keep the clamped Gaussian (NaN for a NaN centre)."""
    h, w, oh, ow = CONFIGS[2]
    kp, vis = TO.edge_batch(h, w, oh, ow)
    x, y = TO.grid_coords(kp, h, w, oh, ow)
    pat = {v: TO.plane_pattern(TO.target_planes(kp, h, w, oh, ow, 1.25, vis if v == "vis" else None)[0]) for v in (None, "vis")}
    on = (x == -1) & (y > 0) & (y < oh)
    assert bool(on.any()) and bool((pat[None][on] == TO.GAUSS).all())
    out = (x < -1) & (y > 0) & (y < oh)
    assert bool((pat[None][out] == TO.ZERO).all())
    nan_y = ~torch.isnan(x) & torch.isnan(y)
    assert bool((pat[None][nan_y] == TO.NAN).all())
    for v, want_bad, want_nan in [(0, TO.ZERO, TO.ZERO), (1, TO.UNIFORM, TO.UNIFORM), (2, TO.ZERO, TO.ZERO),
                                  (3, TO.GAUSS, TO.NAN), (-1, TO.GAUSS, TO.NAN)]:
        rows = vis == v
        assert bool((pat["vis"][rows & out] == want_bad).all()), v
        assert bool((pat["vis"][rows & torch.isnan(x)] == want_nan).all()), v


@pytest.mark.parametrize("sigma", SIGMAS)
def test_keep_gradients_restatement_is_the_closed_form(sigma):
    """The autograd gradient equals sum G g (c - xbar) / sigma^2 * sx (and the same in y) on unclamped Gaussian planes,
    is 0 on a clamped coordinate and on zero / uniform planes, and NaN where the plane is NaN."""
    h, w, oh, ow = CONFIGS[2]
    kp, vis = TO.edge_batch(h, w, oh, ow)
    gout = torch.randn(kp.shape[0], kp.shape[1], oh, ow, generator=torch.Generator().manual_seed(3), dtype=F64)
    planes, mode, gk = TO.target_planes(kp, h, w, oh, ow, sigma, vis, keep_gradients=True, gout=gout)
    x, y = TO.grid_coords(kp, h, w, oh, ow)
    sx, sy = TO.grid_scale(h, w, oh, ow)
    cols, rows = torch.arange(ow, dtype=F64), torch.arange(oh, dtype=F64)
    pg = planes * gout
    xbar = (planes * cols).sum((-1, -2))
    ybar = (planes * rows[:, None]).sum((-1, -2))
    gx = ((pg * cols).sum((-1, -2)) - xbar * pg.sum((-1, -2))) / sigma**2 * float(sx)
    gy = ((pg * rows[:, None]).sum((-1, -2)) - ybar * pg.sum((-1, -2))) / sigma**2 * float(sy)
    gauss = mode == TO.GAUSS
    inx, iny = (x >= -1) & (x <= ow + 1), (y >= -1) & (y <= oh + 1)
    fin = gauss & ~torch.isnan(planes).any(-1).any(-1)
    torch.testing.assert_close(gk[..., 0][fin & inx], gx[fin & inx], rtol=1e-9, atol=1e-12)
    torch.testing.assert_close(gk[..., 1][fin & iny], gy[fin & iny], rtol=1e-9, atol=1e-12)
    assert bool((gk[..., 0][~gauss | ~inx] == 0).all()) and bool((gk[..., 1][~gauss | ~iny] == 0).all())
    # a NaN plane: NaN in the coordinate the clamp passes, 0 in a NaN one (torch.clamp's gradient mask is false there)
    assert bool(torch.isnan(gk[..., 0][gauss & ~fin & inx]).all()) and bool(torch.isnan(gk[..., 1][gauss & ~fin & iny]).all())
    assert bool((gauss & ~fin & (inx | iny)).any())


def test_mse_restatement():
    """Loss = sum over kept planes / n_kept, gradient 2 (p - t) / n_kept; nothing kept: NaN loss, zero gradient."""
    h, w, oh, ow = CONFIGS[1]
    kp, vis = TO.edge_batch(h, w, oh, ow)
    preds = torch.rand(kp.shape[0], kp.shape[1], oh, ow, generator=torch.Generator().manual_seed(4), dtype=F64) * 2 / (oh * ow)
    t, _ = TO.target_planes(kp, h, w, oh, ow, 1.25, vis)
    fin = ~torch.isnan(t).any(-1).any(-1)
    v = torch.where(fin, vis, 0)
    loss, grad = TO.mse_from_keypoints(kp, preds, h, w, 1.25, v)
    keep = fin & ~(t == 0).all(-1).all(-1)
    want = O.heatmap_mse_loss(t.float(), preds.float())  # the CPU oracle's loss on the materialised targets
    t = torch.where(fin[..., None, None], t, 0.0)
    assert abs(float(loss) - float(((t - preds)[keep] ** 2).sum() / keep.sum())) <= 1e-12 * float(loss)
    assert abs(float(loss) - float(O.heatmap_mse_loss(t.float(), preds.float()))) <= 1e-5 * float(loss)
    assert torch.isnan(want)
    torch.testing.assert_close(grad, torch.where(keep[..., None, None], 2 * (preds - t) / keep.sum(), 0.0), rtol=1e-12, atol=0)
    loss0, grad0 = TO.mse_from_keypoints(kp, preds, h, w, 1.25, torch.zeros_like(vis))
    assert torch.isnan(loss0) and bool((grad0 == 0).all())


def test_mask_oob_and_window_restatements():
    kp = torch.tensor([[[384.0, 5.0], [float(np.nextafter(np.float32(384), np.float32(0))), 5.0], [-0.0, 3.0],
                        [float("nan"), 2.0], [3.0, 406.0], [3.0, -1e-30]]])
    out = TO.mask_oob(kp, 406, 384)
    assert bool(torch.isnan(out[0, [0, 4, 5]]).all())
    assert torch.equal(out[0, 1], kp[0, 1]) and torch.equal(out[0, 2].view(torch.int32), kp[0, 2].view(torch.int32))
    assert torch.isnan(out[0, 3, 0]) and out[0, 3, 1] == 2.0
    hm = torch.arange(2 * 5 * 6, dtype=torch.float32).reshape(1, 2, 5, 6)
    locs = torch.tensor([[[-0.5, 4.999], [5.999, 0.0]]])
    got = TO.window_sum(hm, locs, 1)
    # (-0.5, 4.999) -> column 0, row 4: rows 3-4, columns 0-1 of plane 0; (5.999, 0) -> column 5, row 0 of plane 1
    assert float(got[0, 0]) == float(hm[0, 0, 3:5, 0:2].sum()) and float(got[0, 1]) == float(hm[0, 1, 0:2, 4:6].sum())
    assert TO.window_radius(1.25, 2) == 2 and TO.window_radius(0.5, 2) == 1 and TO.window_radius(1.6, 2) == 3


# (at sigma 0.5, 2 sigma^2 == sigma, so only sigma 1.25 and 3.0 tell the "2 sigma^2" mutation apart)
MUTATIONS = {
    "clamp bound counted bad (<= for <)": dict(clamp_inclusive=True),
    "NaN test applied to y as well": dict(nan_y=True),
    "sigma read as 2 sigma^2": dict(sigma_as_two_s2=True),
    "sx and sy swapped": dict(swap_scale=True),
}


@pytest.mark.parametrize("name", MUTATIONS)
def test_edge_batch_rejects_plausible_wrong_rules(name):
    """Each wrong rule changes at least one plane of the edge batch beyond what ``check_planes`` accepts, for some config
    and sigma of the GPU tests, with and without a visibility; the right rule passes everywhere."""
    rejected = 0
    for h, w, oh, ow in CONFIGS:
        kp, vis = TO.edge_batch(h, w, oh, ow)
        for sigma in SIGMAS:
            for v in (None, vis):
                ref = TO.target_planes(kp, h, w, oh, ow, sigma, v)[0]
                TO.check_planes(ref.clone(), ref)
                wrong = TO.target_planes(kp, h, w, oh, ow, sigma, v, **MUTATIONS[name])[0]
                try:
                    TO.check_planes(wrong, ref, name)
                except AssertionError:
                    rejected += 1
    assert rejected >= 1, f"{name}: no plane of the edge batch tells it apart"
