"""CPU: the bars of tests/test_cameras_edges_gpu.py have teeth, the edge cases are what they claim, and the camera
entries refuse what they cannot compute before anything reaches the device.

Each mutant below is a plausible slip in csrc/cameras.cu restated in the float64 oracle; its outputs, rounded to fp32
as the kernels' are, must miss the bar on the named case, while the unmutated oracle rounded to fp32 meets every bar."""
import ctypes

import numpy as np
import pytest
import torch

import cameras_oracle as O

CASES = O.edge_cases(np.load(O.GOLDEN_PATH))


def _swap(*pairs):
    perm = list(range(12))
    for a, b in pairs:
        perm[a], perm[b] = b, a
    return perm


# mutant -> (oracle keywords for a case, the case that must reject it)
MUTANTS = {
    "undistort_4_iterations": (lambda c: dict(num_iters=4), "dist_P4_k1"),
    "s1_s3_swapped": (lambda c: dict(dist_perm=_swap((8, 10))), "dist_P12_s1"),
    "p1_p2_swapped": (lambda c: dict(dist_perm=_swap((2, 3))), "dist_P4_p1"),
    "distortion_numerator_denominator_swapped": (lambda c: dict(dist_perm=_swap((0, 5), (1, 6), (4, 7))), "dist_P8_k4"),
    "dehomogenise_without_eps": (lambda c: dict(eps=0.0), "dehomog_principal_plane"),
    "dehomogenise_without_eps_far": (lambda c: dict(eps=0.0), "dehomog_far_points"),
    "dlt_in_float32": (lambda c: dict(dlt_dtype=torch.float32), "dist_P4_k1"),
    "pairs_in_reverse_order": (lambda c: dict(pairs=O.camera_pairs(c.x["K"].shape[1])[::-1]), "nan"),
    "pair_mean_gradient_without_1_over_pairs": (lambda c: dict(pair_mean_grad_scaled=False), "dist_P4_k1"),
    "frame_to_model_gradient_keeps_offset": (lambda c: dict(f2m_keep_offset=True), "bbox_degenerate"),
}


def as_kernel(c, out):
    """float64 outputs as the kernels return them: rounded to fp32, a NaN gradient of NaN data written as 0"""
    r = {}
    for k, v in out.items():
        v = v.astype(np.float32).astype(np.float64)
        if k.endswith("_grad") and c.grad_nonfinite == "zero":
            v = np.where(np.isnan(v), 0.0, v)
        r[k] = v
    return r


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_misses_the_bar(mutant):
    kw, name = MUTANTS[mutant]
    c = CASES[name]
    fails = O.bar_failures(c, as_kernel(c, O.case_outputs(c, **kw(c))), O.case_outputs(c), O.case_sensitivity(c))
    assert fails, f"{mutant} passes every bar of {name}"
    print(f"{mutant}: rejected by {fails[0]}")


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_rounding_meets_the_bar(name):
    """the bars leave room for the kernels' own fp32 rounding of an exact float64 result"""
    c = CASES[name]
    ref = O.case_outputs(c)
    assert not O.bar_failures(c, as_kernel(c, ref), ref, O.case_sensitivity(c))


@pytest.mark.parametrize("p", [4, 5, 8, 12])
def test_each_distortion_coefficient_moves_points_by_1e_2(p):
    for i in range(p):
        c = CASES[f"dist_P{p}_{O.DIST_NAMES[i]}"]
        x = c.x
        assert (x["dist"] != 0).sum(-1).max() == 1 and (x["dist"][1, 1] == 0).all() and torch.signbit(x["dist"][1, 1]).all()
        moved = O.project_points_ref(x["points3d"], x["K"], x["E"], x["dist"]) - O.project_points_ref(x["points3d"], x["K"], x["E"], 0 * x["dist"])
        assert float((moved[:, [0, 2]].abs() / x["K"][:, [0, 2], 0, 0][:, :, None, None]).max()) >= 1e-2, O.DIST_NAMES[i]


def test_divergence_case_has_no_fixed_point():
    """past the turn-over the 5 iterations do not undistort: re-distorting misses the keypoints by pixels"""
    x = CASES["distortion_divergence"].x
    eye = torch.eye(3, dtype=torch.float64).expand(*x["K"].shape[:2], 3, 3)
    und = O.undistort_points(x["points"], x["K"], x["dist"], new_K=eye)
    back = O.distort_points(und, eye, x["dist"], new_K=eye) * x["K"][..., 0:1, 0, None] + x["K"][..., None, 0:2, 2]
    miss = (back - x["points"]).norm(dim=-1)
    assert torch.isfinite(und).all() and float(miss.max()) > 10.0 and float(miss.min()) < 1e-2


def test_dehomogenisation_cases_cross_the_switch():
    """|v3| runs through 1e-2 .. 1e-9 (both sides of 1e-8); camera-0 depths sit at 0, inside +-1e-8, just past it
    and behind the camera"""
    v3 = CASES["dehomog_far_points"].v3
    assert float(v3.max()) > 9e-3 and float(v3.min()) <= 1e-9 and ((v3 > 1e-8) & (v3 < 2e-8)).any() and ((v3 < 1e-8) & (v3 > 5e-9)).any()
    z = CASES["dehomog_principal_plane"].x["points3d"][..., 2]
    assert (z == 0).any() and ((z.abs() < 1e-8) & (z != 0)).any() and ((z > 1e-8) & (z < 2e-8)).any() and (z < -1e-8).any()


# ---- refusals, no GPU ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["fresh", "zero_width_slice"])
def test_project_points_refuses_an_empty_pair_axis(how):
    """n_pairs = 0 tells the kernels there is no pair axis: (B, 0, K, 3) would project the first B K points of
    whatever the pointer holds.  Refused before the device check, so CPU tensors reach it."""
    from lightning_pose_b200 import ops

    p3 = torch.zeros(2, 0, 5, 3) if how == "fresh" else torch.rand(2, 3, 5, 3)[:, :0]
    K, E, D = torch.eye(3).expand(2, 3, 3, 3), torch.zeros(2, 3, 3, 4), torch.zeros(2, 3, 5)
    with pytest.raises(ValueError, match="no pairs to average over"):
        ops.project_points(p3, K, E, D, mean_over_pairs=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):  # a non-empty pair axis gets to the device check
        ops.project_points(torch.zeros(2, 1, 5, 3), K, E, D, mean_over_pairs=True)


def test_more_than_64_views_is_refused():
    """CAM_MAX_VIEWS = 64: every entry that takes V refuses 65 with LPB_ERR_INVALID (dummy pointers: nothing may be
    launched)"""
    from lightning_pose_b200 import _lib

    L, p = _lib.lib, ctypes.c_void_p(16)
    for rc in (
        L.lpb_triangulate_pairs_fwd(p, p, p, p, 1, 65, 2, 5, p, None),
        L.lpb_triangulate_pairs_bwd(p, p, p, p, p, 1, 65, 2, 5, p, None),
        L.lpb_project_points_fwd(p, 0, p, p, p, None, 0.0, 0.0, 1, 65, 2, 5, p, None),
        L.lpb_project_points_bwd(p, 0, p, p, p, None, 0.0, 0.0, p, 1, 65, 2, 5, p, None),
    ):
        assert rc == -1 and b"bad V (65)" in L.lpb_last_error()
