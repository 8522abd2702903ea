"""CPU: the context-prediction row rule (what lpb_pack_context_predictions implements) against the reference's own
reader / unpack / fix-up functions and against tests/golden/context_predict.npz, plus the new ABI entry's argument
checks and the Python surface without a GPU."""
import ctypes
import filecmp
import inspect

import numpy as np
import pytest
import torch

import context_predict_oracle as O

CASES = [c[0] for c in O.CASES]
NEEDS_REF = pytest.mark.skipif(not O.reference_tree_available(), reason="needs the reference tree")


def _stored(g):
    return sorted({k[: -len("_meta")] for k in g.files if k.endswith("_meta")})


def test_golden_covers_the_row_rule_cases(golden):
    g = golden("context_predict")
    seen = set()
    for p in _stored(g):
        n, s, uf = (int(v) for v in g[f"{p}_meta"][:3])
        t = s - 4
        r = n if t == 1 else t * (-(-(n - s) // t) + 1)
        seen.add(("R>=N" if r >= n else "R<N", uf))
        seen |= {("R=N-1", uf)} if r == n - 1 else set()
        seen |= {("N=5", uf)} if n == 5 else set()
        seen |= {("N<S", uf)} if n < s else set()
    for uf in (1, 2):
        assert {("R>=N", uf), ("R<N", uf), ("R=N-1", uf), ("N=5", uf), ("N<S", uf)} <= seen


def test_row_rule_matches_stored_row_maps(golden):
    g = golden("context_predict")
    for p in _stored(g):
        n, s = (int(v) for v in g[f"{p}_meta"][:2])
        np.testing.assert_array_equal(O.row_rule(n, s), g[f"{p}_rows"], err_msg=p)


def test_row_rule_issue_example():
    rows = O.row_rule(100, 16)  # R = 96 < 100: the last four rows repeat frame 2
    assert list(rows[:3]) == [2, 2, 2] and list(rows[94:]) == [94, 95, 2, 2, 2, 2]
    rows = O.row_rule(25, 12)  # R = 24 = N - 1: row 23 is frame 23 (its window reaches frame 25, the padding)
    assert list(rows[21:]) == [21, 22, 23, 2]
    rows = O.row_rule(30, 12)  # R = 32 >= N: both edges replicate
    assert list(rows[:3]) == [2, 2, 2] and list(rows[-4:]) == [26, 27, 27, 27]


@NEEDS_REF
def test_row_rule_matches_reference_source():
    fns = O.source_functions()
    for n in range(5, 121):
        for s in range(5, 41):
            np.testing.assert_array_equal(O.row_rule(n, s), O.reference_row_map(fns, n, s), err_msg=f"N={n} S={s}")


@NEEDS_REF
def test_reference_has_no_window_below_five_frames():
    fns = O.source_functions()
    for n in range(1, 5):
        assert O.num_iters(fns, n, 12) <= 0
        with pytest.raises(RuntimeError):  # torch.vstack of no windows
            O.reference_row_map(fns, n, 12)


@NEEDS_REF
def test_regenerating_context_golden_is_byte_identical(tmp_path):
    O.main(str(tmp_path / "context_predict.npz"))
    assert filecmp.cmp(O.GOLDEN_PATH, str(tmp_path / "context_predict.npz"), shallow=False)


# ---- ABI, no GPU --------------------------------------------------------------------------------------------------------
def test_pack_context_entry_validates_without_gpu():
    from lightning_pose_b200 import _lib

    L, p = _lib.lib, ctypes.c_void_p(16)
    call = lambda **kw: L.lpb_pack_context_predictions(*[kw.get(k, v) for k, v in (
        ("kp_sf", p), ("cf_sf", p), ("kp_mf", p), ("cf_mf", p), ("n", 4), ("K", 3), ("bbox", p), ("mh", 64.0), ("mw", 64.0),
        ("table", p), ("n_rows", 10), ("cursor", None), ("frame0", 0), ("step", 4), ("stream", None))])
    for kw in ({"kp_sf": None}, {"cf_sf": None}, {"kp_mf": None}, {"cf_mf": None}, {"bbox": None}, {"table": None}):
        assert call(**kw) == -1 and b"null pointer" in L.lpb_last_error(), kw
    for kw in ({"n": -1}, {"K": 0}):
        assert call(**kw) == -1 and b"bad shape" in L.lpb_last_error(), kw
    assert call(n_rows=4) == -1 and b"at least 5 frames" in L.lpb_last_error()
    assert call(step=0) == -1 and b"step" in L.lpb_last_error()
    assert call(mh=0.0) == -1 and b"model dims" in L.lpb_last_error()
    assert call(frame0=-1) == -1 and b"frame0" in L.lpb_last_error()
    assert call(n=0) == 0  # nothing to do: no launch


def test_pack_context_wrapper_refuses_cpu_tensors():
    from lightning_pose_b200 import ops

    kp, cf, bb = torch.zeros(4, 6), torch.zeros(4, 3), torch.ones(4, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.pack_context_predictions(kp, cf, kp, cf, bb, 64, 64, torch.zeros(10, 9), 4)


def test_context_predictor_arguments():
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    head = HeatmapMHCRNNHead("vits_dino", 32, 3, upsampling_factor=1)
    with pytest.raises(ValueError, match="at least 5 frames"):  # the reference has no window (its vstack of none fails)
        BatchedPredictor(head, 3, 4, 8, (64, 64), device="cpu")
    with pytest.raises(ValueError, match="not supported for multiview"):
        BatchedPredictor(head, 3, 20, 8, (64, 64), device="cpu", num_views=2)
    with pytest.raises(ValueError, match="chunk"):
        BatchedPredictor(head, 3, 20, 0, (64, 64), device="cpu")
    bp = BatchedPredictor(head, 3, 20, 8, (64, 64), device="cpu")
    assert bp.context and bp._kp_sf.shape == (10, 6) and bp._box.shape == (10, 4)
    assert bp._idx.tolist()[:2] == [[0, 1, 2, 3, 4], [1, 2, 3, 4, 5]]


def test_dataframe_frame_aligned_keyword():
    from lightning_pose_b200.utils.predictions import PredictionHandler

    assert inspect.signature(PredictionHandler.dataframe).parameters["frame_aligned"].default is False
    n, k = 9, 2
    table = np.arange(n * 3 * k, dtype=np.float64).reshape(n, 3 * k)
    ph = PredictionHandler(["a", "b"], n, model_type="heatmap_mhcrnn")
    np.testing.assert_array_equal(ph.dataframe(table, frame_aligned=True).to_numpy(), table)
    shifted = ph.dataframe(table).to_numpy()  # default: the reference's shift-and-fill of a row-per-window table
    np.testing.assert_array_equal(shifted[2], table[0])
    np.testing.assert_array_equal(shifted[-1], table[n - 5])
