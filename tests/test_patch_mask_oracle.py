"""CPU: tests/golden/patch_mask.npz against the reference when its tree is present, PatchMasker's schedule, defaults and
surface against the file, and the argument checks of the two patch-masking ABI entries (csrc/patchmask.cu)."""
import ast
import ctypes
import filecmp
import inspect
import math
import os

import numpy as np
import pytest
import torch

import patch_mask_oracle as O
from oracle import ref_loader as R

CASES = [c[0] for c in O.CASES]


def masker_for(row):
    from lightning_pose_b200.callbacks import PatchMasker

    init_step, final_step, r0, r1 = row
    return PatchMasker({"init_step": int(init_step), "final_step": int(final_step), "init_ratio": float(r0), "final_ratio": float(r1)})


# ---- goldens ---------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not O.reference_tree_available(), reason="needs the reference tree to regenerate the goldens")
def test_regenerating_patch_mask_golden_is_byte_identical(tmp_path):
    O.main(str(tmp_path / "patch_mask.npz"))
    assert filecmp.cmp(O.GOLDEN_PATH, str(tmp_path / "patch_mask.npz"), shallow=False)


@pytest.mark.parametrize("name", CASES)
def test_golden_case_is_the_masking_contract(golden, name):
    """The reference's masked images are its inputs with the mask's zero patches zeroed, and each view masks
    int(ratio * P) patches, where the ratio is the schedule's."""
    g = golden("patch_mask")
    x, out, mask = g[f"case_{name}_in_images"], g[f"case_{name}_out_images"], g[f"case_{name}_out_mask"]
    b, v, _, h, w = x.shape
    ph, pw = h // 16, w // 16
    assert mask.shape == (b, v, ph * pw) and set(np.unique(mask)) <= {0.0, 1.0}
    keep = np.ones((b, v, 1, h, w), bool)
    keep[..., : 16 * ph, : 16 * pw] = np.repeat(np.repeat(mask.reshape(b, v, 1, ph, pw), 16, 3), 16, 4) != 0
    bits = (lambda a: a.view(np.uint32)) if x.dtype == np.float32 else (lambda a: a)
    np.testing.assert_array_equal(bits(out), np.where(keep, bits(x), 0))
    m = masker_for(g["case_in_config"]).patches_to_mask(int(g[f"case_{name}_in_step"]), ph * pw)
    assert ((mask == 0).sum(-1) == m).all()


def test_golden_covers_the_issue_cases(golden):
    g = golden("patch_mask")
    init_step, final_step = g["case_in_config"][:2]
    steps = {int(g[f"case_{n}_in_step"]) for n in CASES}
    assert min(steps) < init_step and init_step in steps and max(steps) > final_step and any(init_step < s < final_step for s in steps)
    shapes = [g[f"case_{n}_in_images"].shape for n in CASES]
    assert {s[1] for s in shapes} == {1, 4, 6}
    assert any(s[3] % 16 == 0 and s[4] % 16 == 0 for s in shapes) and any(s[3] % 16 and s[4] % 16 for s in shapes)
    assert (200, 180) in {s[3:] for s in shapes}
    assert {g[f"case_{n}_in_images"].dtype for n in CASES} == {np.dtype(np.float32), np.dtype(np.uint16)}
    # the sweep holds products ratio * P just below an integer, where int() and round() differ
    prod = g["sched_ratio"] * g["sched_P"]
    assert ((prod != np.round(prod)) & (np.abs(prod - np.round(prod)) < 1e-9) & (g["sched_m"] < np.round(prod))).any()


def test_schedule_matches_golden(golden):
    g = golden("patch_mask")
    for i in range(len(g["sched_step"])):
        masker = masker_for(g["sched_config"][i])
        step, p = int(g["sched_step"][i]), int(g["sched_P"][i])
        assert masker.mask_ratio(step) == g["sched_ratio"][i], i  # bit for bit
        assert masker.patches_to_mask(step, p) == g["sched_m"][i], i
        info = masker.get_training_schedule_info(step)
        assert info == {"step": step, "mask_ratio": g["sched_ratio"][i], "curriculum_progress": str(g["sched_progress"][i]),
                        "steps_to_patch_masking": g["sched_to_start"][i], "steps_to_max_masking": g["sched_to_max"][i]}, i
        assert masker.should_start_patch_masking(step) == (step == masker.patch_init_step)


def test_kernel_arithmetic_restated_in_fp64_matches_golden(golden):
    """patches_to_mask of csrc/patchmask.cu: each operation rounded once (no fused multiply-add), as Python rounds."""
    g = golden("patch_mask")
    for i in range(len(g["sched_step"])):
        init_step, final_step, r0, r1 = g["sched_config"][i]
        step, p = int(g["sched_step"][i]), int(g["sched_P"][i])
        if step < init_step:
            m = 0
        else:
            progress = min(np.float64(step - init_step) / np.float64(final_step - init_step), 1.0)
            x = (np.float64(r0) + progress * (np.float64(r1) - np.float64(r0))) * np.float64(p)
            m = 0 if not x > 0 else min(int(x), p)
        assert m == g["sched_m"][i], i


def test_defaults_and_disabled_shapes_match_golden(golden):
    from lightning_pose_b200.callbacks import PatchMasker

    g = golden("patch_mask")
    d = PatchMasker()
    assert [d.patch_init_step, d.patch_final_step, d.patch_init_ratio, d.patch_final_ratio] == g["defaults"].tolist()
    assert d.use_patch_masking and d.patch_seed == 0
    b, v = g["disabled_out_mask_shape"][:2]
    assert g["eval_out_mask_shape"].tolist() == [b, v, (72 // 16) * (88 // 16)] and (g["eval_out_mask"] == 1).all()
    assert g["disabled_out_mask_shape"].tolist() == [b, v] and (g["disabled_out_mask"] == 1).all()


# ---- Python surface, no GPU ------------------------------------------------------------------------------------------
def test_patch_masker_constructor():
    from lightning_pose_b200.callbacks import PatchMasker

    with pytest.raises(ValueError, match="final_step > init_step"):
        PatchMasker({"init_step": 100, "final_step": 100})
    with pytest.raises(ValueError, match="final_step > init_step"):
        PatchMasker({"init_step": 100, "final_step": 50, "final_ratio": 0.3})
    off = PatchMasker({"init_step": 100, "final_step": 100, "final_ratio": 0.0})  # disabled: nothing divides
    assert not off.use_patch_masking and not off.should_start_patch_masking(100)
    assert off.get_training_schedule_info(5) == {"step": 5, "mask_ratio": 0.0, "curriculum_progress": "0.0%",
                                                 "steps_to_patch_masking": 0, "steps_to_max_masking": 0}
    assert PatchMasker(patch_seed=None).patch_seed is None


def test_epoch_to_step_conversion():
    """train.py:335-340: ceil(epoch * steps_per_epoch); the default multi-view config's curriculum is in epochs."""
    from lightning_pose_b200.callbacks import patch_mask_steps_from_epochs

    cfg = {"init_epoch": 2.5, "final_epoch": 30, "init_ratio": 0.1, "final_ratio": 0.5}
    out = patch_mask_steps_from_epochs(cfg, 7)
    assert out["init_step"] == math.ceil(2.5 * 7) == 18 and out["final_step"] == 210 and out["final_ratio"] == 0.5
    assert "init_step" not in cfg  # the input is not modified
    assert patch_mask_steps_from_epochs({"init_step": 3, "final_step": 9}, 7) == {"init_step": 3, "final_step": 9}


def test_patch_masker_refuses_cpu_tensors():
    from lightning_pose_b200.callbacks import PatchMasker

    x = torch.zeros(1, 2, 3, 32, 32)
    for call in (lambda: PatchMasker().apply_patch_masking(x, 800), lambda: PatchMasker().apply_patch_masking(x, 800, is_training=False),
                 lambda: PatchMasker().apply_masking(x, 800)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()


def test_patch_masker_names_match_reference():
    from lightning_pose_b200.callbacks import PatchMasker
    from lightning_pose_b200.models.heatmap_tracker import HeatmapTracker
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    sig = lambda f: list(inspect.signature(f).parameters)
    assert sig(PatchMasker.__init__) == ["self", "patch_mask_config", "patch_seed"]
    assert sig(PatchMasker.apply_patch_masking) == ["self", "images", "training_step", "is_training"]
    assert sig(PatchMasker.apply_masking) == ["self", "images", "training_step", "is_training"]
    assert sig(HeatmapTrackerMultiviewTransformer.training_step) == sig(HeatmapTracker.training_step)
    assert "patch_masker" in sig(HeatmapTrackerMultiviewTransformer.__init__)
    path = os.path.join(R.REF_ROOT, "lightning_pose", "callbacks.py")
    if os.path.isfile(path):
        cls = [n for n in ast.parse(open(path).read()).body if isinstance(n, ast.ClassDef) and n.name == "PatchMasker"][0]
        fns = {n.name: [a.arg for a in n.args.args] for n in cls.body if isinstance(n, ast.FunctionDef)}
        for name, args in fns.items():
            assert sig(getattr(PatchMasker, name)) == args, name


def test_multiview_tracker_step_counter_is_not_state():
    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    tr = HeatmapTrackerMultiviewTransformer(3, 2, torch.nn.Identity(), torch.nn.Identity(), 8)
    assert tr.global_step.tolist() == [0] and tr.global_step.dtype == torch.int64
    assert "global_step" not in tr.state_dict() and tr.patch_masker is None and tr.current_patch_mask is None


# ---- ABI, no GPU -------------------------------------------------------------------------------------------------------
def test_patch_mask_entry_points_validate_without_gpu():
    from lightning_pose_b200 import _lib

    L, p = _lib.lib, ctypes.c_void_p(16)
    sel = lambda **kw: L.lpb_patch_mask_select(*[kw.get(k, v) for k, v in (
        ("step", p), ("B", 2), ("V", 4), ("H", 64), ("W", 80), ("seed", 7), ("init", 10), ("final", 50), ("r0", 0.1), ("r1", 0.5),
        ("mask", p), ("stream", None))])
    for kw in ({"step": None}, {"mask": None}):
        assert sel(**kw) == -1 and b"null pointer" in L.lpb_last_error(), kw
    for kw in ({"B": -1}, {"V": -1}, {"H": -16}, {"V": 65536}):
        assert sel(**kw) == -1 and b"bad shape" in L.lpb_last_error(), kw
    assert sel(H=1040, W=1024) == -1 and b"4160 patches per view; at most 4096" in L.lpb_last_error()
    assert sel(init=50) == -1 and b"final_step" in L.lpb_last_error()
    assert sel(r1=float("nan")) == -1 and b"NaN" in L.lpb_last_error()
    assert sel(B=0) == 0 and sel(H=15) == 0 and sel(H=1024, W=1024, V=0) == 0  # nothing to draw: no launch

    q = ctypes.c_void_p(1 << 30)
    app = lambda **kw: L.lpb_patch_mask_apply(*[kw.get(k, v) for k, v in (
        ("images", p), ("B", 2), ("V", 4), ("C", 3), ("H", 64), ("W", 80), ("fmt", 0), ("mask", p), ("out", q), ("stream", None))])
    for kw in ({"images": None}, {"out": None}, {"mask": None}):
        assert app(**kw) == -1 and b"null pointer" in L.lpb_last_error(), kw
    for kw in ({"B": -1}, {"C": -1}, {"W": -1}, {"H": 65536, "W": 65536}):
        assert app(**kw) == -1 and b"bad shape" in L.lpb_last_error(), kw
    for fmt in (2, 3, -1):
        assert app(fmt=fmt) == -1 and b"format" in L.lpb_last_error()
    assert app(H=1024, W=1040) == -1 and b"at most 4096" in L.lpb_last_error()
    assert app(out=ctypes.c_void_p(16 + 4 * 64 * 80)) == -1 and b"alias" in L.lpb_last_error()
    assert app(B=0) == 0 and app(H=8, mask=None, B=0) == 0
