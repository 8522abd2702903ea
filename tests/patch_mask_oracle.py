"""Golden generator for curriculum patch masking.  TEST INFRASTRUCTURE ONLY.

``python tests/patch_mask_oracle.py`` writes ``tests/golden/patch_mask.npz`` by running the reference's own, unmodified
``PatchMasker`` (``lightning_pose/callbacks.py:279-459``, loaded through ``oracle/ref_loader.py``) on the CPU.
``callbacks.py`` imports Lightning's ``Callback``, ``EarlyStopping``, ``LearningRateMonitor``, ``ModelCheckpoint``,
``LightningModule`` and ``Trainer``; ``PatchMasker`` uses none of them, so they are placeholder names here.  Needs the full
reference tree; the GPU tests only read the committed npz.  Nothing under ``lightning_pose_b200/`` imports this module.

Cases
  case_<name>:  images (B, V, 3, H, W) (fp32, or bf16 stored as its uint16 bits) with a few NaN and -0.0 entries, a
                curriculum config (init_step, final_step, init_ratio, final_ratio), patch_seed and step; the reference's
                mask (B, V, P) and masked images (same storage as the input).
  eval_/disabled_: the not-training call and apply_masking with final_ratio = 0: the reference's mask shapes.
  sched_*:      a sweep of (config, P, step) -> the reference's mask ratio (get_training_schedule_info), the number of
                patches its apply_patch_masking zeroes per view, and the rest of get_training_schedule_info.
  defaults:     PatchMasker()'s init_step, final_step, init_ratio, final_ratio.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "patch_mask.npz")

CURRICULUM = {"init_step": 10, "final_step": 50, "init_ratio": 0.1, "final_ratio": 0.5}
# (name, dtype, B, V, H, W, step): H and W multiples of 16 and not; 1, 4 and 6 views; steps before, at, between and past
# the curriculum
CASES = [
    ("f32_v1_mult", torch.float32, 2, 1, 64, 80, 30),
    ("f32_v4_odd", torch.float32, 1, 4, 72, 88, 30),
    ("f32_v6_mult", torch.float32, 1, 6, 48, 64, 80),
    ("f32_v1_200x180", torch.float32, 1, 1, 200, 180, 10),
    ("f32_v4_before", torch.float32, 1, 4, 48, 64, 5),
    ("bf16_v4_mult", torch.bfloat16, 2, 4, 64, 80, 30),
    ("bf16_v6_odd", torch.bfloat16, 1, 6, 72, 88, 80),
    ("bf16_v1_200x180", torch.bfloat16, 1, 1, 200, 180, 40),
    ("bf16_v4_at", torch.bfloat16, 1, 4, 72, 88, 10),
]
PATCH_SEED = 7

# schedule sweep: (config, patch counts, steps)
SCHED = [
    ({}, (1, 20, 132, 576, 4096), (0, 699, 700, 701, 1000, 2850, 4999, 5000, 5001, 20000)),
    (CURRICULUM, (6, 20, 100, 132), tuple(range(0, 61, 3))),
    # ratio = step / 100 on P = 100 and 50: ratio * P lands on or next to an integer (0.07 * 100 = 7.000000000000001,
    # 0.29 * 100 = 28.999999999999996, ...)
    ({"init_step": 0, "final_step": 100, "init_ratio": 0.0, "final_ratio": 1.0}, (25, 50, 100), tuple(range(0, 102))),
    ({"init_step": 3, "final_step": 7, "init_ratio": 0.3, "final_ratio": 0.7}, (10, 30, 1000), tuple(range(0, 10))),
    ({"init_step": 0, "final_step": 3, "init_ratio": 0.0, "final_ratio": 0.9}, (10, 30, 1000), (0, 1, 2, 3, 4)),
    # final_ratio below init_ratio: a shrinking curriculum
    ({"init_step": 2, "final_step": 12, "init_ratio": 0.6, "final_ratio": 0.2}, (20, 132), (0, 2, 5, 7, 12, 13)),
]


def reference_tree_available() -> bool:
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return os.path.isfile(os.path.join(R.REF_ROOT, "lightning_pose", "callbacks.py"))


def load_reference():
    """The reference's ``lightning_pose/callbacks.py``, loaded unmodified."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    R.install()
    placeholders = {n: type(n, (), {"__init__": lambda self, *a, **k: None})
                    for n in ("Callback", "EarlyStopping", "LearningRateMonitor", "ModelCheckpoint", "Trainer")}
    light = sys.modules["lightning"]
    light.LightningModule, light.Trainer = torch.nn.Module, placeholders["Trainer"]  # type: ignore[attr-defined]
    cb = types.ModuleType("lightning.pytorch.callbacks")
    for n in ("Callback", "EarlyStopping", "LearningRateMonitor", "ModelCheckpoint"):
        setattr(cb, n, placeholders[n])
    sys.modules["lightning.pytorch.callbacks"] = cb
    sys.modules["lightning.pytorch"].callbacks = cb  # type: ignore[attr-defined]
    return importlib.import_module("lightning_pose.callbacks")


def images_for(dtype, b, v, h, w, seed: int) -> torch.Tensor:
    """Values in {-1, -0.5, 0, 0.5} (exact in bf16; the file compresses), a few NaN and -0.0."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randint(-2, 2, (b, v, 3, h, w), generator=gen).float() / 2.0
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=gen)[:24]
    flat[idx[:12]] = float("nan")
    flat[idx[12:]] = -0.0
    return x.to(dtype)


def as_stored(t: torch.Tensor) -> np.ndarray:
    return t.view(torch.int16).numpy().view(np.uint16) if t.dtype == torch.bfloat16 else t.numpy()


def gen_cases(cbm) -> dict:
    g = {}
    masker = cbm.PatchMasker(patch_mask_config=dict(CURRICULUM), patch_seed=PATCH_SEED)
    for i, (name, dtype, b, v, h, w, step) in enumerate(CASES):
        x = images_for(dtype, b, v, h, w, 500 + i)
        out, mask = masker.apply_patch_masking(x, training_step=step, is_training=True)
        g[f"case_{name}_in_images"], g[f"case_{name}_out_images"] = as_stored(x), as_stored(out)
        g[f"case_{name}_in_step"] = np.asarray(step, np.int64)
        g[f"case_{name}_out_mask"] = mask.numpy()
    g["case_in_config"] = np.asarray([CURRICULUM[k] for k in ("init_step", "final_step", "init_ratio", "final_ratio")], np.float64)
    g["case_in_seed"] = np.asarray(PATCH_SEED, np.int64)
    x = images_for(torch.float32, 2, 4, 72, 88, 600)
    same, mask = masker.apply_patch_masking(x, training_step=30, is_training=False)
    assert same is x
    g["eval_out_mask_shape"] = np.asarray(mask.shape, np.int64)
    g["eval_out_mask"] = mask.numpy()
    off = cbm.PatchMasker(patch_mask_config={**CURRICULUM, "final_ratio": 0.0}, patch_seed=PATCH_SEED)
    same, mask = off.apply_masking(x, training_step=30, is_training=True)
    assert same is x and not off.use_patch_masking
    g["disabled_out_mask_shape"] = np.asarray(mask.shape, np.int64)
    g["disabled_out_mask"] = mask.numpy()
    return g


def gen_schedule(cbm) -> dict:
    rows = {k: [] for k in ("config", "P", "step", "ratio", "m", "progress", "to_start", "to_max")}
    for cfg, counts, steps in SCHED:
        masker = cbm.PatchMasker(patch_mask_config=dict(cfg), patch_seed=0)
        full = [masker.patch_init_step, masker.patch_final_step, masker.patch_init_ratio, masker.patch_final_ratio]
        for p in counts:
            img = torch.zeros(1, 1, 1, 16, 16 * p) + 1.0  # one row of p patches, one channel
            for s in steps:
                _, mask = masker.apply_patch_masking(img, training_step=s, is_training=True)
                info = masker.get_training_schedule_info(s)
                assert info["step"] == s
                rows["config"].append(full)
                rows["P"].append(p)
                rows["step"].append(s)
                rows["ratio"].append(info["mask_ratio"])
                rows["m"].append(int((mask == 0).sum()))
                rows["progress"].append(info["curriculum_progress"])
                rows["to_start"].append(info["steps_to_patch_masking"])
                rows["to_max"].append(info["steps_to_max_masking"])
    g = {
        "sched_config": np.asarray(rows["config"], np.float64),
        "sched_P": np.asarray(rows["P"], np.int64),
        "sched_step": np.asarray(rows["step"], np.int64),
        "sched_ratio": np.asarray(rows["ratio"], np.float64),
        "sched_m": np.asarray(rows["m"], np.int64),
        "sched_progress": np.asarray(rows["progress"], dtype="<U8"),
        "sched_to_start": np.asarray(rows["to_start"], np.int64),
        "sched_to_max": np.asarray(rows["to_max"], np.int64),
    }
    d = cbm.PatchMasker()
    g["defaults"] = np.asarray([d.patch_init_step, d.patch_final_step, d.patch_init_ratio, d.patch_final_ratio], np.float64)
    return g


def main(path: str = GOLDEN_PATH) -> None:
    assert reference_tree_available(), "needs the full reference tree (lightning_pose/callbacks.py)"
    cbm = load_reference()
    with torch.no_grad():
        arrays = gen_cases(cbm)
        arrays.update(gen_schedule(cbm))
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: {len(arrays)} arrays, {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main(*sys.argv[1:])
