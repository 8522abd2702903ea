"""Curriculum patch masking of multi-view transformer training: ``PatchMasker`` of ``lightning_pose/callbacks.py:279-459``.

The reference's ``PatchMasking`` callback (:199-276) masks the images of every training batch of a
``heatmap_multiview_transformer`` before the forward pass (``get_callbacks`` :718-726 installs it; the default multi-view
config turns it on).  Lightning is not used here, so the callback's work is done by
``HeatmapTrackerMultiviewTransformer.training_step`` with a ``PatchMasker`` attached (``patch_masker=``).

``PatchMasker`` keeps the reference's constructor, defaults, attributes and methods.  ``apply_patch_masking`` runs two
kernels (``csrc/patchmask.cu``): one draws every view's patch mask from the step held in device memory, one zeroes the
masked patches of the whole batch.  Nothing synchronises with the host, so a training step that masks captures into a
CUDA graph and replays with its step advancing.

Divergences from the reference:
  * the patches chosen differ: each view masks the same number of patches, ``int(ratio * P)``, as a uniformly random
    subset fixed by (``patch_seed``, step, example, view) through a counter-based generator, where the reference seeds
    ``torch.randperm`` with ``patch_seed + step + 1000 b + 100 v`` (which repeats: step 1000 of example 0 draws what step
    0 of example 1 draws);
  * ``final_step <= init_step`` with masking enabled raises at construction (the reference divides by zero at the first
    masked step);
  * more than 4096 patches per view (images past 1024 x 1024) raise.
"""
from __future__ import annotations

import logging
import math
from typing import Any

import torch

from lightning_pose_b200 import ops

__all__ = ["PatchMasker", "patch_mask_steps_from_epochs"]

logger = logging.getLogger(__name__)


def patch_mask_steps_from_epochs(patch_mask_config: dict, steps_per_epoch: int) -> dict:
    """``init_epoch`` / ``final_epoch`` -> ``init_step`` / ``final_step`` = ceil(epoch * steps_per_epoch), as
    ``lightning_pose/train.py:335-340`` converts the default config's curriculum; a config without ``init_epoch`` is
    returned unchanged."""
    cfg = dict(patch_mask_config)
    if "init_epoch" in cfg:
        cfg["init_step"] = math.ceil(cfg["init_epoch"] * steps_per_epoch)
        cfg["final_step"] = math.ceil(cfg["final_epoch"] * steps_per_epoch)
    return cfg


class PatchMasker:
    """Curriculum masking of 16 x 16 image patches (reference ``callbacks.py:279-459``).

    ``patch_mask_config`` keys (defaults): ``init_step`` (700), ``final_step`` (5000), ``init_ratio`` (0.1),
    ``final_ratio`` (0.5).  No masking before ``init_step``; from there the ratio grows linearly from ``init_ratio`` to
    ``final_ratio`` at ``final_step`` and stays there.  Masking is on when ``final_ratio > 0``."""

    patch_size = ops.PATCH_SIZE

    def __init__(self, patch_mask_config: dict | None = None, patch_seed: int | None = 0) -> None:
        self.patch_seed = patch_seed
        if patch_mask_config is None:
            patch_mask_config = {}
        self.patch_init_step = patch_mask_config.get("init_step", 700)
        self.patch_final_step = patch_mask_config.get("final_step", 5000)
        self.patch_init_ratio = patch_mask_config.get("init_ratio", 0.1)
        self.patch_final_ratio = patch_mask_config.get("final_ratio", 0.5)
        self.use_patch_masking = self.patch_final_ratio > 0.0
        if self.use_patch_masking and patch_seed is None:
            logger.warning("patch_seed is None but patch masking is enabled; results may not be reproducible")
        if self.use_patch_masking and not self.patch_final_step > self.patch_init_step:
            raise ValueError(f"patch masking needs final_step > init_step; got init_step={self.patch_init_step}, "
                             f"final_step={self.patch_final_step}")

    # ---- the curriculum (callbacks.py:344-357), on the host ---------------------------------------------------------
    def mask_ratio(self, training_step: int) -> float:
        """The fraction of patches masked at ``training_step``."""
        if training_step < self.patch_init_step:
            return 0.0
        curr_steps_for_patch = self.patch_final_step - self.patch_init_step
        progress = min((training_step - self.patch_init_step) / curr_steps_for_patch, 1.0)
        return self.patch_init_ratio + progress * (self.patch_final_ratio - self.patch_init_ratio)

    def patches_to_mask(self, training_step: int, num_patches: int) -> int:
        """Patches masked per view at ``training_step`` out of ``num_patches``: what the selection kernel computes."""
        return min(max(int(self.mask_ratio(training_step) * num_patches), 0), num_patches)

    # ---- masking ---------------------------------------------------------------------------------------------------
    def apply_patch_masking(
        self,
        images: torch.Tensor,
        training_step: int | torch.Tensor = 0,
        is_training: bool = True,
    ) -> tuple[torch.Tensor, torch.Tensor]:
        """(B, V, C, H, W) fp32 / bf16 CUDA images -> (masked images, patch mask (B, V, P) fp32, 1 = kept).

        ``training_step``: an int, or a one-element int64 tensor on the images' device that the kernel reads (a captured
        graph then masks with whatever step the tensor holds at replay).  Not training: the images themselves and an
        all-ones mask.  Otherwise the masked images are a new tensor; the input is not modified.  The kernel refuses
        ``final_step <= init_step`` (which the constructor only rejects with masking enabled)."""
        b, v, _, h, w = ops._patch_images(images)
        num_patches = (h // self.patch_size) * (w // self.patch_size)
        if not is_training:
            return images, torch.ones(b, v, num_patches, device=images.device)
        if isinstance(training_step, torch.Tensor):
            step = training_step
        else:  # a fill kernel, not a host copy: graph-capturable as well
            step = torch.full((1,), int(training_step), dtype=torch.int64, device=images.device)
        # the schedule applies whether or not use_patch_masking is set, as in the reference (apply_masking checks it)
        seed = 0 if self.patch_seed is None else int(self.patch_seed)
        mask = ops.patch_mask_select(images, step, seed, int(self.patch_init_step), int(self.patch_final_step),
                                     float(self.patch_init_ratio), float(self.patch_final_ratio))
        return ops.patch_mask_apply(images, mask), mask

    def apply_masking(
        self,
        images: torch.Tensor,
        training_step: int | torch.Tensor = 0,
        is_training: bool = True,
    ) -> tuple[torch.Tensor, torch.Tensor]:
        """``apply_patch_masking`` when masking is on; else the images and a (B, V) all-ones mask (:403-417)."""
        if self.use_patch_masking:
            return self.apply_patch_masking(images, training_step, is_training)
        return images, torch.ones(images.shape[0], images.shape[1], device=images.device)

    # ---- schedule reporting (callbacks.py:419-459) -------------------------------------------------------------------
    def get_training_schedule_info(self, current_step: int) -> dict[str, Any]:
        if self.use_patch_masking:
            if current_step < self.patch_init_step:
                current_mask_ratio = 0.0
                curriculum_progress = "0.0%"
                steps_to_patch_masking = self.patch_init_step - current_step
                steps_to_max_masking = self.patch_final_step - current_step
            else:
                curr_steps_for_patch = self.patch_final_step - self.patch_init_step
                progress = min((current_step - self.patch_init_step) / curr_steps_for_patch, 1.0)
                current_mask_ratio = self.patch_init_ratio + progress * (self.patch_final_ratio - self.patch_init_ratio)
                curriculum_progress = f"{progress * 100:.1f}%"
                steps_to_patch_masking = 0
                steps_to_max_masking = max(0, self.patch_final_step - current_step)
        else:
            current_mask_ratio = 0.0
            curriculum_progress = "0.0%"
            steps_to_max_masking = 0
            steps_to_patch_masking = 0
        return {
            "step": current_step,
            "mask_ratio": current_mask_ratio,
            "curriculum_progress": curriculum_progress,
            "steps_to_patch_masking": steps_to_patch_masking,
            "steps_to_max_masking": steps_to_max_masking,
        }

    def should_start_patch_masking(self, current_step: int) -> bool:
        return self.use_patch_masking and current_step == self.patch_init_step
