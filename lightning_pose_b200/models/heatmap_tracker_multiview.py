"""Multi-view transformer tracker: the hot-path part of ``lightning_pose/models/heatmap_tracker_multiview.py``.

``HeatmapTrackerMultiviewTransformer`` (:36-...) fuses the camera views inside the ViT: patch tokens of all views of
one example are concatenated into ONE attention sequence after a learnable per-view embedding is added
(``forward_vit`` :143-232), then every view's token grid goes through the SAME heatmap head and the per-view heatmaps are
folded into the channel dimension: (batch, views * K, h, w) (``forward`` :234-258).  Decode, model->frame remap and the
supervised / multi-view PCA losses then run on that folded tensor.

The transformer blocks themselves are the backbone (dense contractions supplied by a library module); this mirror owns
what sits on this repository's path: the view-embedding / token bookkeeping of ``forward_vit``, the head on
``views * batch`` feature maps (BASELINE config 4: (8 x 4, 384, 24, 24) -> (8, 68, 96, 96) through the banded tensor-core
kernels), the fold, and the loss inputs.  Calibrated batches (``keypoints_3d`` plus per-view intrinsics, extrinsics and
distortions) also get the 3-D entries the pairwise-projection and reprojection losses read (:263-303), computed by the
camera kernels without a host sync; uncalibrated batches get ``None`` there, as in the reference (:300-303).  Unlike
the reference, malformed camera inputs raise instead of being logged and turned into ``None``.

Training with curriculum patch masking (the reference's ``PatchMasking`` callback, ``callbacks.py:199-276``): pass a
``PatchMasker`` as ``patch_masker``; ``training_step`` then masks ``batch_dict["images"]`` at the step held by the device
counter ``global_step`` (0 at construction, one more after every ``training_step``, as Lightning's ``global_step``
advances once per optimizer step) and stores the mask in ``current_patch_mask``.  The step never leaves the device, so
a training step captured into a CUDA graph masks with a fresh step on every replay.

``SemiSupervisedHeatmapTrackerMultiviewTransformer`` (reference :370-484) adds the unlabeled multi-view video branch
and its unsupervised losses (``pca_multiview``, ``pca_singleview``, ``temporal``, ``temporal_heatmap_*``) with the anneal
weight held on the device, so its semi-supervised step captures into one CUDA graph as the labeled step does.
"""
from __future__ import annotations

import math
from typing import Any, Callable, Literal

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.callbacks import PatchMasker
from lightning_pose_b200.data.bboxes import model_to_frame_batch
from lightning_pose_b200.data.cameras import project_camera_pairs_to_3d
from lightning_pose_b200.data.heatmaps import GaussianTargets
from lightning_pose_b200.losses.factory import LossFactory
from lightning_pose_b200.losses.losses import RegressionRMSELoss
from lightning_pose_b200.models.backbones import tokens_to_feature_map
from lightning_pose_b200.models.heads.heatmap import HeatmapHead

__all__: list[str] = []


class HeatmapTrackerMultiviewTransformer(nn.Module):
    """Images (batch, views, 3, H, W) -> per-view heatmaps folded to (batch, views * K, h, w).

    ``patch_embed``: (views * batch, 3, H, W) -> (views * batch, N, D) patch tokens (position embeddings included, CLS
    removed); ``encoder``: (batch, views * N, D) -> same (the transformer blocks + final layer norm).
    """

    def __init__(
        self,
        num_keypoints: int,
        num_views: int,
        patch_embed: nn.Module | Callable,
        encoder: nn.Module | Callable,
        embedding_dim: int,
        loss_factory: LossFactory | None = None,
        backbone_arch: str = "vits_dino",
        downsample_factor: Literal[1, 2, 3] = 2,
        torch_seed: int = 123,
        patch_masker: PatchMasker | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__()
        torch.manual_seed(torch_seed)
        self.patch_masker = patch_masker
        self.current_patch_mask: torch.Tensor | None = None
        # training steps taken (Lightning's global_step), on the device; not part of the state dict
        self.register_buffer("global_step", torch.zeros(1, dtype=torch.int64), persistent=False)
        self.num_keypoints, self.num_views, self.downsample_factor = num_keypoints, num_views, downsample_factor
        self.num_fc_input_features = embedding_dim
        self.patch_embed, self.encoder = patch_embed, encoder
        generator = torch.Generator().manual_seed(torch_seed)
        self.view_embeddings = nn.Parameter(torch.randn(num_views, embedding_dim, generator=generator) * 0.02)
        self.head = HeatmapHead(backbone_arch=backbone_arch, in_channels=embedding_dim, out_channels=num_keypoints, downsample_factor=downsample_factor)
        self.loss_factory = loss_factory
        self.rmse_loss = RegressionRMSELoss()

    def forward_vit(self, images: torch.Tensor, channels_last: bool = False) -> torch.Tensor:
        """(view * batch, 3, H, W) -> (view * batch, D, h, w), views attending to each other (reference :143-232).

        Contiguous NCHW, as the reference returns it; with ``channels_last`` the same values as a view of the encoder's
        tokens (``tokens_to_feature_map``), which is what the head is fed: it reads them in place."""
        tokens = self.patch_embed(images)  # (view * batch, N, D)
        vb, n, d = tokens.shape
        batch = vb // self.num_views
        view_idx = torch.arange(self.num_views, device=tokens.device).repeat(batch)  # [0..V-1, 0..V-1, ...]
        tokens = tokens + self.view_embeddings[view_idx].to(tokens.dtype).unsqueeze(1)
        seq = self.encoder(tokens.reshape(batch, self.num_views * n, d))  # all views of an example in one sequence
        h_img, w_img = images.shape[-2:]
        patch = math.isqrt(h_img * w_img // n)  # square patches: n = (H / patch) * (W / patch), so H != W works too
        features = tokens_to_feature_map(seq.reshape(vb, n, d), (h_img // patch, w_img // patch))
        return features if channels_last else features.contiguous()

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        batch, views, c, h, w = images.shape
        heatmaps = self.head(self.forward_vit(images.reshape(-1, c, h, w), channels_last=True))
        return heatmaps.reshape(batch, -1, heatmaps.shape[-2], heatmaps.shape[-1])

    def forward_with_keypoints(self, images: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        batch, views, c, h, w = images.shape
        hm, kp, cf = self.head.forward_with_keypoints(self.forward_vit(images.reshape(-1, c, h, w), channels_last=True))
        return hm.reshape(batch, -1, hm.shape[-2], hm.shape[-1]), kp.reshape(batch, -1), cf.reshape(batch, -1)

    def get_loss_inputs_labeled(self, batch_dict: dict) -> dict:
        pred_heatmaps, pred_keypoints, confidence = self.forward_with_keypoints(batch_dict["images"])
        if "heatmaps" in batch_dict:  # reference flow: DataLoader workers rendered the targets
            heatmaps_targ = batch_dict["heatmaps"]
            target_keypoints = model_to_frame_batch(batch_dict, batch_dict["keypoints"])
        else:
            heatmaps_targ = self._keypoint_targets(batch_dict)
            target_keypoints = model_to_frame_batch(batch_dict, heatmaps_targ.keypoints.reshape(batch_dict["keypoints"].shape), in_place=False)
        pred_keypoints = model_to_frame_batch(batch_dict, pred_keypoints)
        keypoints_targ_3d = keypoints_pred_3d = keypoints_pred_2d_reprojected = None
        # calibrated batches (reference :263-303): triangulate every camera pair; with the reprojection loss registered,
        # also project the pair mean back into every view, in model coordinates (one launch: mean + project + frame->model)
        if "keypoints_3d" in batch_dict and batch_dict["keypoints_3d"].shape[-1] == 3:
            num_views = batch_dict["images"].shape[1]
            num_keypoints = pred_keypoints.shape[1] // 2 // num_views
            cameras = (batch_dict["intrinsic_matrix"], batch_dict["extrinsic_matrix"], batch_dict["distortions"])
            keypoints_pred_3d = project_camera_pairs_to_3d(pred_keypoints.reshape(-1, num_views, num_keypoints, 2), *cameras)
            keypoints_targ_3d = batch_dict["keypoints_3d"]
            assert self.loss_factory is not None
            if "supervised_reprojection_heatmap_mse" in self.loss_factory.loss_instance_dict:
                images = batch_dict["images"]
                keypoints_pred_2d_reprojected = ops.project_points(
                    keypoints_pred_3d, *cameras, mean_over_pairs=True, bbox=batch_dict["bbox"], model_size=images.shape[-2:],
                ).reshape(-1, num_views * num_keypoints, 2)
        return {
            "heatmaps_targ": heatmaps_targ,
            "heatmaps_pred": pred_heatmaps,
            "keypoints_targ": target_keypoints,
            "keypoints_pred": pred_keypoints,
            "confidences": confidence,
            "keypoints_targ_3d": keypoints_targ_3d,  # (batch, num_keypoints, 3)
            "keypoints_pred_3d": keypoints_pred_3d,  # (batch, cam_pairs, num_keypoints, 3)
            "keypoints_pred_2d_reprojected": keypoints_pred_2d_reprojected,  # (batch, num_views * num_keypoints, 2)
        }

    def _keypoint_targets(self, batch_dict: dict) -> GaussianTargets:
        """Targets of a labeled batch that ships ``keypoints`` (B, V * K * 2) model pixels (and ``visibility``
        (B, V * K)) without ``heatmaps``: planes view-major, v * K + k, the order of the reference's ``fusion``
        (``datasets.py:1129-1148``), each (H, W) / 2**downsample_factor.

        The out-of-frame -> NaN rule applies unless the batch carries ``"ignore_nans": True``, a Python bool (a
        tensor would cost a host sync): the reference's dataset skips the rule for calibrated batches
        (``datasets.py:1161-1164``) and recomputes the targets of calibrated training batches after the 3-D
        augmentation with the rule applied (:1094-1101), so pass True for calibrated validation batches only.  As
        there (the rule writes NaN into the example's keypoints), the masked keypoints are also the RMSE targets.
        Building the targets is one kernel launch and no host sync, so a labeled step still captures into a CUDA
        graph."""
        images = batch_dict["images"]
        h_img, w_img = images.shape[-2], images.shape[-1]
        shape_hm = (h_img // 2**self.downsample_factor, w_img // 2**self.downsample_factor)
        return GaussianTargets(batch_dict["keypoints"], h_img, w_img, shape_hm, sigma=1.25, visibility=batch_dict.get("visibility"),
                               ignore_nans=bool(batch_dict.get("ignore_nans", False)))

    def predict_step(self, batch_dict: dict, batch_idx: int, return_heatmaps: bool = False):
        images = batch_dict["images"] if "images" in batch_dict else batch_dict["frames"]
        with torch.no_grad():
            heatmaps = self.forward(images)
            keypoints, confidence = self.head.run_subpixelmaxima(heatmaps)
        keypoints = model_to_frame_batch(batch_dict, keypoints)
        return (keypoints, confidence, heatmaps) if return_heatmaps else (keypoints, confidence)

    def get_parameters(self) -> list[dict]:
        backbone = [p for m in (self.patch_embed, self.encoder) if isinstance(m, nn.Module) for p in m.parameters()]
        return [{"params": backbone, "name": "backbone", "lr": 0.0}, {"params": list(self.head.parameters()) + [self.view_embeddings], "name": "head"}]

    def evaluate_labeled(self, batch_dict: dict, stage=None, anneal_weight=None) -> torch.Tensor:
        data_dict = self.get_loss_inputs_labeled(batch_dict)
        assert self.loss_factory is not None
        loss, self.last_logs = self.loss_factory(stage=stage, anneal_weight=anneal_weight, **data_dict)
        self.last_rmse, _ = self.rmse_loss(stage=stage, **data_dict)
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        """One labeled training step: patch masking (with an enabled ``patch_masker``), forward, the supervised losses (the
        3-D ones on calibrated batches), then ``global_step`` + 1.

        The loss is ``evaluate_labeled``'s total, the sum over the loss factory of weight * loss in its order, computed
        without the host: each weight is made on the device by a fill kernel instead of copied from the host, and the
        RMSE diagnostic (a host-synchronising NaN filter) is left to ``evaluate_labeled``.  So the whole step captures
        into one CUDA graph.  ``last_logs`` holds detached values (what Lightning's ``log`` keeps): a step's autograd
        graph must not outlive it, or the next step's backward would meet the previous step's gradient nodes, whose
        stream may be another than the one being captured (``LossFactory.total_on_device``)."""
        total = self._labeled_step_loss(batch_dict, anneal_weight=None)
        self.global_step.add_(1)
        return {"loss": total}

    def _labeled_step_loss(self, batch_dict: dict, anneal_weight: torch.Tensor | None) -> torch.Tensor:
        """Patch masking of ``batch_dict["images"]`` at ``global_step`` (with an enabled ``patch_masker``), forward and
        the labeled losses summed on the device; ``last_logs`` holds their detached values."""
        masker = self.patch_masker
        if masker is not None and masker.use_patch_masking:  # PatchMasking.on_train_batch_start (callbacks.py:222-263)
            batch_dict["images"], self.current_patch_mask = masker.apply_patch_masking(
                batch_dict["images"], training_step=self.global_step, is_training=True)
        assert self.loss_factory is not None
        total, self.last_logs = self.loss_factory.total_on_device("train", anneal_weight, **self.get_loss_inputs_labeled(batch_dict))
        return total


def view_transforms(transforms: torch.Tensor, num_views: int) -> torch.Tensor | None:
    """The augmentation matrices of a multi-view unlabeled batch as (views, 2, 3), or None for an unaugmented batch
    (a last dimension other than 3, e.g. the (views, 1) sentinel of ``frames_to_unlabeled_batch``).

    Accepts the shapes the reference squeezes (``heatmap_tracker_multiview.py:449-462``): (views, 1, 2, 3) as
    ``frames_to_unlabeled_batch`` returns it, (1, views, 2, 3) and (views, 2, 3).  Any other shape raises (the reference
    logs a warning and undoes the wrong matrices)."""
    if transforms.shape[-1] != 3:
        return None
    if transforms.dim() == 4:
        if transforms.shape[1] == 1:
            transforms = transforms.squeeze(1)
        elif transforms.shape[0] == 1:
            transforms = transforms.squeeze(0)
    if tuple(transforms.shape) != (num_views, 2, 3):
        raise ValueError(f"expected transforms (views, 2, 3) with views = {num_views}, (views, 1, 2, 3) or (1, views, 2, 3); "
                         f"got {tuple(transforms.shape)}")
    return transforms


class SemiSupervisedHeatmapTrackerMultiviewTransformer(HeatmapTrackerMultiviewTransformer):
    """Adds the unlabeled multi-view video branch and its unsupervised loss factory (reference :370-484).

    An unlabeled batch holds frames (T, views, 3, H, W), one sequence per camera, as ``frames_to_unlabeled_batch``
    returns them.  Its heatmaps are folded like the labeled ones, (T, views * K, h, w), so the temporal losses compare
    consecutive frames of each view and ``pca_multiview`` reads the views of a frame side by side.

    ``total_unsupervised_importance`` (the reference's attribute, which its ``AnnealWeight`` callback sets) is a device
    scalar buffer here: a schedule changes it in place, ``model.total_unsupervised_importance.fill_(w)``, and a
    ``training_step`` captured into a CUDA graph then uses the new value on its next replay.  Assigning a new tensor to
    the attribute instead works eagerly but is not seen by a captured graph."""

    def __init__(
        self,
        num_keypoints: int,
        num_views: int,
        patch_embed: nn.Module | Callable,
        encoder: nn.Module | Callable,
        embedding_dim: int,
        loss_factory: LossFactory | None = None,
        loss_factory_unsupervised: LossFactory | None = None,
        backbone_arch: str = "vits_dino",
        downsample_factor: Literal[1, 2, 3] = 2,
        torch_seed: int = 123,
        patch_masker: PatchMasker | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__(
            num_keypoints, num_views, patch_embed, encoder, embedding_dim, loss_factory=loss_factory,
            backbone_arch=backbone_arch, downsample_factor=downsample_factor, torch_seed=torch_seed,
            patch_masker=patch_masker, **kwargs,
        )
        self.loss_factory_unsup = loss_factory_unsupervised
        # not part of the state dict, as the reference's plain attribute is not
        self.register_buffer("total_unsupervised_importance", torch.ones(()), persistent=False)

    def get_loss_inputs_unlabeled(self, batch_dict: dict) -> dict:
        """Frames (T, views, 3, H, W) -> heatmaps (T, views * K, h, w), keypoints and confidences; the per-view affine
        undo and the model -> frame map in one launch (reference :434-484)."""
        frames = batch_dict["frames"]
        if frames.dim() != 5 or frames.shape[1] != self.num_views:
            raise ValueError(f"expected frames (T, {self.num_views}, 3, H, W); got {tuple(frames.shape)}")
        pred_heatmaps, pred_keypoints_augmented, confidence = self.forward_with_keypoints(frames)
        pred_keypoints = ops.remap_keypoints(
            pred_keypoints_augmented, view_transforms(batch_dict["transforms"], self.num_views), batch_dict["bbox"],
            frames.shape[-2], frames.shape[-1], is_multiview=True, num_views=self.num_views,
        )
        return {
            "heatmaps_pred": pred_heatmaps,
            "keypoints_pred": pred_keypoints,
            "keypoints_pred_augmented": pred_keypoints_augmented,
            "confidences": confidence,
        }

    def evaluate_unlabeled(self, batch_dict: dict, stage=None, anneal_weight=1.0) -> torch.Tensor:
        data_dict = self.get_loss_inputs_unlabeled(batch_dict)
        assert self.loss_factory_unsup is not None
        loss, self.last_logs_unsup = self.loss_factory_unsup(stage=stage, anneal_weight=anneal_weight, **data_dict)
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        """One semi-supervised step on ``{"labeled": ..., "unlabeled": ...}`` (the reference's mixin,
        ``models/base.py:660-701``), then ``global_step`` + 1.

        Labeled branch: the parent's ``training_step`` (patch masking of ``labeled["images"]``, the 3-D losses on
        calibrated batches).  The unlabeled frames are not masked; the reference's ``PatchMasking`` callback looks for
        top-level ``images`` / ``frames`` keys only (``callbacks.py:233-243``), so it masks neither branch of a
        semi-supervised batch, while the labeled branch here is masked as a labeled step is.  Both branches' losses are scaled by ``total_unsupervised_importance`` except the
        heatmap losses, which keep weight 1, as the reference's loss factory does.  Both sums run on the device
        (``LossFactory.total_on_device``), so the whole step captures into one CUDA graph; ``last_logs`` and
        ``last_logs_unsup`` hold detached values."""
        anneal = self.total_unsupervised_importance
        loss_super = self._labeled_step_loss(batch_dict["labeled"], anneal_weight=anneal)
        assert self.loss_factory_unsup is not None
        loss_unsuper, self.last_logs_unsup = self.loss_factory_unsup.total_on_device(
            "train", anneal, **self.get_loss_inputs_unlabeled(batch_dict["unlabeled"]))
        self.global_step.add_(1)
        return {"loss": loss_super + loss_unsuper}
