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
"""
from __future__ import annotations

import math
from typing import Any, Callable, Literal

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.data.bboxes import model_to_frame_batch
from lightning_pose_b200.data.cameras import project_camera_pairs_to_3d
from lightning_pose_b200.losses.factory import LossFactory
from lightning_pose_b200.losses.losses import RegressionRMSELoss
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
        **kwargs: Any,
    ) -> None:
        super().__init__()
        torch.manual_seed(torch_seed)
        self.num_keypoints, self.num_views, self.downsample_factor = num_keypoints, num_views, downsample_factor
        self.num_fc_input_features = embedding_dim
        self.patch_embed, self.encoder = patch_embed, encoder
        generator = torch.Generator().manual_seed(torch_seed)
        self.view_embeddings = nn.Parameter(torch.randn(num_views, embedding_dim, generator=generator) * 0.02)
        self.head = HeatmapHead(backbone_arch=backbone_arch, in_channels=embedding_dim, out_channels=num_keypoints, downsample_factor=downsample_factor)
        self.loss_factory = loss_factory
        self.rmse_loss = RegressionRMSELoss()

    def forward_vit(self, images: torch.Tensor) -> torch.Tensor:
        """(view * batch, 3, H, W) -> (view * batch, D, h, w), views attending to each other (reference :143-232)."""
        tokens = self.patch_embed(images)  # (view * batch, N, D)
        vb, n, d = tokens.shape
        batch = vb // self.num_views
        view_idx = torch.arange(self.num_views, device=tokens.device).repeat(batch)  # [0..V-1, 0..V-1, ...]
        tokens = tokens + self.view_embeddings[view_idx].to(tokens.dtype).unsqueeze(1)
        seq = self.encoder(tokens.reshape(batch, self.num_views * n, d))  # all views of an example in one sequence
        side = math.isqrt(n)
        out = seq.reshape(batch, self.num_views, side, side, d).permute(0, 1, 4, 2, 3)
        return out.reshape(vb, d, side, side).contiguous()

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        batch, views, c, h, w = images.shape
        heatmaps = self.head(self.forward_vit(images.reshape(-1, c, h, w)))
        return heatmaps.reshape(batch, -1, heatmaps.shape[-2], heatmaps.shape[-1])

    def forward_with_keypoints(self, images: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        batch, views, c, h, w = images.shape
        hm, kp, cf = self.head.forward_with_keypoints(self.forward_vit(images.reshape(-1, c, h, w)))
        return hm.reshape(batch, -1, hm.shape[-2], hm.shape[-1]), kp.reshape(batch, -1), cf.reshape(batch, -1)

    def get_loss_inputs_labeled(self, batch_dict: dict) -> dict:
        pred_heatmaps, pred_keypoints, confidence = self.forward_with_keypoints(batch_dict["images"])
        target_keypoints = model_to_frame_batch(batch_dict, batch_dict["keypoints"])
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
            "heatmaps_targ": batch_dict["heatmaps"],
            "heatmaps_pred": pred_heatmaps,
            "keypoints_targ": target_keypoints,
            "keypoints_pred": pred_keypoints,
            "confidences": confidence,
            "keypoints_targ_3d": keypoints_targ_3d,  # (batch, num_keypoints, 3)
            "keypoints_pred_3d": keypoints_pred_3d,  # (batch, cam_pairs, num_keypoints, 3)
            "keypoints_pred_2d_reprojected": keypoints_pred_2d_reprojected,  # (batch, num_views * num_keypoints, 2)
        }

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
