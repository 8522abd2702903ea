"""Context (MHCRNN) heatmap trackers: mirror of ``lightning_pose/models/heatmap_tracker_mhcrnn.py`` on the hot path.

``HeatmapTrackerMHCRNN`` (:33-229) / ``SemiSupervisedHeatmapTrackerMHCRNN`` (:232-330) keep the reference's method
surface (``forward`` -> (heatmaps_sf, heatmaps_mf), ``get_loss_inputs_labeled`` with the sf/mf concatenation,
``predict_step`` picking the more confident of the two heads per keypoint, ``get_parameters``) as plain ``nn.Module``s.

H100 specifics: an unlabeled video sequence ``(seq, 3, H, W)`` is pushed through the backbone once and handed to
``HeatmapMHCRNNHead.forward_sequence`` - the (seq, 5, C, h, w) window tensor of
``get_context_from_sequence`` (``models/base.py:159-196, :372-390``) is never built; labeled context batches
``(batch, 5, 3, H, W)`` follow the reference's reshape (their windows do not overlap).
"""
from __future__ import annotations

from typing import Any, Literal

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.data.bboxes import model_to_frame_batch
from lightning_pose_b200.data.heatmaps import GaussianTargets
from lightning_pose_b200.losses.factory import LossFactory
from lightning_pose_b200.losses.losses import RegressionRMSELoss
from lightning_pose_b200.models.backbones import BACKBONE_STRIDES
from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

__all__: list[str] = []


class HeatmapTrackerMHCRNN(nn.Module):
    """Images (with temporal context) -> backbone features -> (single-frame, multi-frame) heatmaps."""

    def __init__(
        self,
        num_keypoints: int,
        num_targets: int | None = None,
        loss_factory: LossFactory | None = None,
        backbone: nn.Module | None = None,
        backbone_arch: str = "resnet50",
        num_fc_input_features: int | None = None,
        downsample_factor: Literal[1, 2, 3] = 2,
        torch_seed: int = 123,
        **kwargs: Any,
    ) -> None:
        super().__init__()
        if downsample_factor != 2:
            raise NotImplementedError("MHCRNN currently only implements downsample_factor=2")
        assert backbone is not None and num_fc_input_features is not None, "pass a backbone module and its feature channels"
        self.torch_seed = torch_seed
        torch.manual_seed(torch_seed)
        self.backbone, self.num_fc_input_features = backbone, num_fc_input_features
        self.do_context = True
        self.num_keypoints = num_keypoints
        self.num_targets = num_keypoints * 2 if num_targets is None else num_targets
        self.downsample_factor = downsample_factor
        self.head = HeatmapMHCRNNHead(
            backbone_arch=backbone_arch, in_channels=num_fc_input_features, out_channels=num_keypoints,
            downsample_factor=downsample_factor, upsampling_factor=1 if BACKBONE_STRIDES.get(backbone_arch, 32) == 16 else 2,
        )
        self.loss_factory = loss_factory
        self.rmse_loss = RegressionRMSELoss()

    def forward(self, images: torch.Tensor, is_multiview: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
        shape = images.shape
        if len(shape) == 4:  # one video sequence (seq, 3, H, W): features once per frame, windows by index
            return self.head.forward_sequence(self.backbone(images))
        if len(shape) == 5 and is_multiview:  # (seq, views, 3, H, W): views stacked along the feature dimension (base.py:342-370)
            seq, views = shape[:2]
            feats = self.backbone(images.reshape(seq * views, *shape[2:]))
            feats = feats.reshape(seq, -1, feats.shape[-2], feats.shape[-1])
            windows = ops.context_gather(feats.contiguous(), 5)[2:-2]
            reps = torch.permute(windows, (0, 2, 3, 4, 1))
            return self.head(reps, shape, True)
        if len(shape) == 6:  # (batch, views, frames, 3, H, W) -> views into the batch
            images = images.reshape(-1, *shape[-4:])
        batch, frames = images.shape[:2]
        feats = self.backbone(images.reshape(batch * frames, *images.shape[2:]))
        reps = torch.permute(feats.reshape(batch, frames, *feats.shape[1:]), (0, 2, 3, 4, 1))
        return self.head(reps, shape, is_multiview)

    def get_loss_inputs_labeled(self, batch_dict: dict) -> dict:
        sf, mf = self.forward(batch_dict["images"])
        kp_sf, cf_sf = self.head.run_subpixelmaxima(sf)
        kp_mf, cf_mf = self.head.run_subpixelmaxima(mf)
        if "heatmaps" in batch_dict:  # reference flow: DataLoader workers rendered the centre frame's targets
            heatmaps_targ = torch.cat([batch_dict["heatmaps"], batch_dict["heatmaps"]], dim=0)
            target = model_to_frame_batch(batch_dict, batch_dict["keypoints"])
        else:
            heatmaps_targ, keypoints = self._keypoint_targets(batch_dict)
            target = model_to_frame_batch(batch_dict, keypoints, in_place=False)
        kp_sf = model_to_frame_batch(batch_dict, kp_sf)
        kp_mf = model_to_frame_batch(batch_dict, kp_mf)
        return {
            "heatmaps_targ": heatmaps_targ,
            "heatmaps_pred": torch.cat([sf, mf], dim=0),
            "keypoints_targ": torch.cat([target, target], dim=0),
            "keypoints_pred": torch.cat([kp_sf, kp_mf], dim=0),
            "confidences": torch.cat([cf_sf, cf_mf], dim=0),
        }

    def _keypoint_targets(self, batch_dict: dict) -> tuple[GaussianTargets, torch.Tensor]:
        """Targets of a labeled batch that ships the centre frame's ``keypoints`` (and ``visibility``) without
        ``heatmaps``: ``GaussianTargets`` standing for ``torch.cat([heatmaps, heatmaps])``, one copy per head (reference
        :158-173), and the keypoints after the out-of-frame -> NaN rule, which the reference's ``compute_heatmap``
        applies in place on the example's keypoints (``datasets.py:486-508``), so it reaches the RMSE targets too.
        ``images`` is (B, 5, 3, H, W) or (B, V, 5, 3, H, W); the heatmaps are (H, W) / 2**downsample_factor."""
        images, keypoints = batch_dict["images"], batch_dict["keypoints"]
        h_img, w_img = images.shape[-2], images.shape[-1]
        shape_hm = (h_img // 2**self.downsample_factor, w_img // 2**self.downsample_factor)
        centre = GaussianTargets(keypoints, h_img, w_img, shape_hm, sigma=1.25, visibility=batch_dict.get("visibility"))
        kp, vis = centre.keypoints, centre.visibility
        both = GaussianTargets(torch.cat([kp, kp], dim=0), h_img, w_img, shape_hm, sigma=1.25,
                               visibility=None if vis is None else torch.cat([vis, vis], dim=0), ignore_nans=True)
        return both, kp.reshape(keypoints.shape)

    def predict_step(self, batch_dict: dict, batch_idx: int, return_heatmaps: bool | None = False):
        images = batch_dict["images"] if "images" in batch_dict else batch_dict["frames"]
        with torch.no_grad():
            sf, mf = self.forward(images)
            kp_sf, cf_sf = self.head.run_subpixelmaxima(sf)
            kp_mf, cf_mf = self.head.run_subpixelmaxima(mf)
        k = cf_sf.shape[1]
        pick = torch.gt(cf_mf, cf_sf)  # the more confident head wins, per keypoint (reference :196-205)
        kp = torch.where(pick[..., None], kp_mf.reshape(-1, k, 2), kp_sf.reshape(-1, k, 2)).reshape(-1, 2 * k)
        cf = torch.where(pick, cf_mf, cf_sf)
        if kp.shape[0] == batch_dict["bbox"].shape[0] or kp.shape[0] + 4 == batch_dict["bbox"].shape[0]:
            kp = model_to_frame_batch(batch_dict, kp.contiguous())
        if return_heatmaps:
            return kp, cf, torch.where(pick[..., None, None], mf, sf)
        return kp, cf

    def get_parameters(self) -> list[dict]:
        return [{"params": self.backbone.parameters(), "name": "backbone", "lr": 0.0}, {"params": self.head.parameters(), "name": "head"}]

    def evaluate_labeled(self, batch_dict: dict, stage=None, anneal_weight=None) -> torch.Tensor:
        data_dict = self.get_loss_inputs_labeled(batch_dict)
        assert self.loss_factory is not None
        loss, self.last_logs = self.loss_factory(stage=stage, anneal_weight=anneal_weight, **data_dict)
        self.last_rmse, _ = self.rmse_loss(stage=stage, **data_dict)
        return loss


class SemiSupervisedHeatmapTrackerMHCRNN(HeatmapTrackerMHCRNN):
    """Adds the unlabeled-video branch (reference :232-330, :264-... of the mixin: both heads' predictions are stacked)."""

    def __init__(self, num_keypoints: int, loss_factory: LossFactory | None = None, loss_factory_unsupervised: LossFactory | None = None, **kwargs: Any) -> None:
        super().__init__(num_keypoints=num_keypoints, loss_factory=loss_factory, **kwargs)
        self.loss_factory_unsup = loss_factory_unsupervised
        self.total_unsupervised_importance = torch.tensor(1.0)

    def get_loss_inputs_unlabeled(self, batch_dict: dict) -> dict:
        frames = batch_dict["frames"]
        is_multiview = bool(batch_dict.get("is_multiview", False))
        sf, mf = self.forward(frames, is_multiview=is_multiview)
        kp_sf_aug, cf_sf = self.head.run_subpixelmaxima(sf)
        kp_mf_aug, cf_mf = self.head.run_subpixelmaxima(mf)
        transforms = batch_dict["transforms"]
        num_views = batch_dict["bbox"].shape[1] // 4 if is_multiview else 1
        tf = transforms if transforms.shape[-1] == 3 else None
        remap = lambda kp: ops.remap_keypoints(kp, tf, batch_dict["bbox"], frames.shape[-2], frames.shape[-1], is_multiview=is_multiview, num_views=num_views)
        return {
            "heatmaps_pred": torch.cat([sf, mf], dim=0),
            "keypoints_pred": torch.cat([remap(kp_sf_aug), remap(kp_mf_aug)], dim=0),
            "confidences": torch.cat([cf_sf, cf_mf], dim=0),
        }

    def evaluate_unlabeled(self, batch_dict: dict, stage=None, anneal_weight=1.0) -> torch.Tensor:
        data_dict = self.get_loss_inputs_unlabeled(batch_dict)
        assert self.loss_factory_unsup is not None
        loss, self.last_logs_unsup = self.loss_factory_unsup(stage=stage, anneal_weight=anneal_weight, **data_dict)
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        w = self.total_unsupervised_importance
        return {"loss": self.evaluate_labeled(batch_dict["labeled"], "train", anneal_weight=w) + self.evaluate_unlabeled(batch_dict["unlabeled"], "train", anneal_weight=w)}
