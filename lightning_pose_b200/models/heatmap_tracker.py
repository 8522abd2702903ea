"""Heatmap trackers: the caller of the hot path (mirror of ``lightning_pose/models/heatmap_tracker.py``).

``HeatmapTracker`` / ``SemiSupervisedHeatmapTracker`` keep the reference's method surface on the path
(``forward`` :107-133, ``get_loss_inputs_labeled`` :135-153, ``predict_step`` :155-191, ``get_parameters``
:193-208, ``get_loss_inputs_unlabeled`` :264-286, plus ``evaluate_labeled/unlabeled`` and ``training_step`` of
``lightning_pose/models/base.py:504-573,627-701``) but are plain ``nn.Module``s: Lightning orchestration
(optimisers, logging, checkpointing) is out of scope.  The backbone is any module mapping images to
``(B, C, H/stride, W/stride)`` features - a dense-contraction provider outside this repository's kernels.

H100 specifics: the head, decode, coordinate remap and losses all run in ``liblpb200.so``; the affine undo
and the model->frame map of the unlabeled branch are one launch; the keypoint tensor handed to the losses
is a fresh tensor (the reference aliases ``keypoints_pred_augmented`` through an in-place view when there
is no augmentation, ``heatmap_tracker.py:272-285`` - harmless there because no loss reads it).
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
from lightning_pose_b200.models.datatypes import HeatmapTrackerLabeledOutputsDict, HeatmapTrackerUnlabeledOutputsDict
from lightning_pose_b200.models.heads.heatmap import HeatmapHead

__all__: list[str] = []


def build_backbone(backbone_arch: str, pretrained: bool = False) -> tuple[nn.Module, int]:
    """torchvision ResNet truncated after ``layer4`` (reference ``backbones/factory.py:238-330``); returns
    (module, feature channels).  Only the ResNet family is wired here; pass your own module otherwise."""
    import torchvision.models as tvm

    if not backbone_arch.startswith("resnet"):
        raise NotImplementedError(f"pass a backbone module for {backbone_arch!r}")
    net = getattr(tvm, backbone_arch)(weights="DEFAULT" if pretrained else None)
    feats = nn.Sequential(*list(net.children())[:-2])
    return feats, net.fc.in_features


class HeatmapTracker(nn.Module):
    """Images -> backbone features -> heatmaps -> soft-argmax keypoints (+ supervised losses)."""

    def __init__(
        self,
        num_keypoints: int,
        num_targets: int | None = None,
        loss_factory: LossFactory | None = None,
        backbone: str | nn.Module = "resnet50",
        downsample_factor: Literal[1, 2, 3] = 2,
        pretrained: bool = False,
        torch_seed: int = 123,
        num_fc_input_features: int | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__()
        self.torch_seed = torch_seed
        torch.manual_seed(torch_seed)
        if isinstance(backbone, nn.Module):
            assert num_fc_input_features is not None, "give num_fc_input_features with a custom backbone"
            self.backbone, self.num_fc_input_features, arch = backbone, num_fc_input_features, kwargs.get("backbone_arch", "resnet50")
        else:
            self.backbone, self.num_fc_input_features = build_backbone(backbone, pretrained)
            arch = backbone
        self.num_keypoints = num_keypoints
        self.num_targets = num_keypoints * 2 if num_targets is None else num_targets
        self.downsample_factor = downsample_factor
        self.head = HeatmapHead(
            backbone_arch=arch,
            in_channels=self.num_fc_input_features,
            out_channels=self.num_keypoints,
            downsample_factor=self.downsample_factor,
        )
        self.loss_factory = loss_factory
        self.rmse_loss = RegressionRMSELoss()

    def get_representations(self, images: torch.Tensor) -> torch.Tensor:
        return self.backbone(images)

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        shape = images.shape
        if len(shape) > 4:  # (batch, views, C, H, W): fold views into the batch and back (reference :120-128)
            heatmaps = self.head(self.get_representations(images.reshape(-1, *shape[-3:])))
            return heatmaps.reshape(shape[0], -1, heatmaps.shape[-2], heatmaps.shape[-1])
        return self.head(self.get_representations(images))

    def forward_with_keypoints(self, images: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``forward`` followed by ``head.run_subpixelmaxima`` as one fused autograd node (training paths)."""
        shape = images.shape
        if len(shape) > 4:
            images = images.reshape(-1, *shape[-3:])
        heatmaps, keypoints, confidence = self.head.forward_with_keypoints(self.get_representations(images))
        if len(shape) > 4:  # fold the views back (reference :120-128); decode is per plane, so it commutes
            heatmaps = heatmaps.reshape(shape[0], -1, heatmaps.shape[-2], heatmaps.shape[-1])
            keypoints = keypoints.reshape(shape[0], -1)
            confidence = confidence.reshape(shape[0], -1)
        return heatmaps, keypoints, confidence

    def get_loss_inputs_labeled(self, batch_dict: dict) -> HeatmapTrackerLabeledOutputsDict:
        predicted_heatmaps, predicted_keypoints, confidence = self.forward_with_keypoints(batch_dict["images"])
        predicted_keypoints = model_to_frame_batch(batch_dict, predicted_keypoints)
        keypoints = batch_dict["keypoints"]
        if "heatmaps" in batch_dict:  # reference flow: DataLoader workers rendered the targets (data/datasets.py:516)
            heatmaps_targ = batch_dict["heatmaps"]
        else:
            # on-GPU target pipeline (SURVEY 8f-2): the batch ships (keypoints, visibility) only; the supervised loss
            # renders the Gaussians itself (HeatmapMSELoss: fused with the loss, planes never written).  The
            # out-of-frame -> NaN rule of HeatmapDataset.compute_heatmap is applied on the device and, as there
            # (in-place on the example's keypoints), also reaches the RMSE targets.
            images = batch_dict["images"]
            h_img, w_img = images.shape[-2], images.shape[-1]
            shape_hm = (h_img // 2**self.downsample_factor, w_img // 2**self.downsample_factor)
            heatmaps_targ = GaussianTargets(keypoints, h_img, w_img, shape_hm, sigma=1.25, visibility=batch_dict.get("visibility"))
            keypoints = heatmaps_targ.keypoints.reshape(keypoints.shape)
        target_keypoints = model_to_frame_batch(batch_dict, keypoints, in_place="heatmaps" in batch_dict)
        return {
            "heatmaps_targ": heatmaps_targ,
            "heatmaps_pred": predicted_heatmaps,
            "keypoints_targ": target_keypoints,
            "keypoints_pred": predicted_keypoints,
            "confidences": confidence,
        }

    def predict_step(self, batch_dict: dict, batch_idx: int, return_heatmaps: bool | None = False):
        images = batch_dict["images"] if "images" in batch_dict else batch_dict["frames"]
        predicted_heatmaps = self.forward(images)
        predicted_keypoints, confidence = self.head.run_subpixelmaxima(predicted_heatmaps)
        predicted_keypoints = model_to_frame_batch(batch_dict, predicted_keypoints)
        if return_heatmaps:
            return predicted_keypoints, confidence, predicted_heatmaps
        return predicted_keypoints, confidence

    def get_parameters(self) -> list[dict]:
        """Order matters: group 0 = backbone (lr 0 until unfrozen), group 1 = head (``callbacks.py:142-146``)."""
        return [
            {"params": self.backbone.parameters(), "lr": 0, "name": "backbone"},
            {"params": self.head.parameters(), "name": "head"},
        ]

    def evaluate_labeled(self, batch_dict: dict, stage=None, anneal_weight=None) -> torch.Tensor:
        data_dict = self.get_loss_inputs_labeled(batch_dict=batch_dict)
        assert self.loss_factory is not None
        loss, self.last_logs = self.loss_factory(stage=stage, anneal_weight=anneal_weight, **data_dict)
        self.last_rmse, _ = self.rmse_loss(stage=stage, **data_dict)
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        anneal = getattr(self, "total_unsupervised_importance", None)
        return {"loss": self.evaluate_labeled(batch_dict, "train", anneal_weight=anneal)}


class SemiSupervisedHeatmapTracker(HeatmapTracker):
    """Adds the unlabeled-video branch and its unsupervised loss factory."""

    def __init__(
        self,
        num_keypoints: int,
        loss_factory: LossFactory | None = None,
        loss_factory_unsupervised: LossFactory | None = None,
        backbone: str | nn.Module = "resnet50",
        downsample_factor: Literal[1, 2, 3] = 2,
        pretrained: bool = False,
        torch_seed: int = 123,
        **kwargs: Any,
    ) -> None:
        super().__init__(
            num_keypoints=num_keypoints, loss_factory=loss_factory, backbone=backbone,
            downsample_factor=downsample_factor, pretrained=pretrained, torch_seed=torch_seed, **kwargs,
        )
        self.loss_factory_unsup = loss_factory_unsupervised
        self.total_unsupervised_importance = torch.tensor(1.0)  # modified by an AnnealWeight-style schedule

    def get_loss_inputs_unlabeled(self, batch_dict: dict) -> HeatmapTrackerUnlabeledOutputsDict:
        frames = batch_dict["frames"]
        pred_heatmaps, pred_keypoints_augmented, confidence = self.forward_with_keypoints(frames)
        is_multiview = bool(batch_dict.get("is_multiview", False))
        transforms = batch_dict["transforms"]
        num_views = batch_dict["bbox"].shape[1] // 4 if is_multiview else 1
        pred_keypoints = ops.remap_keypoints(  # affine undo + model->frame in one launch
            pred_keypoints_augmented, transforms if transforms.shape[-1] == 3 else None, batch_dict["bbox"],
            frames.shape[-2], frames.shape[-1], is_multiview=is_multiview, num_views=num_views,
        )
        return {
            "heatmaps_pred": pred_heatmaps,
            "keypoints_pred": pred_keypoints,
            "keypoints_pred_augmented": pred_keypoints_augmented,
            "confidences": confidence,
        }

    def evaluate_unlabeled(self, batch_dict: dict, stage=None, anneal_weight=1.0) -> torch.Tensor:
        data_dict = self.get_loss_inputs_unlabeled(batch_dict=batch_dict)
        assert self.loss_factory_unsup is not None
        loss, self.last_logs_unsup = self.loss_factory_unsup(stage=stage, anneal_weight=anneal_weight, **data_dict)
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        w = self.total_unsupervised_importance
        loss_super = self.evaluate_labeled(batch_dict["labeled"], "train", anneal_weight=w)
        loss_unsuper = self.evaluate_unlabeled(batch_dict["unlabeled"], "train", anneal_weight=w)
        return {"loss": loss_super + loss_unsuper}
