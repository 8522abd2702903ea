"""Regression trackers (mirror of ``lightning_pose/models/regression_tracker.py``): images -> backbone -> pooled linear
head -> (x, y) of every keypoint, in model pixels.

``RegressionTracker`` / ``SemiSupervisedRegressionTracker`` keep the reference's constructor keywords and method surface
(``forward`` :91-102, ``get_loss_inputs_labeled`` :104-114, ``predict_step`` :116-138, ``get_parameters`` :140-153,
``get_loss_inputs_unlabeled`` :206-221, plus ``evaluate_labeled/unlabeled`` and ``training_step`` of
``lightning_pose/models/base.py``) but are plain ``nn.Module``s, like the heatmap trackers here.

H100 specifics: the reference's backbone keeps torchvision's ``avgpool`` (``backbones/factory.py:324``); here the
backbone stops before it and ``LinearRegressionHead`` averages the feature map itself, in the same launch that reads it
(``avgpool`` has no parameters, so the state-dict keys are the reference's).  The supervised loss and the RMSE
diagnostic are one launch (``ops.regression_losses``), the affine undo of the unlabeled branch is one launch, and the
temporal / PCA losses share the existing ``ops.unsup_losses`` launch.  ``training_step`` sums the losses on the device
(``LossFactory.total_on_device``), so a step captures into one CUDA graph.
"""
from __future__ import annotations

from typing import Any

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.losses.factory import LossFactory
from lightning_pose_b200.losses.losses import FUSED_REGRESSION_KEY, RegressionRMSELoss
from lightning_pose_b200.models.datatypes import RegressionTrackerLabeledOutputsDict, RegressionTrackerUnlabeledOutputsDict
from lightning_pose_b200.models.heads.regression import LinearRegressionHead
from lightning_pose_b200.models.heatmap_tracker import build_backbone

__all__: list[str] = []


def _unit_boxes(n: int, device) -> torch.Tensor:
    """(n, 4) boxes [0, 0, 1, 1]: with a 1 x 1 model size, ``ops.remap_keypoints`` then undoes the affine only (the
    reference's regression branch has no bbox remap), exactly: x * 1 * 1 + 0.  Made by fill kernels, so capturable."""
    boxes = torch.zeros((n, 4), device=device, dtype=torch.float32)
    boxes[:, 2:] = 1.0
    return boxes


class RegressionTracker(nn.Module):
    """Images -> backbone features -> pooled linear head -> keypoints (+ supervised losses)."""

    def __init__(
        self,
        num_keypoints: int,
        loss_factory: LossFactory | None = None,
        backbone: str | nn.Module = "resnet50",
        pretrained: bool = True,
        torch_seed: int = 123,
        optimizer: str = "Adam",
        optimizer_params: dict | None = None,
        lr_scheduler: str = "multisteplr",
        lr_scheduler_params: dict | None = None,
        num_fc_input_features: int | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__()
        self.torch_seed = torch_seed
        torch.manual_seed(torch_seed)
        if isinstance(backbone, nn.Module):
            assert num_fc_input_features is not None, "give num_fc_input_features with a custom backbone"
            self.backbone, self.num_fc_input_features = backbone, num_fc_input_features
        else:
            if "vit" in backbone:
                raise ValueError("Regression trackers are not compatible with ViT backbones")
            # stops before avgpool: the head pools (module docstring)
            self.backbone, self.num_fc_input_features = build_backbone(backbone, pretrained)
        kwargs.pop("do_context", None)  # backwards compatibility, as the reference
        self.optimizer, self.optimizer_params = optimizer, optimizer_params
        self.lr_scheduler, self.lr_scheduler_params = lr_scheduler, lr_scheduler_params
        self.num_keypoints = num_keypoints
        self.num_targets = self.num_keypoints * 2
        self.loss_factory = loss_factory
        self.head = LinearRegressionHead(self.num_fc_input_features, self.num_targets)
        self.rmse_loss = RegressionRMSELoss()

    def get_representations(self, images: torch.Tensor) -> torch.Tensor:
        return self.backbone(images)

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        """(B, 3, H, W) images -> (B, 2K) keypoints in model pixels."""
        return self.head(self.get_representations(images))

    def get_loss_inputs_labeled(self, batch_dict: dict) -> RegressionTrackerLabeledOutputsDict:
        predicted_keypoints = self.forward(batch_dict["images"])
        return {"keypoints_targ": batch_dict["keypoints"], "keypoints_pred": predicted_keypoints}

    def predict_step(self, batch_dict: dict, batch_idx: int, **kwargs: Any) -> tuple[torch.Tensor, torch.Tensor]:
        """(keypoints (B, 2K) in model pixels, confidence (B, K) of zeros).  The reference makes its zeros on the host
        (``regression_tracker.py:136-138``); these are on the keypoints' device."""
        images = batch_dict["images"] if "images" in batch_dict else batch_dict["frames"]
        predicted_keypoints = self.forward(images)
        confidence = torch.zeros((predicted_keypoints.shape[0], predicted_keypoints.shape[1] // 2), device=predicted_keypoints.device)
        return predicted_keypoints, confidence

    def get_parameters(self) -> list[dict]:
        """Order matters: group 0 = backbone (lr 0 until unfrozen), group 1 = head (``callbacks.py:142-146``)."""
        return [
            {"params": self.backbone.parameters(), "lr": 0, "name": "backbone"},
            {"params": self.head.parameters(), "name": "head"},
        ]

    def _labeled(self, batch_dict: dict) -> dict:
        """``get_loss_inputs_labeled`` plus the one-launch MSE / RMSE result, which the loss factory's ``regression``
        loss reads instead of launching again; sets ``last_rmse`` (a device scalar)."""
        data_dict = dict(self.get_loss_inputs_labeled(batch_dict))
        fused = ops.regression_losses(data_dict["keypoints_targ"], data_dict["keypoints_pred"])
        self.last_rmse = fused[2]
        return {**data_dict, FUSED_REGRESSION_KEY: fused}

    def evaluate_labeled(self, batch_dict: dict, stage=None, anneal_weight=None) -> torch.Tensor:
        assert self.loss_factory is not None
        loss, self.last_logs = self.loss_factory(stage=stage, anneal_weight=anneal_weight, **self._labeled(batch_dict))
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        """The labeled losses summed on the device (``LossFactory.total_on_device``): no host sync, so the step (with a
        device-side ingest in front of it) captures into one CUDA graph.  ``last_logs`` holds detached values."""
        assert self.loss_factory is not None
        total, self.last_logs = self.loss_factory.total_on_device("train", None, **self._labeled(batch_dict))
        return {"loss": total}


class SemiSupervisedRegressionTracker(RegressionTracker):
    """Adds the unlabeled-video branch and its unsupervised loss factory (temporal, PCA)."""

    def __init__(
        self,
        num_keypoints: int,
        loss_factory: LossFactory | None = None,
        loss_factory_unsupervised: LossFactory | None = None,
        backbone: str | nn.Module = "resnet50",
        pretrained: bool = True,
        torch_seed: int = 123,
        optimizer: str = "Adam",
        optimizer_params: dict | None = None,
        lr_scheduler: str = "multisteplr",
        lr_scheduler_params: dict | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__(
            num_keypoints=num_keypoints, loss_factory=loss_factory, backbone=backbone, pretrained=pretrained,
            torch_seed=torch_seed, optimizer=optimizer, optimizer_params=optimizer_params, lr_scheduler=lr_scheduler,
            lr_scheduler_params=lr_scheduler_params, **kwargs,
        )
        self.loss_factory_unsup = loss_factory_unsupervised
        # a device scalar that a schedule changes in place (fill_), so that a captured step sees the new value on replay;
        # not part of the state dict, as the reference's plain attribute is not
        self.register_buffer("total_unsupervised_importance", torch.ones(()), persistent=False)

    def get_loss_inputs_unlabeled(self, batch_dict: dict) -> RegressionTrackerUnlabeledOutputsDict:
        """Frames (T, 3, H, W) -> keypoints (T, 2K) with the augmentation's affine undone (reference :206-221): one
        launch, no bbox remap and no confidences, as there."""
        frames = batch_dict["frames"]
        predicted_keypoints = self.forward(frames)
        transforms = batch_dict["transforms"]
        if transforms.shape[-1] == 3:
            predicted_keypoints = ops.remap_keypoints(predicted_keypoints, transforms,
                                                      _unit_boxes(predicted_keypoints.shape[0], frames.device), 1.0, 1.0)
        return {"keypoints_pred": predicted_keypoints}

    def evaluate_unlabeled(self, batch_dict: dict, stage=None, anneal_weight=1.0) -> torch.Tensor:
        assert self.loss_factory_unsup is not None
        loss, self.last_logs_unsup = self.loss_factory_unsup(stage=stage, anneal_weight=anneal_weight,
                                                             **self.get_loss_inputs_unlabeled(batch_dict))
        return loss

    def training_step(self, batch_dict: dict, batch_idx: int) -> dict[str, torch.Tensor]:
        """Both branches summed on the device, every loss scaled by ``total_unsupervised_importance`` (the regression
        loss is not exempt from annealing in the reference's factory either)."""
        anneal = self.total_unsupervised_importance
        assert self.loss_factory is not None and self.loss_factory_unsup is not None
        loss_super, self.last_logs = self.loss_factory.total_on_device("train", anneal, **self._labeled(batch_dict["labeled"]))
        loss_unsuper, self.last_logs_unsup = self.loss_factory_unsup.total_on_device(
            "train", anneal, **self.get_loss_inputs_unlabeled(batch_dict["unlabeled"]))
        return {"loss": loss_super + loss_unsuper}
