"""Loss classes on H100: drop-in for ``lightning_pose.losses.losses``.

Every class keeps the reference's constructor keywords, attributes (``loss_name``, ``epsilon``,
``log_weight``, ``weight``), staged methods (``remove_nans`` / ``compute_loss`` /
``rectify_epsilon`` / ``reduce_loss`` / ``log_loss``) and - load-bearing for
``lightning_pose/models/factory.py:116-136`` - the ``__call__`` parameter names and defaults.

``__call__`` is where the work happens, and there it differs from the reference: instead of the
staged pipeline (boolean-mask gathers, python loops over frames, a dozen tiny launches) each loss
is one fused CUDA reduction (``csrc/losses.cu``) that produces the same scalar:

* ``HeatmapMSELoss/KLLoss/JSLoss``  -> ``ops.heatmap_loss`` (all-zero target planes dropped on device), or
                                       ``ops.heatmap_loss_from_keypoints`` given ``GaussianTargets``
* ``TemporalLoss`` / ``PCALoss``     -> ``ops.unsup_losses`` (one launch; the factory shares it)
* ``TemporalHeatmapLoss``           -> ``ops.temporal_heatmap_loss``
* ``ReprojectionHeatmapLoss``       -> ``ops.generate_heatmaps`` (differentiable) + ``ops.heatmap_loss``, or
                                       ``ops.heatmap_loss_from_keypoints("mse")`` given ``GaussianTargets``
* ``PairwiseProjectionsLoss``       -> ``ops.pairwise_projections_loss`` (NaN entries dropped on device)
* ``RegressionMSELoss``             -> ``ops.regression_losses`` on CUDA inputs (NaN targets dropped on device, one
                                       launch with the RMSE diagnostic; the regression trackers share it)

The staged methods remain as small tensor utilities for callers/tests that use them directly.
``RegressionRMSELoss``, the always-on diagnostic of the heatmap trackers, keeps the staged tensor code.
"""
from __future__ import annotations

import os
from typing import Any, Literal

import torch
from torch.nn import functional as F

from lightning_pose_b200 import ops
from lightning_pose_b200.data.heatmaps import GaussianTargets
from lightning_pose_b200.utils.pca import KeypointPCA

__all__ = [
    "Loss",
    "HeatmapLoss",
    "HeatmapMSELoss",
    "HeatmapKLLoss",
    "HeatmapJSLoss",
    "PCALoss",
    "TemporalLoss",
    "TemporalHeatmapLoss",
    "RegressionMSELoss",
    "RegressionRMSELoss",
    "PairwiseProjectionsLoss",
    "ReprojectionHeatmapLoss",
]

_DEFAULT_TORCH_DEVICE = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}" if torch.cuda.is_available() else "cpu"

LossOutput = tuple[torch.Tensor, list[dict]]


class Loss:
    """Base class: hyper-parameters + the shared epsilon / reduction / logging helpers."""

    loss_name: str

    def __init__(self, data_module=None, epsilon: float | list[float] = 0.0, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__()
        self.data_module = data_module
        self.epsilon = torch.tensor(epsilon, dtype=torch.float)
        self.log_weight = torch.tensor(log_weight, dtype=torch.float)
        self.reduce_methods_dict = {"mean": torch.mean, "sum": torch.sum}

    @property
    def weight(self) -> torch.Tensor:
        """``1 / (2 exp(log_weight))`` (reference :89-100)."""
        return 1.0 / (2.0 * torch.exp(self.log_weight))

    def device_epsilon(self, device: torch.device) -> torch.Tensor:
        """``epsilon`` on ``device``, copied there once (again only when ``epsilon`` is replaced): the kernels read it
        without a copy from pageable host memory in the step, so the loss launch captures into a CUDA graph."""
        cache = self.__dict__.setdefault("_device_epsilon", {})
        key = (torch.device(device), id(self.epsilon))
        if key not in cache:
            cache.clear()
            cache[key] = self.epsilon.to(device)
        return cache[key]

    def remove_nans(self, **kwargs: Any) -> Any:
        raise NotImplementedError

    def compute_loss(self, **kwargs: Any) -> torch.Tensor:
        raise NotImplementedError

    def rectify_epsilon(self, loss: torch.Tensor) -> torch.Tensor:
        return F.relu(loss - self.epsilon.to(loss.device))

    def reduce_loss(self, loss: torch.Tensor, method: str = "mean") -> torch.Tensor:
        return self.reduce_methods_dict[method](loss)

    def log_loss(self, loss: torch.Tensor, stage: Literal["train", "val", "test"] | None) -> list[dict]:
        return [
            {"name": f"{stage}_{self.loss_name}_loss", "value": loss, "prog_bar": True},
            {"name": f"{self.loss_name}_weight", "value": self.weight},
        ]

    def __call__(self, *args: Any, **kwargs: Any) -> LossOutput:
        raise NotImplementedError


# --------------------------------------------------------------------------------------
# supervised heatmap losses (reference :201-423)
# --------------------------------------------------------------------------------------
class HeatmapLoss(Loss):
    """Parent of the heatmap-shaped losses; subclasses set ``_kind`` and ``compute_loss``."""

    _kind = "mse"

    def __init__(self, data_module=None, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(data_module=data_module, log_weight=log_weight)

    def remove_nans(self, targets: torch.Tensor, predictions: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """Drop planes whose target is all-zero (unlabeled keypoints); staged helper, host-synchronising."""
        keep = ~torch.all(targets.reshape(targets.shape[0], targets.shape[1], -1) == 0.0, dim=-1)
        return targets[keep], predictions[keep]

    def __call__(
        self,
        heatmaps_targ: torch.Tensor,
        heatmaps_pred: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        if isinstance(heatmaps_targ, GaussianTargets):  # targets made on the GPU from (keypoints, visibility), never written
            scalar_loss = ops.heatmap_loss_from_keypoints(self._kind, heatmaps_targ.keypoints, heatmaps_pred, heatmaps_targ.height,
                                                          heatmaps_targ.width, sigma=heatmaps_targ.sigma, visibility=heatmaps_targ.visibility)
            return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)
        scalar_loss = ops.heatmap_loss(heatmaps_targ, heatmaps_pred, self._kind)
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


class HeatmapMSELoss(HeatmapLoss):
    """Pixel MSE scaled by h*w, mean over the pixels of kept planes (reference :293-335)."""

    loss_name = "heatmap_mse"
    _kind = "mse"

    def __init__(self, data_module=None, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(data_module=data_module, log_weight=log_weight)

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        return (targets - predictions) ** 2 * (targets.shape[1] * targets.shape[2])


def _kl_planes(pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    return (torch.xlogy(target, target) - target * torch.log(pred)).reshape(pred.shape[0], -1).sum(-1)


class HeatmapKLLoss(HeatmapLoss):
    """KL(target + 1e-10 || pred + 1e-10) per plane, mean over kept planes (reference :338-378)."""

    loss_name = "heatmap_kl"
    _kind = "kl"

    def __init__(self, data_module=None, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(data_module=data_module, log_weight=log_weight)

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        return _kl_planes(predictions + 1e-10, targets + 1e-10)


class HeatmapJSLoss(HeatmapLoss):
    """Jensen-Shannon divergence per plane, mean over kept planes (reference :382-423)."""

    loss_name = "heatmap_js"
    _kind = "js"

    def __init__(self, data_module=None, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(data_module=data_module, log_weight=log_weight)

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        p, t = predictions + 1e-10, targets + 1e-10
        m = 0.5 * (p + t)
        return 0.5 * _kl_planes(m, t) + 0.5 * _kl_planes(m, p)


# --------------------------------------------------------------------------------------
# unsupervised losses on the keypoint tensor (reference :426-703)
# --------------------------------------------------------------------------------------
_FUSED_KEY = "_lpb_fused_unsup"  # LossFactory passes the shared one-launch result through **kwargs


class PCALoss(Loss):
    """Penalise keypoints outside the PCA subspace: relu(reprojection error - eps), mean."""

    LOSS_NAME_MULTIVIEW = "pca_multiview"
    LOSS_NAME_SINGLEVIEW = "pca_singleview"

    def __init__(
        self,
        loss_name: Literal["pca_singleview", "pca_multiview"],
        components_to_keep: int | float = 0.95,
        empirical_epsilon_percentile: float = 99.0,
        epsilon: float | None = None,
        empirical_epsilon_multiplier: float = 1.0,
        mirrored_column_matches=None,
        columns_for_singleview_pca=None,
        data_module=None,
        log_weight: float = 0.0,
        device: str | torch.device = _DEFAULT_TORCH_DEVICE,
        centering_method: Literal["mean", "median"] | None = None,
        **kwargs: Any,
    ) -> None:
        super().__init__(data_module=data_module, log_weight=log_weight)
        self.device = device
        if loss_name not in (self.LOSS_NAME_MULTIVIEW, self.LOSS_NAME_SINGLEVIEW):
            raise ValueError(f"Invalid loss_name: {loss_name}")
        self.loss_name = loss_name
        if loss_name == "pca_multiview" and mirrored_column_matches is None:
            raise ValueError("must provide mirrored_column_matches in data config")
        assert data_module is not None, "PCALoss requires a data_module to fit PCA"
        self.pca = KeypointPCA(
            loss_type=self.loss_name,
            data_module=data_module,
            components_to_keep=components_to_keep,
            empirical_epsilon_percentile=empirical_epsilon_percentile,
            mirrored_column_matches=mirrored_column_matches,
            columns_for_singleview_pca=columns_for_singleview_pca,
            device=device,
            centering_method=centering_method,
        )
        self.pca()  # one-off host-side fit
        if epsilon is not None:
            self.epsilon = torch.tensor(epsilon, dtype=torch.float, device=self.device)
        else:
            self.epsilon = self.pca.parameters["epsilon"] * empirical_epsilon_multiplier

    def remove_nans(self, **kwargs: Any) -> Any:
        pass

    def compute_loss(self, predictions: torch.Tensor) -> torch.Tensor:
        assert predictions.device == torch.device(self.device), (predictions.device, torch.device(self.device))
        return self.pca.compute_reprojection_error(data_arr=predictions)

    def kernel_params(self, num_keypoints: int) -> ops.PcaParams:
        """Device-side parameter block, built once per keypoint count: no host sync (``float(epsilon)``) and no
        pageable upload in the step, so the unsupervised loss launch is CUDA-graph capturable."""
        cache = self.__dict__.setdefault("_kernel_params", {})
        eps = self.epsilon
        key = (int(num_keypoints), id(eps))
        if key not in cache:
            cache.clear()
            cache[key] = self.pca.kernel_params(num_keypoints, float(eps))
        return cache[key]

    def __call__(
        self, keypoints_pred: torch.Tensor, stage: Literal["train", "val", "test"] | None = None, **kwargs: Any
    ) -> LossOutput:
        assert keypoints_pred.device == torch.device(self.device), (keypoints_pred.device, torch.device(self.device))
        fused = kwargs.get(_FUSED_KEY)
        slot = 1 if self.loss_name == self.LOSS_NAME_SINGLEVIEW else 2
        if fused is None:
            params = self.kernel_params(keypoints_pred.shape[1] // 2)
            fused = ops.unsup_losses(keypoints_pred, **{self.loss_name: params})
        scalar_loss = fused[slot]
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


class TemporalLoss(Loss):
    """relu(||kp[t+1] - kp[t]|| - eps_k), zeroed where either frame is low-confidence, mean."""

    loss_name = "temporal"

    def __init__(
        self,
        data_module=None,
        epsilon: float | list[float] = 0.0,
        prob_threshold: float = 0.0,
        log_weight: float = 0.0,
        **kwargs: Any,
    ) -> None:
        super().__init__(data_module=data_module, epsilon=epsilon, log_weight=log_weight)
        self.prob_threshold = torch.tensor(prob_threshold, dtype=torch.float)

    def rectify_epsilon(self, loss: torch.Tensor) -> torch.Tensor:
        return F.relu(loss - self.epsilon.to(loss.device).reshape(1, -1))

    def remove_nans(self, loss: torch.Tensor, confidences: torch.Tensor) -> torch.Tensor:
        low = confidences < self.prob_threshold.to(confidences.device)
        return loss.masked_fill(low[:-1] | low[1:], 0.0)

    def compute_loss(self, predictions: torch.Tensor) -> torch.Tensor:
        d = torch.diff(predictions, dim=0)
        return torch.linalg.norm(d.reshape(d.shape[0], -1, 2), ord=2, dim=2)

    def __call__(
        self,
        keypoints_pred: torch.Tensor,
        confidences: torch.Tensor | None = None,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        fused = kwargs.get(_FUSED_KEY)
        if fused is None:
            fused = ops.unsup_losses(
                keypoints_pred, confidences, temporal_eps=self.device_epsilon(keypoints_pred.device), prob_threshold=float(self.prob_threshold)
            )
        scalar_loss = fused[0]
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


class TemporalHeatmapLoss(Loss):
    """Frame-to-frame heatmap difference (mean-pixel MSE or KL) with the TemporalLoss masking."""

    LOSS_NAME_MSE = "temporal_heatmap_mse"
    LOSS_NAME_KL = "temporal_heatmap_kl"

    def __init__(
        self,
        loss_name: Literal["temporal_heatmap_mse", "temporal_heatmap_kl"],
        data_module=None,
        epsilon: float | list[float] = 0.0,
        prob_threshold: float = 0.0,
        log_weight: float = 0.0,
        **kwargs: Any,
    ) -> None:
        super().__init__(data_module=data_module, epsilon=epsilon, log_weight=log_weight)
        if loss_name not in (self.LOSS_NAME_MSE, self.LOSS_NAME_KL):
            raise ValueError(f"Invalid loss_name: {loss_name}")
        self.loss_name = loss_name
        self._kind = "mse" if loss_name == self.LOSS_NAME_MSE else "kl"
        self.prob_threshold = torch.tensor(prob_threshold, dtype=torch.float)

    def rectify_epsilon(self, loss: torch.Tensor) -> torch.Tensor:
        return F.relu(loss - self.epsilon.to(loss.device).reshape(1, -1))

    def remove_nans(self, confidences: torch.Tensor, loss: torch.Tensor) -> torch.Tensor:
        low = confidences < self.prob_threshold.to(confidences.device)
        return loss.masked_fill(low[:-1] | low[1:], 0.0)

    def compute_loss(self, predictions: torch.Tensor) -> torch.Tensor:
        a, b = predictions[:-1], predictions[1:]
        if self._kind == "mse":
            return ((a - b) ** 2).reshape(a.shape[0], a.shape[1], -1).mean(-1)
        return _kl_planes((a + 1e-10).flatten(0, 1), (b + 1e-10).flatten(0, 1)).reshape(a.shape[0], a.shape[1])

    def __call__(
        self,
        heatmaps_pred: torch.Tensor,
        confidences: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        scalar_loss = ops.temporal_heatmap_loss(
            heatmaps_pred, confidences, self._kind, self.device_epsilon(heatmaps_pred.device), float(self.prob_threshold)
        )
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


# --------------------------------------------------------------------------------------
# coordinate-regression losses (reference :857-996)
# --------------------------------------------------------------------------------------
FUSED_REGRESSION_KEY = "_lpb_fused_regression"  # a regression tracker passes its one-launch (mse, kept, rmse, pairs)


class RegressionMSELoss(Loss):
    """Mean of (t - p)^2 over the non-NaN target entries.  ``__call__`` on CUDA tensors is one device reduction
    (``ops.regression_losses``: no data-dependent shapes, no host sync, capturable); on CPU tensors it is the staged
    ``remove_nans`` / ``compute_loss`` / ``reduce_loss`` pipeline."""

    loss_name = "regression"

    def __init__(self, data_module=None, epsilon: float = 0.0, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(data_module=data_module, epsilon=epsilon, log_weight=log_weight)

    def remove_nans(self, targets: torch.Tensor, predictions: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        mask = ~torch.isnan(targets)
        return torch.masked_select(targets, mask), torch.masked_select(predictions, mask)

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        return (targets - predictions) ** 2

    def __call__(
        self,
        keypoints_targ: torch.Tensor,
        keypoints_pred: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        fused = kwargs.get(FUSED_REGRESSION_KEY)
        if fused is None and keypoints_pred.is_cuda:
            fused = ops.regression_losses(keypoints_targ, keypoints_pred)
        if fused is not None:
            scalar_loss = fused[0]
            return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)
        return self._staged_call(keypoints_targ, keypoints_pred, stage)

    def _staged_call(self, keypoints_targ: torch.Tensor, keypoints_pred: torch.Tensor, stage) -> LossOutput:
        t, p = self.remove_nans(targets=keypoints_targ, predictions=keypoints_pred)
        scalar_loss = self.reduce_loss(self.compute_loss(targets=t, predictions=p), method="mean")
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


class RegressionRMSELoss(RegressionMSELoss):
    """Per-keypoint Euclidean pixel error; the always-on diagnostic of every tracker.  Staged tensor code on every
    device (a regression tracker reads the same value from its one-launch ``ops.regression_losses`` instead)."""

    loss_name = "rmse"

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        d2 = (targets.reshape(-1, 2) - predictions.reshape(-1, 2)) ** 2
        return torch.sqrt(d2.mean(dim=1))

    def __call__(
        self,
        keypoints_targ: torch.Tensor,
        keypoints_pred: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        return self._staged_call(keypoints_targ, keypoints_pred, stage)


class PairwiseProjectionsLoss(Loss):
    """3D consistency across camera pairs (multiview + calibration only).  ``__call__`` is one CUDA reduction
    (``ops.pairwise_projections_loss``); ``compute_loss`` / ``remove_nans`` stay as the staged tensor helpers."""

    loss_name = "supervised_pairwise_projections"

    def __init__(self, log_weight: float = 0.0, **kwargs: Any) -> None:
        super().__init__(log_weight=log_weight)

    def remove_nans(self, loss: torch.Tensor) -> torch.Tensor:
        mask = ~torch.isnan(loss)
        valid = torch.masked_select(loss, mask)
        if valid.numel() == 0:
            return torch.where(mask, loss, torch.zeros_like(loss)).sum()
        return valid

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        nan_t = torch.isnan(targets).any(dim=-1)
        nan_any = nan_t.unsqueeze(1) | torch.isnan(predictions).any(dim=-1)
        t = torch.where(nan_t.unsqueeze(-1), torch.zeros_like(targets), targets)
        p = torch.where(nan_any.unsqueeze(-1), torch.zeros_like(predictions), predictions)
        d = torch.linalg.norm(t.unsqueeze(1) - p, ord=2, dim=-1)
        return torch.where(nan_any, torch.full_like(d, float("nan")), d)

    def __call__(
        self,
        keypoints_targ_3d: torch.Tensor,
        keypoints_pred_3d: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        if keypoints_targ_3d is None or keypoints_pred_3d is None:
            raise ValueError(
                f"3D keypoints not available for {stage} stage. Camera params file is required but not found;"
                "Turn off supervised_pairwise_projections loss to avoid this error."
            )
        scalar_loss = ops.pairwise_projections_loss(keypoints_targ_3d, keypoints_pred_3d)
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)


class ReprojectionHeatmapLoss(Loss):
    """Heatmaps regenerated from reprojected 2D keypoints vs target heatmaps (differentiable in the
    keypoints).  Also the slot a "unimodal" consistency loss would occupy (SURVEY finding 1)."""

    loss_name = "supervised_reprojection_heatmap_mse"

    def __init__(
        self,
        original_image_height: int,
        original_image_width: int,
        downsampled_image_height: int,
        downsampled_image_width: int,
        log_weight: float = 0.0,
        **kwargs: Any,
    ) -> None:
        super().__init__(log_weight=log_weight)
        self.original_image_height = original_image_height
        self.original_image_width = original_image_width
        self.downsampled_image_height = downsampled_image_height
        self.downsampled_image_width = downsampled_image_width

    def remove_nans(self, loss: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        valid = ~torch.all(targets.reshape(targets.shape[0], targets.shape[1], -1) == 0.0, dim=-1)
        mask = valid[..., None, None].expand_as(loss)
        sel = torch.masked_select(loss, mask)
        if sel.numel() == 0:
            return torch.where(mask, loss, torch.zeros_like(loss)).sum()
        return sel

    def compute_loss(self, targets: torch.Tensor, predictions: torch.Tensor) -> torch.Tensor:
        # reference quirk (:1216-1219): called with 4-D tensors, so the scale is shape[1]*shape[2]
        return (targets - predictions) ** 2 * (targets.shape[1] * targets.shape[2])

    def __call__(
        self,
        heatmaps_targ: torch.Tensor,
        keypoints_pred_2d_reprojected: torch.Tensor,
        stage: Literal["train", "val", "test"] | None = None,
        **kwargs: Any,
    ) -> LossOutput:
        if keypoints_pred_2d_reprojected is None:
            raise ValueError(
                f"Reprojected keypoints not available for {stage} stage. Camera params file is required but not found;"
                "Turn off supervised_reprojection_heatmap loss to avoid this error."
            )
        heatmaps_pred = ops.generate_heatmaps(
            keypoints_pred_2d_reprojected,
            self.original_image_height,
            self.original_image_width,
            (self.downsampled_image_height, self.downsampled_image_width),
            keep_gradients=True,
        )
        if isinstance(heatmaps_targ, GaussianTargets):  # targets evaluated where the predictions are read, never written
            mse, n_kept = ops.heatmap_loss_from_keypoints("mse", heatmaps_targ.keypoints, heatmaps_pred, heatmaps_targ.height, heatmaps_targ.width,
                                                          sigma=heatmaps_targ.sigma, visibility=heatmaps_targ.visibility, return_count=True)
        else:
            mse, n_kept = ops.heatmap_loss(heatmaps_targ, heatmaps_pred, "mse", return_count=True)
        # sum((t-p)^2) / n_kept  ->  mean over kept pixels of (t-p)^2 * (K*h)
        scale = heatmaps_targ.shape[1] / heatmaps_targ.shape[3]
        scalar_loss = torch.where(n_kept > 0, mse * scale, torch.zeros_like(mse))
        return scalar_loss, self.log_loss(loss=scalar_loss, stage=stage)
