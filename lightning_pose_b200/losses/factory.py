"""Loss registry and weighted combination: drop-in for ``lightning_pose.losses.factory``.

* ``get_loss_classes``   name -> class, the reference's 11 registry names (``losses/factory.py:73-91``)
* ``get_loss_factories`` cfg -> {'supervised': LossFactory, 'unsupervised': LossFactory} (:94-194)
* ``LossFactory``        holds the instantiated losses, returns ``sum_l anneal_l * weight_l * loss_l``
  plus the logging dicts (:197-285); heatmap_{mse,kl,js} are exempt from annealing (:267).

H100 specifics: the running total never touches the host (the reference starts it as a CPU
tensor and ``.to(device)``s it every iteration, :250,273), and when a factory holds more than one
of {temporal, pca_singleview, pca_multiview} they are evaluated by ONE kernel launch whose result
is handed to each loss object.  ``LossFactory.total_on_device`` is the same sum with device-made
weights and a device-held anneal weight, for training steps captured into a CUDA graph.
"""
from __future__ import annotations

from typing import Any, Literal

import numpy as np
import torch

from lightning_pose_b200 import ops
from lightning_pose_b200.losses import losses as L

try:  # the reference derives LossFactory from LightningModule; fall back to nn.Module without lightning
    import lightning.pytorch as pl

    _FactoryBase = pl.LightningModule
except Exception:  # pragma: no cover - lightning is not installed in this image
    _FactoryBase = torch.nn.Module

__all__: list[str] = []

_ANNEAL_EXEMPT = ("heatmap_mse", "heatmap_kl", "heatmap_js")


def get_loss_classes() -> dict[str, type[L.Loss]]:
    registry: dict[str, type[L.Loss]] = {}
    for cls in (L.RegressionMSELoss, L.HeatmapMSELoss, L.HeatmapKLLoss, L.HeatmapJSLoss, L.TemporalLoss,
                L.PairwiseProjectionsLoss, L.ReprojectionHeatmapLoss):
        registry[cls.loss_name] = cls
    for cls in (L.PCALoss, L.TemporalHeatmapLoss):
        for attr in vars(cls):
            if attr.startswith("LOSS_NAME_"):
                registry[getattr(cls, attr)] = cls
    return registry


def _cfg_get(node: Any, key: str, default: Any = None) -> Any:
    if node is None:
        return default
    if hasattr(node, "get"):
        return node.get(key, default)
    return getattr(node, key, default)


def _to_plain(node: Any) -> Any:
    try:
        from omegaconf import OmegaConf

        if OmegaConf.is_config(node):
            return OmegaConf.to_object(node)
    except Exception:
        pass
    if isinstance(node, dict):
        return {k: _to_plain(v) for k, v in node.items()}
    return node


def get_loss_factories(cfg: Any, data_module: Any) -> dict:
    """Build the supervised / unsupervised factories from a hydra-style config (dict or OmegaConf)."""
    losses_cfg = _to_plain(cfg.losses) or {}
    model_type = cfg.model.model_type
    sup: dict[str, dict] = {}
    unsup: dict[str, dict] = {}

    if "heatmap" in model_type:
        sup["heatmap_" + cfg.model.heatmap_loss_type] = {"log_weight": 0.0}
        if "multiview" in model_type and _cfg_get(cfg.data, "camera_params_file"):
            lw = _cfg_get(losses_cfg.get("supervised_pairwise_projections", {}), "log_weight")
            if lw is not None:
                sup["supervised_pairwise_projections"] = {"log_weight": lw}
            lw = _cfg_get(losses_cfg.get("supervised_reprojection_heatmap_mse", {}), "log_weight")
            if lw is not None:
                dims = cfg.data.image_resize_dims
                h_img, w_img = _cfg_get(dims, "height"), _cfg_get(dims, "width")
                shrink = 2 ** _cfg_get(cfg.data, "downsample_factor", 2)
                sup["supervised_reprojection_heatmap_mse"] = {
                    "log_weight": lw,
                    "original_image_height": h_img,
                    "original_image_width": w_img,
                    "downsampled_image_height": int(h_img // shrink),
                    "downsampled_image_width": int(w_img // shrink),
                }
    else:
        sup[model_type] = {"log_weight": 0.0}

    view_names = _cfg_get(cfg.data, "view_names", None)
    true_multiview = bool(view_names) and len(view_names) > 1
    for name in (_cfg_get(cfg.model, "losses_to_use") or []):
        params = dict(losses_cfg[name])
        params["loss_name"] = name
        if name == "pca_multiview":
            mcm = _to_plain(cfg.data.mirrored_column_matches)
            if true_multiview and isinstance(mcm[0], int):
                nk = cfg.data.num_keypoints
                mcm = [(v * nk + np.asarray(mcm, dtype=int)).tolist() for v in range(len(view_names))]
            params["mirrored_column_matches"] = mcm
        elif name == "pca_singleview":
            if true_multiview:
                raise NotImplementedError("The Pose PCA loss is currently not implemented for multiview data.")
            params["columns_for_singleview_pca"] = _to_plain(_cfg_get(cfg.data, "columns_for_singleview_pca", None))
        unsup[name] = params

    return {
        "supervised": LossFactory(losses_params_dict=sup, data_module=data_module),
        "unsupervised": LossFactory(losses_params_dict=unsup, data_module=data_module),
    }


class LossFactory(_FactoryBase):
    """One object per requested loss; ``__call__`` returns the weighted total and the log list."""

    _FUSABLE = ("temporal", "pca_singleview", "pca_multiview")

    def __init__(self, losses_params_dict: dict[str, dict], data_module: Any) -> None:
        super().__init__()
        self.losses_params_dict = losses_params_dict
        self.data_module = data_module
        self._initialize_loss_instances()

    def _initialize_loss_instances(self) -> None:
        classes = get_loss_classes()
        self.loss_instance_dict = {
            name: classes[name](data_module=self.data_module, **params) for name, params in self.losses_params_dict.items()
        }

    def _fused_unsupervised(self, kwargs: dict) -> torch.Tensor | None:
        """temporal + PCA losses in one launch when at least two of them are registered."""
        names = [n for n in self._FUSABLE if n in self.loss_instance_dict]
        kp = kwargs.get("keypoints_pred")
        if len(names) < 2 or kp is None or not kp.is_cuda:
            return None
        args: dict[str, Any] = {}
        if "temporal" in names:
            t = self.loss_instance_dict["temporal"]
            args.update(temporal_eps=t.device_epsilon(kp.device), prob_threshold=float(t.prob_threshold), confidences=kwargs.get("confidences"))
        for n in ("pca_singleview", "pca_multiview"):
            if n in names:
                args[n] = self.loss_instance_dict[n].kernel_params(kp.shape[1] // 2)
        return ops.unsup_losses(kp, **args)

    def __call__(
        self,
        stage: Literal["train", "val", "test"] | None = None,
        anneal_weight: float | torch.Tensor | None = 1.0,
        **kwargs: Any,
    ) -> tuple[torch.Tensor, list[dict]]:
        fused = self._fused_unsupervised(kwargs)
        if fused is not None:
            kwargs = {**kwargs, L._FUSED_KEY: fused}
        total: torch.Tensor | None = None
        logs: list[dict] = []
        for name, inst in self.loss_instance_dict.items():
            value, entries = inst(stage=stage, **kwargs)
            weighted = inst.weight.to(value.device) * value
            anneal = 1.0 if (anneal_weight is None or name in _ANNEAL_EXEMPT) else anneal_weight
            scaled = anneal * weighted
            total = scaled if total is None else total + scaled
            logs += entries + [{"name": f"{stage}_{name}_loss_weighted", "value": weighted}]
        if total is None:
            total = torch.tensor(0.0)
        return total, logs

    def total_on_device(
        self,
        stage: Literal["train", "val", "test"] | None = None,
        anneal_weight: torch.Tensor | None = None,
        **kwargs: Any,
    ) -> tuple[torch.Tensor, list[dict]]:
        """``__call__``'s total and logs without the host, so that a training step captures into one CUDA graph.

        Each weight is made on the device by a fill kernel instead of copied from the host.  ``anneal_weight`` is a
        device scalar read by the multiply (a replay sees its value at replay time), or None for no annealing; the
        ``_ANNEAL_EXEMPT`` losses keep weight 1 either way.  The logged values are detached (what Lightning's ``log``
        keeps): a step's autograd graph must not outlive it, or the next step's backward would meet the previous
        step's gradient nodes, whose stream may be another than the one being captured."""
        fused = self._fused_unsupervised(kwargs)
        if fused is not None:
            kwargs = {**kwargs, L._FUSED_KEY: fused}
        total: torch.Tensor | None = None
        logs: list[dict] = []
        for name, inst in self.loss_instance_dict.items():
            value, entries = inst(stage=stage, **kwargs)
            weighted = torch.full((), float(inst.weight), device=value.device) * value
            scaled = weighted if (anneal_weight is None or name in _ANNEAL_EXEMPT) else anneal_weight * weighted
            total = scaled if total is None else total + scaled
            logs += [{**e, "value": e["value"].detach()} if isinstance(e["value"], torch.Tensor) else e for e in entries]
            logs.append({"name": f"{stage}_{name}_loss_weighted", "value": weighted.detach()})
        if total is None:
            raise ValueError("the loss factory holds no losses")
        return total, logs
