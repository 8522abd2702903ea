"""CPU: the float64 regression oracle (tests/regression_oracle.py) against the reference's own outputs
(tests/golden/regression.npz, written by scripts/gen_regression_golden.py), and the regression surface the reference's
model factory reads (lightning_pose/models/factory.py:116-192)."""
import inspect
import typing

import numpy as np
import pytest
import torch

import regression_oracle as O


def test_head_matches_reference(golden):
    g = golden("regression")
    out, _ = O.head_forward(g["head_features"], g["head_param_linear_layer.weight"], g["head_param_linear_layer.bias"])
    np.testing.assert_allclose(out, g["head_out"], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("case", ["clean", "whole_pairs", "x_only_shift", "mixed", "all_nan"])
def test_losses_match_reference(golden, case):
    g = golden("regression")
    t, p = g[f"loss_{case}_targ"], g[f"loss_{case}_pred"]
    np.testing.assert_allclose(O.regression_mse(t, p)[0], g[f"loss_{case}_mse"], rtol=1e-12, equal_nan=True)
    np.testing.assert_allclose(O.regression_rmse(t, p), g[f"loss_{case}_rmse"], rtol=1e-12, equal_nan=True)


def test_x_only_nan_shifts_the_rmse_pairing(golden):
    """The reference compacts before it pairs: one x-only NaN re-pairs every later entry, so its RMSE is not the mean
    over keypoints with both coordinates kept."""
    g = golden("regression")
    t, p = g["loss_x_only_shift_targ"].ravel(), g["loss_x_only_shift_pred"].ravel()
    both = ~np.isnan(t.reshape(-1, 2)).any(1)
    per_keypoint = np.sqrt(((t - p).reshape(-1, 2)[both] ** 2).mean(1)).mean()
    assert abs(float(g["loss_x_only_shift_rmse"]) - per_keypoint) > 1e-3
    assert np.isnan(g["loss_all_nan_mse"]) and np.isnan(g["loss_all_nan_rmse"])


def test_affine_undo_matches_reference(golden):
    g = golden("regression")
    np.testing.assert_allclose(O.undo_affine(g["affine_kp"], g["affine_tf"]), g["affine_out"], rtol=1e-10, atol=1e-9)


def test_head_loads_reference_state_dict(golden):
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead

    g = golden("regression")
    ref = {k[len("head_param_"):]: torch.from_numpy(g[k]).float() for k in g.files if k.startswith("head_param_")}
    head = LinearRegressionHead(48, 34)
    assert set(head.state_dict()) == set(ref) == {"linear_layer.weight", "linear_layer.bias"}
    head.load_state_dict(ref)  # strict
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        head(torch.from_numpy(g["head_features"]).float())


def test_tracker_loads_reference_layout_state_dict():
    """The reference's regression backbone is torchvision's children up to and including avgpool; avgpool has no
    parameters, so its state dict is the one of the backbone cut before avgpool, and a reference checkpoint loads."""
    import torchvision.models as tvm
    from torch import nn

    from lightning_pose_b200.models.heads.regression import LinearRegressionHead
    from lightning_pose_b200.models.regression_tracker import RegressionTracker

    torch.manual_seed(0)
    ref_backbone = nn.Sequential(*list(tvm.resnet18(weights=None).children())[:-1])  # keeps avgpool (factory.py:324)
    ref_sd = {f"backbone.{k}": v for k, v in ref_backbone.state_dict().items()}
    ref_sd.update({f"head.{k}": v for k, v in LinearRegressionHead(512, 10).state_dict().items()})
    m = RegressionTracker(5, backbone="resnet18", pretrained=False)
    assert set(m.state_dict()) == set(ref_sd)
    m.load_state_dict(ref_sd)
    assert torch.equal(m.backbone[0].weight, ref_sd["backbone.0.weight"])


def test_tracker_surface():
    from lightning_pose_b200.models.regression_tracker import RegressionTracker, SemiSupervisedRegressionTracker

    lab = typing.get_type_hints(RegressionTracker.get_loss_inputs_labeled)["return"]
    unl = typing.get_type_hints(SemiSupervisedRegressionTracker.get_loss_inputs_unlabeled)["return"]
    assert set(lab.__annotations__) == {"keypoints_targ", "keypoints_pred"}
    assert set(unl.__annotations__) == {"keypoints_pred"}
    assert list(inspect.signature(RegressionTracker.__init__).parameters)[1:10] == [
        "num_keypoints", "loss_factory", "backbone", "pretrained", "torch_seed", "optimizer", "optimizer_params",
        "lr_scheduler", "lr_scheduler_params"]
    assert list(inspect.signature(SemiSupervisedRegressionTracker.__init__).parameters)[1:11] == [
        "num_keypoints", "loss_factory", "loss_factory_unsupervised", "backbone", "pretrained", "torch_seed", "optimizer",
        "optimizer_params", "lr_scheduler", "lr_scheduler_params"]
    assert list(inspect.signature(RegressionTracker.predict_step).parameters)[1:3] == ["batch_dict", "batch_idx"]
    m = SemiSupervisedRegressionTracker(17, backbone="resnet18", pretrained=False, do_context=False)
    assert [g["name"] for g in m.get_parameters()] == ["backbone", "head"] and m.get_parameters()[0]["lr"] == 0
    assert m.num_targets == 34 and float(m.total_unsupervised_importance) == 1.0
    assert m.head.linear_layer.in_features == 512 and m.head.linear_layer.out_features == 34
    with pytest.raises(ValueError, match="ViT"):
        RegressionTracker(17, backbone="vits_dino")


def test_loss_factories_for_regression_models():
    from lightning_pose_b200.losses import losses as L
    from lightning_pose_b200.losses.factory import get_loss_factories

    cfg = type("Cfg", (), {})()
    cfg.losses = {"temporal": {"log_weight": 5.0, "epsilon": 20.0, "prob_threshold": 0.05}}
    cfg.model = type("M", (), {"model_type": "regression", "losses_to_use": ["temporal"]})()
    cfg.data = type("D", (), {})()
    f = get_loss_factories(cfg, None)
    assert list(f["supervised"].loss_instance_dict) == ["regression"]
    assert isinstance(f["supervised"].loss_instance_dict["regression"], L.RegressionMSELoss)
    assert list(f["unsupervised"].loss_instance_dict) == ["temporal"]


def test_regression_losses_stay_staged_on_cpu(golden):
    """On CPU tensors RegressionMSELoss keeps the staged pipeline, and the heatmap trackers' RMSE diagnostic is staged on
    every device."""
    from lightning_pose_b200.losses import losses as L

    g = golden("regression")
    t, p = torch.from_numpy(g["loss_mixed_targ"]), torch.from_numpy(g["loss_mixed_pred"])
    mse, logs = L.RegressionMSELoss()(keypoints_targ=t, keypoints_pred=p, stage="train")
    assert float(mse) == pytest.approx(float(g["loss_mixed_mse"]), rel=1e-12) and logs[0]["name"] == "train_regression_loss"
    rmse, _ = L.RegressionRMSELoss()(keypoints_targ=t, keypoints_pred=p)
    assert float(rmse) == pytest.approx(float(g["loss_mixed_rmse"]), rel=1e-12)
