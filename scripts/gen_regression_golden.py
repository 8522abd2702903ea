"""Write tests/golden/regression.npz: the reference's own regression head, losses and affine undo on seeded inputs.

    python scripts/gen_regression_golden.py        (needs the reference tree; the tests then need neither it nor this script)

Runs lightning_pose.models.heads.regression.LinearRegressionHead, losses.losses.RegressionMSELoss / RegressionRMSELoss
and data.utils.undo_affine_transform through oracle/ref_loader.py (unmodified reference files).  Stored:
``head_*`` (features (B, C, 1, 1), the module's parameters under their state-dict keys as ``head_param_<key>``, its
output), ``loss_<case>_{targ,pred,mse,rmse}`` for NaN patterns including x-only NaN pairs and an all-NaN batch, and
``affine_{kp,tf,out}``.  The script asserts that tests/regression_oracle.py reproduces every value.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import regression_oracle as O  # noqa: E402
from oracle import ref_loader  # noqa: E402


def main() -> None:
    heads = ref_loader.load("lightning_pose.models.heads.regression")
    losses = ref_loader.load("lightning_pose.losses.losses")
    utils = ref_loader.load("lightning_pose.data.utils")
    torch.manual_seed(20261017)
    out: dict[str, np.ndarray] = {}

    head = heads.LinearRegressionHead(48, 34).double()
    feats = torch.randn(5, 48, 1, 1, dtype=torch.float64)
    out["head_features"] = feats.numpy()
    for k, v in head.state_dict().items():
        out[f"head_param_{k}"] = v.numpy()
    out["head_out"] = head(feats).detach().numpy()
    np.testing.assert_allclose(O.head_forward(feats.numpy(), head.linear_layer.weight.detach().numpy(),
                                              head.linear_layer.bias.detach().numpy())[0], out["head_out"], rtol=1e-12, atol=1e-12)

    nan = float("nan")
    targ = torch.rand(4, 10, dtype=torch.float64) * 100
    pred = targ + torch.randn(4, 10, dtype=torch.float64) * 3
    cases = {"clean": targ.clone()}
    t = targ.clone()
    t[0, 2:4] = nan  # a whole keypoint
    t[2, 6:8] = nan
    cases["whole_pairs"] = t
    t = targ.clone()
    t[0, 2] = nan  # x only: every later pair shifts by one entry ...
    t[3, 5] = nan  # ... until a y-only NaN brings the count back to even
    cases["x_only_shift"] = t
    t = targ.clone()
    t[1, 0] = nan
    t[1, 3] = nan
    t[2, :] = nan
    cases["mixed"] = t
    cases["all_nan"] = torch.full_like(targ, nan)
    mse_fn, rmse_fn = losses.RegressionMSELoss(), losses.RegressionRMSELoss()
    for name, t in cases.items():
        mse, _ = mse_fn(keypoints_targ=t, keypoints_pred=pred)
        rmse, _ = rmse_fn(keypoints_targ=t, keypoints_pred=pred)
        out[f"loss_{name}_targ"], out[f"loss_{name}_pred"] = t.numpy(), pred.numpy()
        out[f"loss_{name}_mse"], out[f"loss_{name}_rmse"] = np.float64(mse), np.float64(rmse)
        np.testing.assert_allclose(O.regression_mse(t.numpy(), pred.numpy())[0], float(mse), rtol=1e-12, equal_nan=True)
        np.testing.assert_allclose(O.regression_rmse(t.numpy(), pred.numpy()), float(rmse), rtol=1e-12, equal_nan=True)

    kp = torch.rand(6, 17, 2, dtype=torch.float64) * 256
    tf = torch.tensor([[1.1, -0.2, 12.0], [0.15, 0.9, -7.5]], dtype=torch.float64)
    res = utils.undo_affine_transform(kp, tf)
    out["affine_kp"], out["affine_tf"], out["affine_out"] = kp.numpy(), tf.numpy(), res.detach().numpy()
    np.testing.assert_allclose(O.undo_affine(kp.numpy(), tf.numpy()), out["affine_out"], rtol=1e-10, atol=1e-9)

    path = os.path.join(ROOT, "tests", "golden", "regression.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == "__main__":
    main()
