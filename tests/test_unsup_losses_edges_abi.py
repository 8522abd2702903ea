"""CPU: ops.unsup_losses refuses PCA keypoint indices outside [0, K) before anything reaches the device.

The kernels read keypoint ``kp_index[i]`` of every frame, so an index past K (or below 0) would read another clip's
keypoints or past the buffer.  ``PcaParams`` keeps the index range on the host when it is built, and ``unsup_losses``
compares it with the K of the keypoints it is given: no device copy and no sync.  The refusal comes before the
device check, so it is testable without a GPU."""
import numpy as np
import pytest
import torch

K = 5


def _ops():
    from lightning_pose_b200 import ops

    return ops


def _sv(idx, device="cpu"):
    idx = np.asarray(idx, np.int32)
    d = 2 * len(idx)
    return _ops().PcaParams(idx, len(idx), 0, None, np.zeros(d, np.float32), np.eye(d, dtype=np.float32)[:1], 1.0, device)


def _mv(mcm, device="cpu"):
    mcm = np.asarray(mcm, np.int32)
    views, n_sel = mcm.shape
    d = 2 * views
    return _ops().PcaParams(mcm.reshape(-1), n_sel, views, None, np.zeros(d, np.float32), np.eye(d, dtype=np.float32)[:1],
                            1.0, device)


def test_index_range_is_kept_on_the_host():
    sv = _sv([3, 0, 4, 4])
    assert (sv.kp_index_min, sv.kp_index_max) == (0, 4)
    mv = _mv([[2, 1], [0, 3]])
    assert (mv.kp_index_min, mv.kp_index_max) == (0, 3)


@pytest.mark.parametrize("idx", [[0, K], [K + 7], [-1, 2], [1, 2, 1 << 20]], ids=["K", "K+7", "-1", "2^20"])
@pytest.mark.parametrize("batched", [False, True], ids=["T,2K", "clips,T,2K"])
def test_singleview_index_out_of_range_is_refused(idx, batched):
    kp = torch.zeros((3, 4, 2 * K) if batched else (4, 2 * K))
    with pytest.raises(ValueError, match=r"pca_singleview: keypoint indices span .* outside \[0, 5\)"):
        _ops().unsup_losses(kp, pca_singleview=_sv(idx))


@pytest.mark.parametrize("mcm", [[[0, 1], [2, K]], [[-3, 1], [2, 3]]], ids=["K", "-3"])
def test_multiview_index_out_of_range_is_refused(mcm):
    with pytest.raises(ValueError, match=r"pca_multiview: keypoint indices span .* outside \[0, 5\)"):
        _ops().unsup_losses(torch.zeros(4, 2 * K), temporal_eps=1.0, pca_singleview=_sv([0, 1]), pca_multiview=_mv(mcm))


def test_in_range_indices_pass_the_check():
    """Indices 0 and K - 1 are in range: the call gets past the index check to the device check (no CPU fallback)."""
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _ops().unsup_losses(torch.zeros(4, 2 * K), pca_singleview=_sv([K - 1, 0]), pca_multiview=_mv([[0, 1], [K - 1, 2]]))
