"""CPU: the argument checks of lpb_heatmap_loss_from_keypoints_fwd / _bwd (fused Gaussian targets + MSE / KL / JS).

Every case here is refused before anything is queued, so the fake pointers are never dereferenced and no device is
needed.  With kind LPB_HM_MSE the new entries refuse exactly what lpb_heatmap_mse_from_keypoints_* refuse; KL and JS
refuse the same cases."""
import ctypes as C

import pytest

FAKE = 0x1000
LPB_ERR_INVALID = -1
KINDS = (0, 1, 2)  # LPB_HM_MSE, LPB_HM_KL, LPB_HM_JS


def _lib():
    from lightning_pose_b200 import _lib

    return _lib.lib


def _args(n_planes=4 * 17, img_h=384.0, img_w=384.0, oh=96, ow=96, sigma=1.25, kp=FAKE, vis=FAKE, preds=FAKE, a=FAKE, b=FAKE,
          c=FAKE):
    """(common arguments, forward tail (out, workspace), backward tail (fwd_out, grad_out, grad_preds))."""
    common = [C.c_void_p(kp), C.c_void_p(vis), C.c_void_p(preds), n_planes, img_h, img_w, oh, ow, sigma]
    return common, [C.c_void_p(a), C.c_void_p(b)], [C.c_void_p(a), C.c_void_p(b), C.c_void_p(c)]


def _fwd_new(kind, **kw):
    common, fwd, _ = _args(**kw)
    return _lib().lpb_heatmap_loss_from_keypoints_fwd(*common, kind, *fwd, None)


def _bwd_new(kind, **kw):
    common, _, bwd = _args(**kw)
    return _lib().lpb_heatmap_loss_from_keypoints_bwd(*common, kind, *bwd, None)


def _fwd_mse(**kw):
    common, fwd, _ = _args(**kw)
    return _lib().lpb_heatmap_mse_from_keypoints_fwd(*common, *fwd, None)


def _bwd_mse(**kw):
    common, _, bwd = _args(**kw)
    return _lib().lpb_heatmap_mse_from_keypoints_bwd(*common, *bwd, None)


BAD = [
    {"kp": 0}, {"preds": 0}, {"a": 0}, {"b": 0},                      # null pointers (out / fwd_out, workspace / grad_out)
    {"oh": 0}, {"ow": 0}, {"oh": -3}, {"oh": 4000, "ow": 4000},         # bad heatmap shapes (oh + ow < 8000)
    {"sigma": 0.0}, {"sigma": -1.0}, {"sigma": float("nan")},          # bad sigma
    {"img_h": 0.0}, {"img_w": -5.0}, {"img_h": float("nan")},          # bad image size
    {"n_planes": 0}, {"n_planes": -1}, {"n_planes": 1 << 31}, {"n_planes": 1 << 40},  # n_planes outside [1, 2^31)
]
BAD_BWD = [{"c": 0}]  # null grad_preds (the forward has no third tail pointer)


def _ids(cases):
    return [",".join(f"{k}={v}" for k, v in c.items()) for c in cases]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bad", BAD, ids=_ids(BAD))
def test_forward_refuses(kind, bad):
    assert _fwd_new(kind, **bad) == LPB_ERR_INVALID
    assert b"heatmap_" in _lib().lpb_last_error() and b"from_keypoints_fwd" in _lib().lpb_last_error()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bad", BAD + BAD_BWD, ids=_ids(BAD + BAD_BWD))
def test_backward_refuses(kind, bad):
    assert _bwd_new(kind, **bad) == LPB_ERR_INVALID
    assert b"heatmap_" in _lib().lpb_last_error() and b"from_keypoints_bwd" in _lib().lpb_last_error()


@pytest.mark.parametrize("kind", [-1, 3, 7, 1 << 30])
def test_bad_kind_refused(kind):
    """A kind outside 0..2 is refused first, whatever else is wrong or right."""
    assert _fwd_new(kind) == LPB_ERR_INVALID
    assert _lib().lpb_last_error() == f"heatmap_loss_from_keypoints_fwd: bad kind {kind}".encode()
    assert _bwd_new(kind) == LPB_ERR_INVALID
    assert _lib().lpb_last_error() == f"heatmap_loss_from_keypoints_bwd: bad kind {kind}".encode()
    assert _fwd_new(kind, kp=0, n_planes=0) == LPB_ERR_INVALID
    assert b"bad kind" in _lib().lpb_last_error()


@pytest.mark.parametrize("bad", BAD + BAD_BWD, ids=_ids(BAD + BAD_BWD))
def test_mse_kind_refuses_what_the_mse_entry_refuses(bad):
    """Same status and same message as lpb_heatmap_mse_from_keypoints_*: kind LPB_HM_MSE runs that entry."""
    if "c" not in bad:
        assert _fwd_mse(**bad) == LPB_ERR_INVALID
        want = _lib().lpb_last_error()
        assert _fwd_new(0, **bad) == LPB_ERR_INVALID
        assert _lib().lpb_last_error() == want
    assert _bwd_mse(**bad) == LPB_ERR_INVALID
    want = _lib().lpb_last_error()
    assert _bwd_new(0, **bad) == LPB_ERR_INVALID
    assert _lib().lpb_last_error() == want


def test_null_visibility_is_not_refused_by_the_checks():
    """visibility may be null ("visibility is None"); a null visibility together with one bad argument is refused for
    that argument alone."""
    for kind in KINDS:
        assert _fwd_new(kind, vis=0, n_planes=0) == LPB_ERR_INVALID
        assert b"bad n_planes" in _lib().lpb_last_error()
        assert _bwd_new(kind, vis=0, sigma=0.0) == LPB_ERR_INVALID
        assert b"bad shape" in _lib().lpb_last_error()


def test_ops_wrapper_checks_shapes_without_gpu():
    """ops.heatmap_loss_from_keypoints refuses CPU tensors (no CPU fallback)."""
    import torch

    from lightning_pose_b200 import ops

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.heatmap_loss_from_keypoints("kl", torch.zeros(2, 3, 2), torch.zeros(2, 3, 8, 8), 32, 32)
