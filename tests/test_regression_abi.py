"""CPU: argument validation of the regression entries (lpb_regression_head_fwd/_bwd, lpb_regression_losses_fwd/_bwd).
Every refusal happens before anything is queued; the pointers are fake, so a launch or CUDA call would show here."""
import ctypes as C

import pytest

FAKE = C.c_void_p(0x1000)
BF16, F32, NCHW, NHWC = 1, 0, 0, 1


def lib():
    from lightning_pose_b200 import _lib

    return _lib.lib


def fwd(**kw):
    a = dict(features=FAKE, format=BF16, layout=NCHW, B=2, C=64, H=12, W=12, weight=FAKE, bias=FAKE, n_out=34, pooled=FAKE,
             out=FAKE)
    a.update(kw)
    return lib().lpb_regression_head_fwd(*a.values(), None)


def bwd(**kw):
    a = dict(grad_out=FAKE, pooled=FAKE, weight=FAKE, format=BF16, layout=NCHW, B=2, C=64, H=12, W=12, n_out=34, dfeatures=FAKE,
             dweight=FAKE, dbias=FAKE, workspace=FAKE)
    a.update(kw)
    return lib().lpb_regression_head_bwd(*a.values(), None)


def refused(rc, msg):
    assert rc == -1, rc
    assert msg in lib().lpb_last_error().decode()


@pytest.mark.parametrize("name", ["features", "weight", "bias", "pooled", "out"])
def test_head_fwd_refuses_null_pointers(name):
    refused(fwd(**{name: None}), "regression_head_fwd: null pointer")


@pytest.mark.parametrize("name", ["grad_out", "pooled", "weight"])
def test_head_bwd_refuses_null_pointers(name):
    refused(bwd(**{name: None}), "regression_head_bwd: null pointer")


@pytest.mark.parametrize("entry", [fwd, bwd])
def test_head_refuses_unknown_codes_and_shapes(entry):
    name = entry.__name__
    refused(entry(format=3), f"regression_head_{name}: unknown feature format 3")
    refused(entry(format=-1), f"regression_head_{name}: unknown feature format -1")
    refused(entry(layout=2), f"regression_head_{name}: unknown feature layout 2")
    for shape in (dict(B=-1), dict(C=0), dict(H=0), dict(W=-3), dict(n_out=0), dict(C=1 << 20, H=64, W=64)):
        refused(entry(**shape), f"regression_head_{name}: bad shape")


def test_head_empty_batch_is_a_no_op():
    assert fwd(B=0, features=None, pooled=None, out=None) == 0


def test_head_refuses_misaligned_features():
    refused(fwd(features=C.c_void_p(0x1001)), "regression_head_fwd: features must be 2-byte aligned")
    refused(fwd(format=F32, features=C.c_void_p(0x1002)), "regression_head_fwd: features must be 4-byte aligned")
    refused(bwd(dfeatures=C.c_void_p(0x1001)), "regression_head_bwd: dfeatures must be 2-byte aligned")


def test_head_bwd_output_pairs():
    refused(bwd(dbias=None), "dweight and dbias are given together")
    refused(bwd(dweight=None), "dweight and dbias are given together")
    refused(bwd(workspace=None), "d features need a workspace")


def test_losses_validate():
    L = lib()
    refused(L.lpb_regression_losses_fwd(FAKE, FAKE, -1, FAKE, None), "regression_losses_fwd: bad shape")
    refused(L.lpb_regression_losses_fwd(FAKE, FAKE, 8, None, None), "regression_losses_fwd: null pointer")
    refused(L.lpb_regression_losses_fwd(None, FAKE, 8, FAKE, None), "regression_losses_fwd: null pointer")
    refused(L.lpb_regression_losses_bwd(FAKE, FAKE, -2, FAKE, FAKE, FAKE, None), "regression_losses_bwd: bad shape")
    for i in range(5):
        args = [FAKE] * 5
        args[i] = None
        refused(L.lpb_regression_losses_bwd(args[0], args[1], 8, args[2], args[3], args[4], None), "regression_losses_bwd: null pointer")
    assert L.lpb_regression_losses_bwd(None, None, 0, None, None, None, None) == 0


def test_python_side_refuses_cpu_and_bad_inputs():
    import torch

    from lightning_pose_b200 import ops

    w, b = torch.zeros(34, 64), torch.zeros(34)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.regression_head(torch.zeros(2, 64, 3, 3), w, b)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.regression_losses(torch.zeros(2, 34), torch.zeros(2, 34))
