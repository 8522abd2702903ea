"""CPU: the fp16 head forward and the ingest output-format codes validate their arguments without a GPU.

lpb_head_fwd_f16 shares the bf16 forward's plan, buffer sizes and alignment rules; its errors name it.  The ingest entries
take an output-format code (LPB_OUT_F32 = 0, LPB_OUT_BF16 = 1, LPB_OUT_F16 = 2) and refuse any other before anything is
queued; the training-only augmented ingest refuses fp16."""
import ctypes

import pytest

FAKE = 0x1000  # a 16-byte-aligned fake device pointer: nothing may be queued with it


def _lib():
    from lightning_pose_b200._lib import lib

    return lib


def _fwd(lib, p, b=2, c=2048, h=12, w=12, c1=17, c2=17):
    return lib.lpb_head_fwd_f16(p["features"], b, c, h, w, p["w1"], p["b1"], c1, p["w2"] if c2 else None, p["b2"] if c2 else None, c2, 1,
                                p["out"], p["saved_xs"], p["workspace"], None)


def _ptrs(**over):
    p = {name: FAKE for name in ("features", "w1", "b1", "w2", "b2", "out", "saved_xs", "workspace")}
    p.update(over)
    return p


@pytest.mark.parametrize("missing", ["features", "w1", "b1", "out", "workspace"])
def test_head_fwd_f16_refuses_null_pointers(missing):
    lib = _lib()
    assert _fwd(lib, _ptrs(**{missing: None})) == -1
    assert lib.lpb_last_error() == b"head_fwd_f16: null pointer"


@pytest.mark.parametrize("misaligned,addr,need", [("features", 0x1002, 16), ("saved_xs", 0x1008, 16), ("workspace", 0x1004, 16),
                                                   ("out", 0x1004, 8)])
@pytest.mark.parametrize("c,h,w,c2", [(2048, 12, 12, 17), (384, 16, 16, 0)])  # fast path, banded path
def test_head_fwd_f16_refuses_misaligned_buffers(misaligned, addr, need, c, h, w, c2):
    lib = _lib()
    assert _fwd(lib, _ptrs(**{misaligned: addr}), c=c, h=h, w=w, c2=c2) == -1
    assert lib.lpb_last_error() == f"head_fwd_f16: {misaligned} must be {need}-byte aligned".encode()


@pytest.mark.parametrize("c,h,w,c1,c2,msg", [
    (100, 12, 12, 17, 17, b"head_fwd_f16: bad feature shape"),              # C % 128
    (2048, 13, 13, 17, 17, b"head_fwd_f16: H*W must be a multiple of 8"),
    (2048, 12, 12, 20, 17, b"head_fwd_f16: channel counts 20/17"),          # no room for the ones channel
    (2048, 12, 12, 17, 81, b"head_fwd_f16: channel counts 17/81"),          # past LPB_HEAD_MAX_CHANNELS
])
def test_head_fwd_f16_refuses_unsupported_shapes(c, h, w, c1, c2, msg):
    lib = _lib()
    assert _fwd(lib, _ptrs(), c=c, h=h, w=w, c1=c1, c2=c2) == -1
    assert lib.lpb_last_error().startswith(msg), lib.lpb_last_error()


def test_head_fwd_f16_needs_the_second_layer():
    lib = _lib()
    p = _ptrs(w2=None)
    rc = lib.lpb_head_fwd_f16(p["features"], 2, 2048, 12, 12, p["w1"], p["b1"], 17, None, None, 17, 1, p["out"], p["saved_xs"], p["workspace"], None)
    assert rc == -1 and lib.lpb_last_error() == b"head_fwd_f16: a two-deconv head needs w2 and b2"


def test_head_fwd_bf16_messages_unchanged():
    """The shared implementation still names the bf16 entry in the bf16 entry's errors."""
    lib = _lib()
    p = _ptrs(features=None)
    rc = lib.lpb_head_fwd_bf16(p["features"], 2, 2048, 12, 12, p["w1"], p["b1"], 17, p["w2"], p["b2"], 17, 1, p["out"], p["saved_xs"], p["workspace"], None)
    assert rc == -1 and lib.lpb_last_error() == b"head_fwd_bf16: null pointer"


def _f3(*v):
    return (ctypes.c_float * 3)(*v)


M3, S3 = _f3(0.485, 0.456, 0.406), _f3(0.229, 0.224, 0.225)


@pytest.mark.parametrize("fmt", [3, -1])
def test_ingest_entries_refuse_unknown_formats(fmt):
    lib = _lib()
    p = ctypes.c_void_p(FAKE)
    assert lib.lpb_frames_normalize(p, 1, 8, 8, 8, 8, M3, S3, 0, fmt, p, None) == -1
    assert lib.lpb_last_error() == f"frames_normalize: unknown output format {fmt}".encode()
    ptrs, hw = (ctypes.c_void_p * 1)(FAKE), (ctypes.c_int * 1)(8)
    assert lib.lpb_frames_normalize_views(ptrs, 1, 1, hw, hw, 8, 8, M3, S3, 0, fmt, p, None) == -1
    assert lib.lpb_last_error() == f"frames_normalize_views: unknown output format {fmt}".encode()
    assert lib.lpb_frames_crop_normalize(p, 0, 1, 8, 8, p, 1, None, 0, 8, 8, M3, S3, 0, fmt, p, p, None) == -1
    assert lib.lpb_last_error() == f"frames_crop_normalize: unknown output format {fmt}".encode()


def test_augmented_ingest_refuses_fp16():
    """Augmentation serves training, which reads fp32 or bf16 frames only."""
    lib = _lib()
    p = ctypes.c_void_p(FAKE)
    for fmt in (2, 3):
        assert lib.lpb_frames_augment_normalize(p, 1, 8, 8, 8, 8, p, p, M3, S3, 0, fmt, p, p, None) == -1
        assert lib.lpb_last_error().startswith(f"frames_augment_normalize: output format {fmt}".encode())


def test_python_wrappers_take_fp16():
    """The ingest wrappers map float16 to its format code; augmentation keeps refusing it.  (Checked on the dtype
    argument alone: the frames are CPU tensors, refused afterwards for want of a GPU.)"""
    import torch

    from lightning_pose_b200 import ops

    assert ops._out_format(torch.float16) == 2 and ops._out_format(torch.bfloat16) == 1 and ops._out_format(torch.float32) == 0
    with pytest.raises(ValueError, match="float32, bfloat16 or float16"):
        ops._out_format(torch.float64)
    assert set(ops._HEAD_FWD_16) == {torch.bfloat16, torch.float16}
