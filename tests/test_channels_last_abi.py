"""Channels-last features: the C ABI's declarations and planning queries, the packing oracle, and the stride logic of the
Python layers.  No GPU."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import channels_last_oracle as O
from lightning_pose_b200 import _lib, ops
from lightning_pose_b200.models.backbones import tokens_to_feature_map

HEADER = (Path(__file__).resolve().parents[1] / "include" / "lpb200.h").read_text()
NCHW, NHWC = ops.FEATURES_NCHW, ops.FEATURES_NHWC
NEW = ["lpb_head_bf16_plan_layout", "lpb_head_fwd_bf16_layout", "lpb_head_fwd_f16_layout",
       "lpb_head_bwd_bf16_workspace_bytes_layout", "lpb_head_bwd_bf16_layout"]


def _ctype(decl):
    decl = decl.strip()
    if "*" in decl:
        if re.match(r"(const )?size_t\*", decl):
            return ctypes.POINTER(ctypes.c_size_t)
        if re.match(r"int\*", decl):
            return ctypes.POINTER(ctypes.c_int)
        return ctypes.c_void_p
    return {"int": ctypes.c_int, "float": ctypes.c_float, "int64_t": ctypes.c_int64}[decl.split()[0]]


@pytest.mark.parametrize("name", NEW)
def test_prototypes_match_ctypes(name):
    m = re.search(rf"\bint {name}\(([^;]*)\);", HEADER)
    assert m, f"{name} is not declared in lpb200.h"
    args = [_ctype(a) for a in m.group(1).replace("\n", " ").split(",")]
    fn = getattr(_lib.lib, name)
    assert fn.restype is ctypes.c_int
    assert list(fn.argtypes) == args
    # its unsuffixed sibling has the same arguments less the layout
    base = re.search(rf"\bint {name[: -len('_layout')]}\(([^;]*)\);", HEADER)
    assert len(base.group(1).split(",")) == len(args) - 1


def test_layout_constants():
    for name, value in (("LPB_FEATURES_NCHW", NCHW), ("LPB_FEATURES_NHWC", NHWC), ("LPB_SHUFFLE_NHWC", ops._SHUFFLE_NHWC)):
        assert re.search(rf"#define {name} {value}\b", HEADER)


def _plan(c, h, w, c1, c2, layout):
    plan = ctypes.c_int(-1)
    rc = _lib.lib.lpb_head_bf16_plan_layout(c, h, w, c1, c2, layout, ctypes.byref(plan))
    return rc, plan.value


@pytest.mark.parametrize("shape", [(2048, 12, 12, 17, 17), (2048, 16, 16, 17, 17), (512, 8, 12, 17, 17), (384, 16, 16, 17, 0),
                                   (384, 24, 24, 17, 0), (2048, 8, 12, 51, 51)])
def test_plan_and_sizes_per_layout(shape):
    c, h, w, c1, c2 = shape
    old = ctypes.c_int(-1)
    assert _lib.lib.lpb_head_bf16_plan(c, h, w, c1, c2, ctypes.byref(old)) == 0
    assert _plan(c, h, w, c1, c2, NCHW) == (0, old.value)
    assert _plan(c, h, w, c1, c2, NHWC) == (0, 0)  # channels-last features always take the banded kernels
    a, b = ctypes.c_size_t(0), ctypes.c_size_t(1)
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes(4, c, h, w, c1, c2, ctypes.byref(a)) == 0
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes_layout(4, c, h, w, c1, c2, NHWC, ctypes.byref(b)) == 0
    assert a.value == b.value > 0
    assert ops.head_bf16_supported((4, c, h, w), [c1, c2][: 2 if c2 else 1], train=True, layout=NHWC)


def test_queries_refuse_what_the_kernels_do_not_serve():
    n = ctypes.c_size_t(0)
    assert _plan(384, 16, 16, 17, 0, 2)[0] != 0  # unknown layout
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes_layout(4, 384, 16, 16, 17, 0, 2, ctypes.byref(n)) != 0
    assert _plan(384, 16, 16, 17, 0, NHWC)[0] == 0 and _plan(200, 16, 16, 17, 0, NHWC)[0] != 0  # C % 128
    # W = 32 trains from NCHW only (the transposing tile of the data gradient does not fit beside its operands) ...
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes_layout(4, 384, 32, 32, 17, 0, NCHW, ctypes.byref(n)) == 0
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes_layout(4, 384, 32, 32, 17, 0, NHWC, ctypes.byref(n)) != 0
    assert b"width 32" in _lib.lib.lpb_last_error()
    # ... and predicts from both
    assert _plan(384, 32, 32, 17, 0, NHWC) == (0, 0)
    # a 64 x 64 map exceeds the NCHW shuffle stage's shared memory, which the channels-last kernel does not use
    assert _plan(384, 60, 60, 17, 0, NCHW)[0] != 0 and _plan(384, 60, 60, 17, 0, NHWC) == (0, 0)


def test_feature_layout_detection():
    x = torch.zeros(2, 8, 4, 6)
    assert ops.feature_layout(x) == NCHW
    assert ops.feature_layout(x.contiguous(memory_format=torch.channels_last)) == NHWC
    assert ops.feature_layout(torch.zeros(2, 1, 4, 6).contiguous(memory_format=torch.channels_last)) == NCHW  # both formats
    assert ops.feature_layout(torch.zeros(2, 8, 1, 1).contiguous(memory_format=torch.channels_last)) == NCHW
    cl = x.contiguous(memory_format=torch.channels_last)
    assert ops.feature_layout(cl[1:]) == NHWC  # whole frames of a channels-last batch stay dense
    assert ops.feature_layout(cl[:, :4]) == NCHW and ops.feature_layout(cl[:, :, 1:]) == NCHW  # neither: copied


def test_tokens_to_feature_map_and_forward_vit():
    tokens = torch.arange(2 * 12 * 8, dtype=torch.float32).reshape(2, 12, 8)
    fm = tokens_to_feature_map(tokens, (3, 4))
    assert fm.shape == (2, 8, 3, 4) and fm.data_ptr() == tokens.data_ptr()
    assert ops.feature_layout(fm) == NHWC
    assert torch.equal(fm, tokens.reshape(2, 3, 4, 8).permute(0, 3, 1, 2).contiguous())
    with pytest.raises(ValueError):
        tokens_to_feature_map(tokens, (3, 3))

    from lightning_pose_b200.models.heatmap_tracker_multiview import HeatmapTrackerMultiviewTransformer

    embed = lambda im: im.flatten(1)[:, : 16 * 128].reshape(im.shape[0], 16, 128)  # noqa: E731
    model = HeatmapTrackerMultiviewTransformer(num_keypoints=3, num_views=2, patch_embed=embed, encoder=lambda t: t * 2.0, embedding_dim=128)
    images = torch.randn(4, 3, 32, 32)
    default, view = model.forward_vit(images), model.forward_vit(images, channels_last=True)
    assert default.shape == (4, 128, 4, 4) and default.is_contiguous()
    assert ops.feature_layout(view) == NHWC and torch.equal(default, view)
    # what the method returned before the view existed
    tok = embed(images) + model.view_embeddings[torch.arange(2).repeat(2)].unsqueeze(1)
    seq = tok.reshape(2, 32, 128) * 2.0
    assert torch.equal(default, seq.reshape(2, 2, 4, 4, 128).permute(0, 1, 4, 2, 3).reshape(4, 128, 4, 4))


@pytest.mark.parametrize("shape", [(2, 64, 2, 4), (1, 32, 4, 2), (3, 128, 2, 2)])
def test_packing_oracle_layouts_agree(shape):
    rng = np.random.default_rng(5)
    feat = rng.integers(1, 2**16, size=shape, dtype=np.uint16)
    a = O.pack_rows_nchw(feat)
    b = O.pack_rows_nhwc(np.ascontiguousarray(feat.transpose(0, 2, 3, 1)))
    assert a.tobytes() == b.tobytes()
    # entry q = 2 di + dj of a pixel holds source channels q, 4 + q, ... of the K-chunk
    pp, lead, rows = O.row_layout(2 * shape[2], 2 * shape[3])
    assert a.shape == (shape[0], shape[1] // 32, rows, 8)
    i, j, kc = 1, 1, shape[1] // 32 - 1
    for q in range(4):
        row = lead + (2 * i + q // 2) * pp + 2 * j + q % 2
        assert np.array_equal(a[0, kc, row], feat[0, 32 * kc + q : 32 * kc + 32 : 4, i, j])
    assert not a[:, :, :lead].any() and not a[:, :, lead + pp - 1].any()  # pads
    assert np.count_nonzero(a) == feat.size
