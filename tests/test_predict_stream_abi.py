"""CPU: lpb_context_ring_push / lpb_context_ring_select refuse null or misaligned pointers and bad sizes with
LPB_ERR_INVALID before they queue anything (the pointers below are fake, so a queued kernel or a CUDA call would show
as a different code), and FramePredictor.push_frame refuses what it cannot stream before it touches the device."""
import ctypes as C

import numpy as np
import pytest

LPB_ERR_INVALID = -1
GOOD = 0x1000  # 16-byte aligned
PUSH_PTRS = ("wf", "wb", "kp_sf", "conf_sf", "bbox", "ring_wf", "ring_wb", "ring_kp", "ring_conf", "ring_box", "count",
             "window_index")
SELECT_PTRS = ("ring_kp", "ring_conf", "ring_box", "kp_mf", "conf_mf", "out", "count")


def _push(K=17, H=64, W=64, **ptrs):
    from lightning_pose_b200 import _lib

    p = {name: GOOD for name in PUSH_PTRS} | ptrs
    return _lib.lib.lpb_context_ring_push(*(C.c_void_p(p[n]) for n in PUSH_PTRS[:5]), K, H, W,
                                          *(C.c_void_p(p[n]) for n in PUSH_PTRS[5:]), None)


def _select(K=17, model_height=256.0, model_width=256.0, **ptrs):
    from lightning_pose_b200 import _lib

    p = {name: GOOD for name in SELECT_PTRS} | ptrs
    return _lib.lib.lpb_context_ring_select(*(C.c_void_p(p[n]) for n in SELECT_PTRS[:5]), K, model_height, model_width,
                                            C.c_void_p(p["out"]), C.c_void_p(p["count"]), None)


PUSH_BAD = ([{n: 0} for n in PUSH_PTRS]                                               # null pointers
            + [{n: GOOD + 8} for n in ("wf", "wb", "ring_wf", "ring_wb")]            # maps: 16 bytes
            + [{"count": GOOD + 4}, {"kp_sf": GOOD + 2}, {"ring_box": GOOD + 1}, {"window_index": GOOD + 2}]
            + [{"K": 0}, {"K": -3}, {"K": 65537}, {"H": 0}, {"W": 0}, {"H": 63}, {"W": 7}, {"H": -2}])
SELECT_BAD = ([{n: 0} for n in SELECT_PTRS]
              + [{"count": GOOD + 4}, {"out": GOOD + 2}, {"kp_mf": GOOD + 1}, {"ring_conf": GOOD + 3}]
              + [{"K": 0}, {"K": -1}, {"K": 65537}, {"model_height": 0.0}, {"model_width": -1.0},
                 {"model_height": float("nan")}])


def _ids(d):
    return ",".join(f"{k}={v}" for k, v in d.items())


@pytest.mark.parametrize("bad", PUSH_BAD, ids=_ids)
def test_ring_push_refuses(bad):
    from lightning_pose_b200 import _lib

    assert _push(**bad) == LPB_ERR_INVALID, _lib.lib.lpb_last_error()
    assert b"context_ring_push" in _lib.lib.lpb_last_error()


@pytest.mark.parametrize("bad", SELECT_BAD, ids=_ids)
def test_ring_select_refuses(bad):
    from lightning_pose_b200 import _lib

    assert _select(**bad) == LPB_ERR_INVALID, _lib.lib.lpb_last_error()
    assert b"context_ring_select" in _lib.lib.lpb_last_error()


def _predictor(kind):
    """A FramePredictor on a CPU head: construction touches no device, and push_frame refuses before it would."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.models.heads.regression import LinearRegressionHead
    from lightning_pose_b200.utils.predictions import FramePredictor

    head = {"frame": lambda: HeatmapHead("resnet50", 64, 4), "regression": lambda: LinearRegressionHead(64, 8),
            "context": lambda: HeatmapMHCRNNHead("resnet50", 64, 4)}[kind]()
    return FramePredictor(head, 4, (64, 64), features_of=lambda x: x)


@pytest.mark.parametrize("kind", ["frame", "regression"])
def test_push_frame_refuses_heads_without_context(kind):
    fp = _predictor(kind)
    with pytest.raises(ValueError, match="predict_frame"):
        fp.push_frame(np.zeros((32, 48, 3), np.uint8))
    with pytest.raises(ValueError, match="predict_frame"):
        fp.reset_stream()


def test_push_frame_refuses_a_five_frame_stack():
    fp = _predictor("context")
    with pytest.raises(ValueError, match="predict_frame"):
        fp.push_frame(np.zeros((5, 32, 48, 3), np.uint8))


@pytest.mark.parametrize("frame,box", [
    (np.zeros((32, 48, 3), np.float32), None),     # not uint8
    (np.zeros((32, 48, 2), np.uint8), None),       # not RGB
    (np.zeros((0, 48, 3), np.uint8), None),        # empty
    (np.zeros((32, 48, 3), np.uint8), (-1, 0, 4, 4)),
    (np.zeros((32, 48, 3), np.uint8), (0, 0, 0, 4)),
    (np.zeros((32, 48, 3), np.uint8), (48, 0, 4, 4)),
], ids=["dtype", "channels", "empty", "origin", "size", "empty-crop"])
def test_push_frame_input_rules(frame, box):
    """The single-frame form's checks, before anything reaches the device."""
    with pytest.raises(ValueError):
        _predictor("context").push_frame(frame, bbox=box)
