"""CPU: the multi-view ingest entry's argument checks, PredictionHandler's per-view split and BatchedPredictor's
multi-view input checks (the GPU side is tests/test_multiview_predict_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from lightning_pose_b200.utils.predictions import BatchedPredictor, PredictionHandler


def test_frames_normalize_views_validates_arguments_without_gpu():
    """lpb_frames_normalize_views refuses null pointers, a view count outside 1..16, non-positive sizes and a bad layout
    with an error code before anything is queued (the device pointers are fake)."""
    from lightning_pose_b200 import _lib

    L = _lib.lib
    fake = C.c_void_p(0x1000)
    m3, s3 = (C.c_float * 3)(0.485, 0.456, 0.406), (C.c_float * 3)(0.229, 0.224, 0.225)

    def call(ptrs, v, f=2, hs=(8,) * 17, ws=(8,) * 17, oh=8, ow=8, layout=0, mean=m3, out=fake):
        arr = (C.c_void_p * max(len(ptrs), 1))(*ptrs) if ptrs is not None else None
        return L.lpb_frames_normalize_views(arr, v, f, (C.c_int * 17)(*hs), (C.c_int * 17)(*ws), oh, ow, mean, s3, layout, 0, out, None)

    cases = [
        (lambda: call(None, 1), b"null pointer"),
        (lambda: call([0x1000, None], 2), b"null pointer"),
        (lambda: call([0x1000], 1, mean=None), b"null pointer"),
        (lambda: call([0x1000], 1, out=None), b"null pointer"),
        (lambda: call([0x1000], 0), b"view count 0 outside 1..16"),
        (lambda: call([0x1000] * 17, 17), b"view count 17 outside 1..16"),
        (lambda: call([0x1000] * 2, 2, hs=(8, 0) + (8,) * 15), b"bad shape/layout"),
        (lambda: call([0x1000], 1, ws=(-4,) * 17), b"bad shape/layout"),
        (lambda: call([0x1000], 1, oh=0), b"bad shape/layout"),
        (lambda: call([0x1000], 1, f=-1), b"bad shape/layout"),
        (lambda: call([0x1000], 1, layout=2), b"bad shape/layout"),
        (lambda: call([0x1000] * 16, 16, f=2**31 // 16), b"F * V must be below 2^31"),
    ]
    for i, (fn, msg) in enumerate(cases):
        assert fn() == -1, i
        assert L.lpb_last_error() == b"frames_normalize_views: " + msg, (i, L.lpb_last_error())
    # F = 0 is a no-op, and the single-view entry keeps its own name in its errors
    assert call([0x1000] * 3, 3, f=0) == 0
    assert L.lpb_frames_normalize(None, 1, 8, 8, 8, 8, m3, s3, 0, 0, fake, None) == -1
    assert L.lpb_last_error() == b"frames_normalize: null pointer"


def test_frames_normalize_views_refuses_bad_input():
    from lightning_pose_b200 import ops

    u8 = torch.zeros(2, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.frames_normalize_views([u8, u8], (8, 8))
    with pytest.raises(ValueError, match="1..16 views"):
        ops.frames_normalize_views([], (8, 8))
    with pytest.raises(ValueError, match="1..16 views"):
        ops.frames_normalize_views([u8] * 17, (8, 8))


def reference_split(stacked_preds, stacked_confs, keypoint_names, view_names, model_type):
    """Restatement of the reference's multi-view branch of PredictionHandler.__call__ (utils/predictions.py:296-315)."""
    import pandas as pd

    k = len(keypoint_names)
    out = {}
    for view_idx, view_name in enumerate(view_names):
        beg, end = view_idx * k, view_idx * k + k
        p, c = stacked_preds[:, beg * 2 : end * 2], stacked_confs[:, beg:end]
        arr = np.zeros((p.shape[0], 3 * k))
        arr[:, 0::3], arr[:, 1::3], arr[:, 2::3] = p[:, 0::2], p[:, 1::2], c
        cols = pd.MultiIndex.from_product([[f"{model_type}_tracker"], keypoint_names, ["x", "y", "likelihood"]],
                                          names=["scorer", "bodyparts", "coords"])
        out[view_name] = pd.DataFrame(arr, columns=cols)
    return out


def test_prediction_handler_splits_views_as_the_reference():
    rng = np.random.default_rng(4)
    names, views, n = ["nose", "ear", "tail"], ["top", "side", "bottom"], 7
    kp = torch.from_numpy(rng.normal(size=(n, 2 * 3 * 3)))
    cf = torch.from_numpy(rng.uniform(size=(n, 3 * 3)))
    h = PredictionHandler(names, n, model_type="heatmap_multiview_transformer", view_names=views)
    got = h([(kp[:4], cf[:4]), (kp[4:], cf[4:])], is_multiview_video=True)
    want = reference_split(kp.numpy(), cf.numpy(), names, views, "heatmap_multiview_transformer")
    assert list(got) == views
    for v in views:
        assert got[v].equals(want[v]), v
        assert got[v].columns[0] == ("heatmap_multiview_transformer_tracker", "nose", "x")
    # the device-table route: the (N, 3 V K) table that BatchedPredictor writes, columns of view v at [3 K v, 3 K (v + 1))
    table = np.concatenate([PredictionHandler.make_pred_arr_undo_resize(kp[:, 6 * v : 6 * v + 6].numpy(), cf[:, 3 * v : 3 * v + 3].numpy())
                            for v in range(3)], axis=1)
    from_table = h.dataframes(torch.from_numpy(table))
    assert list(from_table) == views and all(from_table[v].equals(want[v]) for v in views)
    # without the flag the call is the single-view form, unchanged
    assert PredictionHandler(names, n)([(kp[:, :6], cf[:, :3])]).equals(want["top"].rename(columns={"heatmap_multiview_transformer_tracker": "heatmap_tracker"}))
    with pytest.raises(ValueError, match="view_names"):
        PredictionHandler(names, n).dataframes(torch.from_numpy(table))
    with pytest.raises(ValueError, match="2 views of 9 expected"):
        PredictionHandler(names, n, view_names=["a", "b"]).dataframes(torch.from_numpy(table))


def multiview_predictor(v=3, **kw):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    head = HeatmapHead("vits_dino", 64, 5)
    return BatchedPredictor(head, 5, 20, 4, (32, 32), features_of=lambda x: x, use_graph=False, num_views=v, **kw)


def test_batched_predictor_multiview_refuses_bad_views():
    bp = multiview_predictor()
    assert bp.table.shape == (20, 3 * 3 * 5)
    u8 = lambda t, h, w: torch.zeros(t, h, w, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="expected 3 views; got 2"):
        bp.feed([u8(4, 16, 16), u8(4, 16, 16)])
    with pytest.raises(ValueError, match="same frame count"):
        bp.feed([u8(4, 16, 16), u8(3, 16, 16), u8(4, 16, 16)])
    with pytest.raises(ValueError, match="fixed-size"):
        bp.feed([u8(3, 16, 16)] * 3)
    with pytest.raises(ValueError, match="boxes from the views"):
        bp.feed([u8(4, 16, 16)] * 3, torch.zeros(4, 12))
    # the first chunk fixes the views' sizes (the ingest itself needs a GPU); a later chunk must match them
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        bp.feed([u8(4, 16, 16), u8(4, 24, 20), u8(4, 32, 32)])
    assert bp._view_bbox.tolist()[0] == [0, 0, 16, 16, 0, 0, 24, 20, 0, 0, 32, 32]
    with pytest.raises(ValueError, match="differ from the first chunk"):
        bp.feed([u8(4, 16, 16), u8(4, 20, 24), u8(4, 32, 32)])
    # frames / features input: (T, V, 3, h, w) or (T V, C, h', w'), boxes (T, 4V)
    with pytest.raises(ValueError, match=r"expected \(T, 3, 3, h, w\)"):
        bp.feed(torch.zeros(4, 2, 3, 32, 32))
    with pytest.raises(ValueError, match="fixed-size"):
        bp.feed(torch.zeros(8, 64, 2, 2))
    with pytest.raises(ValueError, match=r"bbox must be \(4, 12\)"):
        bp.feed(torch.zeros(12, 64, 2, 2), torch.zeros(4, 4))
    with pytest.raises(ValueError, match="need features_of"):
        BatchedPredictor(bp.head, 5, 20, 4, (32, 32), use_graph=False, num_views=3).feed([u8(4, 16, 16)] * 3)


def test_multiview_refusals_stay():
    """Context heads and crop mode still refuse several views."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    with pytest.raises(ValueError, match="context prediction is not supported for multiview models"):
        BatchedPredictor(HeatmapMHCRNNHead("vits_dino", 64, 5), 5, 20, 4, (32, 32), num_views=2)
    with pytest.raises(ValueError, match="bbox cropping is not supported for multiview models"):
        multiview_predictor(v=2, bboxes=torch.zeros(20, 4), frame_hw=(64, 64))
