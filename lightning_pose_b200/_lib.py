"""ctypes binding of ``liblpb200.so`` (the C-ABI declared in ``include/lpb200.h``).

The library is hand-written sm_90a CUDA built in-tree by ``build.sh`` /
``__graft_entry__.build()``.  There is no CPU implementation behind these symbols: if the shared
object is missing, importing this module raises, and every wrapper in ``ops.py`` refuses non-CUDA
tensors.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblpb200.so")


class PcaDesc(C.Structure):
    """mirror of ``lpb_pca_desc`` (include/lpb200.h)."""

    _fields_ = [
        ("kp_index", C.c_void_p),
        ("n_sel", C.c_int32),
        ("n_views", C.c_int32),
        ("centering", C.c_int32),
        ("n_components", C.c_int32),
        ("mean", C.c_void_p),
        ("kept", C.c_void_p),
        ("epsilon", C.c_float),
    ]


class MseTargets(C.Structure):
    """mirror of ``lpb_mse_targets`` (include/lpb200.h)."""

    _fields_ = [
        ("keypoints", C.c_void_p),
        ("visibility", C.c_void_p),
        ("img_height", C.c_float),
        ("img_width", C.c_float),
        ("sigma", C.c_float),
        ("fwd_out", C.c_void_p),
        ("grad_out", C.c_void_p),
    ]


class Head3Sizes(C.Structure):
    """mirror of ``lpb_head3_sizes`` (include/lpb200.h)."""

    _fields_ = [
        ("plan", C.c_int),
        ("fwd_workspace", C.c_size_t),
        ("saved", C.c_size_t),
        ("bwd_workspace", C.c_size_t),
        ("bwd_workspace_targets", C.c_size_t),
    ]


_P, _I, _L, _F, _Z = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t

# symbol -> (restype, argtypes); this table is also what tests/test_abi.py checks against the header
SIGNATURES = {
    "lpb_version": (C.c_int, []),
    "lpb_last_error": (C.c_char_p, []),
    "lpb_build_arch": (C.c_char_p, []),
    "lpb_set_tuning": (C.c_int, [_I, _I]),
    "lpb_get_tuning": (C.c_int, [_I]),
    "lpb_decode_prepare": (C.c_int, [_I, _I, _I]),
    "lpb_decode_fwd_workspace_bytes": (C.c_int, [_L, C.POINTER(_Z)]),
    "lpb_decode_fwd": (C.c_int, [_P, _L, _I, _I, _I, _F, _P, _P, _P, _P, _P]),
    "lpb_decode_fwd_banded": (C.c_int, [_P, _L, _I, _I, _I, _F, _P, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_decode_bwd": (C.c_int, [_P, _P, _P, _L, _I, _I, _I, _F, _P, _P]),
    "lpb_decode_bwd_windows": (C.c_int, [_P, _P, _P, _L, _I, _I, _I, _F, _P, _P, _P, _P, _P]),
    "lpb_upsample2x": (C.c_int, [_P, _L, _I, _I, _P, _P]),
    "lpb_generate_heatmaps": (C.c_int, [_P, _P, _L, _F, _F, _I, _I, _F, _P, _P]),
    "lpb_keypoints_mask_oob": (C.c_int, [_P, _L, _F, _F, _P, _P]),
    "lpb_generate_heatmaps_bwd": (C.c_int, [_P, _P, _P, _L, _F, _F, _I, _I, _F, _P, _P]),
    "lpb_evaluate_heatmaps_at_location": (C.c_int, [_P, _P, _L, _I, _I, _I, _P, _P]),
    "lpb_convt_fwd_f32": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P]),
    "lpb_plane_softmax_f32": (C.c_int, [_P, _L, _I, _P]),
    "lpb_convt_bwd_f32_workspace_bytes": (C.c_int, [_I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_convt_bwd_f32_ws": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _P, _I, _P, _P, _P, _P, _Z, _P]),
    "lpb_head_bf16_plan": (C.c_int, [_I, _I, _I, _I, _I, C.POINTER(_I)]),
    "lpb_head_bf16_workspace_bytes": (C.c_int, [_I, _I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_head_bf16_saved_bytes": (C.c_int, [_I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_head_fwd_bf16": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P]),
    "lpb_head_fwd_f16": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P]),
    "lpb_head_bwd_bf16_workspace_bytes": (C.c_int, [_I, _I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_head_bwd_bf16": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P]),
    "lpb_head_bf16_plan_layout": (C.c_int, [_I, _I, _I, _I, _I, _I, C.POINTER(_I)]),
    "lpb_head_fwd_bf16_layout": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    "lpb_head_fwd_f16_layout": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    "lpb_head_band_max_dims": (C.c_int, [_I, _I, C.POINTER(_I), C.POINTER(_I)]),
    "lpb_head_fwd_bf16_band_max": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_head_fwd_f16_band_max": (C.c_int, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_head_bwd_bf16_workspace_bytes_layout": (C.c_int, [_I, _I, _I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_head_bwd_bf16_layout": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _I, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "lpb_head_bwd_bf16_workspace_bytes_targets": (C.c_int, [_I, _I, _I, _I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_head_bwd_bf16_targets": (C.c_int, [_P, C.POINTER(MseTargets), _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _I, _P, _I, _I, _P, _P, _P,
                                            _P, _P, _P, _P]),
    "lpb_head3_query": (C.c_int, [_I, _I, _I, _I, _I, _I, _I, _I, _I, C.POINTER(Head3Sizes)]),
    "lpb_head3_fwd": (C.c_int, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_head3_bwd": (C.c_int, [_P, C.POINTER(MseTargets), _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _I, _P, _I, _P, _I, _P, _P, _P,
                                _P, _P, _P, _P, _P, _P]),
    "lpb_remap_keypoints": (C.c_int, [_P, _L, _I, _P, _I, _I, _P, _L, _F, _F, _P, _P]),
    "lpb_remap_keypoints_bwd": (C.c_int, [_P, _L, _I, _P, _I, _I, _P, _L, _F, _F, _P, _P]),
    "lpb_crnn_prepare": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _P, _P]),
    "lpb_crnn_prepare_bwd": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_crnn_combine_fwd": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "lpb_crnn_combine_bwd_workspace_bytes": (C.c_int, [_I, _I, _I, _I, _I, C.POINTER(_Z)]),
    "lpb_crnn_combine_bwd_ws": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    "lpb_context_gather": (C.c_int, [_P, _L, _L, _I, _P, _P]),
    "lpb_context_gather_bwd": (C.c_int, [_P, _L, _L, _I, _I, _P, _P]),
    "lpb_frames_normalize": (C.c_int, [_P, _I, _I, _I, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I, _P, _P]),
    "lpb_frames_normalize_views": (C.c_int, [C.POINTER(_P), _I, _I, C.POINTER(_I), C.POINTER(_I), _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I, _P, _P]),
    "lpb_frames_normalize_ragged": (C.c_int, [_P, _L, _I, _P, _P, _P, _I, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I,
                                              _P, _P, _P]),
    "lpb_frames_crop_normalize_ragged": (C.c_int, [_P, _L, _I, _P, _P, _P, _I, _P, _L, _I, _I, C.POINTER(C.c_float),
                                                   C.POINTER(C.c_float), _I, _I, _P, _P, _P]),
    "lpb_frames_augment_normalize": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I, _P, _P, _P]),
    "lpb_frames_crop_resize_cv2": (C.c_int, [_P, _I, _I, _I, _P, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I, _P, _P, _P]),
    "lpb_patch_mask_select": (C.c_int, [_P, _I, _I, _I, _I, _L, _L, _L, C.c_double, C.c_double, _P, _P]),
    "lpb_patch_mask_apply": (C.c_int, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "lpb_frames_crop_normalize":(C.c_int, [_P, _I, _I, _I, _I, _P, _L, _P, _L, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _I, _I, _P, _P, _P]),
    "lpb_bboxes_from_keypoints": (C.c_int, [_P, _L, _I, _L, _I, C.POINTER(C.c_int32), _I, C.c_double, _I, _I, _P, _P]),
    "lpb_bboxes_rolling_median": (C.c_int, [_P, _L, _I, _P, _P]),
    "lpb_pack_predictions": (C.c_int, [_P, _P, _I, _I, _P, _L, _P, _L, _P]),
    "lpb_pack_context_predictions": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _F, _F, _P, _L, _P, _L, _L, _P]),
    "lpb_pack_context_predictions_segments": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _F, _F, _P, _L, _P, _P, _P, _I, _L, _P, _P]),
    "lpb_context_ring_push": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "lpb_context_ring_select": (C.c_int, [_P, _P, _P, _P, _P, _I, _F, _F, _P, _P, _P]),
    "lpb_adam_step": (C.c_int, [_I, _P, _P, _P, _P, _P, _P, _P, _F, _P, C.c_double, C.c_double, _F, _F, _I, _P]),
    "lpb_plane_softmax_bwd": (C.c_int, [_P, _P, _L, _I, _P, _P]),
    "lpb_heatmap_loss_fwd": (C.c_int, [_P, _P, _L, _I, _I, _I, _P, _P, _P]),
    "lpb_heatmap_loss_bwd": (C.c_int, [_P, _P, _L, _I, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_heatmap_mse_from_keypoints_fwd": (C.c_int, [_P, _P, _P, _L, _F, _F, _I, _I, _F, _P, _P, _P]),
    "lpb_heatmap_mse_from_keypoints_bwd": (C.c_int, [_P, _P, _P, _L, _F, _F, _I, _I, _F, _P, _P, _P, _P]),
    "lpb_heatmap_loss_from_keypoints_fwd": (C.c_int, [_P, _P, _P, _L, _F, _F, _I, _I, _F, _I, _P, _P, _P]),
    "lpb_heatmap_loss_from_keypoints_bwd": (C.c_int, [_P, _P, _P, _L, _F, _F, _I, _I, _F, _I, _P, _P, _P, _P]),
    "lpb_temporal_heatmap_loss_fwd": (C.c_int, [_P, _P, _L, _I, _I, _I, _I, _P, _F, _P, _P, _P]),
    "lpb_temporal_heatmap_loss_bwd": (C.c_int, [_P, _P, _P, _L, _I, _I, _I, _I, _P, _F, _P, _P, _P]),
    "lpb_unsup_losses_fwd": (C.c_int, [_P, _P, _L, _I, _I, _P, _F, _I, C.POINTER(PcaDesc), C.POINTER(PcaDesc), _P, _P]),
    "lpb_unsup_losses_bwd": (C.c_int, [_P, _P, _L, _I, _I, _P, _F, _I, C.POINTER(PcaDesc), C.POINTER(PcaDesc), _P, _P, _P]),
    "lpb_triangulate_pairs_fwd": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "lpb_triangulate_pairs_bwd": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "lpb_project_points_fwd": (C.c_int, [_P, _I, _P, _P, _P, _P, _F, _F, _I, _I, _I, _I, _P, _P]),
    "lpb_project_points_bwd": (C.c_int, [_P, _I, _P, _P, _P, _P, _F, _F, _P, _I, _I, _I, _I, _P, _P]),
    "lpb_frame_to_model": (C.c_int, [_P, _I, _I, _I, _P, _F, _F, _I, _P, _P]),
    "lpb_pairwise_projections_loss_fwd": (C.c_int, [_P, _P, _I, _I, _I, _P, _P]),
    "lpb_pairwise_projections_loss_bwd": (C.c_int, [_P, _P, _I, _I, _I, _P, _P, _P, _P]),
    "lpb_regression_head_fwd": (C.c_int, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _P]),
    "lpb_regression_head_bwd": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "lpb_regression_losses_fwd": (C.c_int, [_P, _P, _L, _P, _P]),
    "lpb_regression_losses_bwd": (C.c_int, [_P, _P, _L, _P, _P, _P, _P]),
}


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build the CUDA library first (./build.sh or "
            "`python -c 'import __graft_entry__ as g; g.build()'`). lightning_pose_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()

# LPB_TUNE="key=value,..." sets tuning switches (include/lpb200.h LPB_TUNE_*): a profiling / bring-up aid
for _kv in filter(None, os.environ.get("LPB_TUNE", "").split(",")):
    _k, _v = _kv.split("=")
    if lib.lpb_set_tuning(int(_k), int(_v)) != 0:
        raise ValueError(f"LPB_TUNE: unknown key {_k}")


class LpbError(RuntimeError):
    pass


def check(rc: int) -> None:
    if rc != 0:
        msg = lib.lpb_last_error()
        raise LpbError(f"lpb200 error {rc}: {msg.decode() if msg else '?'}")
