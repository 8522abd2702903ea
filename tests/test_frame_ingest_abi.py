"""CPU: lpb_frames_crop_resize_cv2 refuses malformed arguments with LPB_ERR_INVALID before it queues anything (the
pointers below are fake, so a queued kernel or a CUDA call would show as a different code)."""
import ctypes as C

import pytest

LPB_ERR_INVALID = -1


def _call(frames=0x1000, F=1, H=8, W=8, box=None, out_h=4, out_w=4, std=(0.229, 0.224, 0.225), layout=0, fmt=0, out=0x1000,
          bbox_out=0x1000):
    from lightning_pose_b200 import _lib

    m3, s3 = (C.c_float * 3)(0.485, 0.456, 0.406), (C.c_float * 3)(*std)
    return _lib.lib.lpb_frames_crop_resize_cv2(C.c_void_p(frames), F, H, W, C.c_void_p(box), out_h, out_w, m3, s3, layout, fmt,
                                               C.c_void_p(out), C.c_void_p(bbox_out), None)


@pytest.mark.parametrize("bad", [
    {"fmt": 3}, {"fmt": -1},                      # output formats
    {"layout": 2}, {"layout": -1},                # layouts
    {"F": 0}, {"F": -1},                          # frame counts
    {"H": 0}, {"W": 0}, {"out_h": 0}, {"out_w": -3},
    {"frames": 0}, {"out": 0}, {"bbox_out": 0},   # null pointers
    {"std": (0.229, 0.0, 0.225)},                 # a zero std
], ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_crop_resize_cv2_refuses(bad):
    from lightning_pose_b200 import _lib

    assert _call(**bad) == LPB_ERR_INVALID, _lib.lib.lpb_last_error()
    assert b"frames_crop_resize_cv2" in _lib.lib.lpb_last_error()
