"""Argument refusals of the band-maxima entries (lpb_decode_fwd_banded, lpb_head_band_max_dims, the head forwards
that write the maxima).  No GPU: every refusal happens before anything is launched."""
import ctypes

from lightning_pose_b200 import _lib

L = _lib.lib
FAKE = ctypes.c_void_p(0x10000)  # never dereferenced: the call is refused first


def banded(band_max, rows, nbands, h=96, w=96, ws=FAKE):
    return L.lpb_decode_fwd_banded(FAKE, 17, h, w, 2, 1000.0, band_max, rows, nbands, FAKE, FAKE, FAKE, ws, None)


def test_band_max_dims_follow_the_softmax_bands():
    r, n = ctypes.c_int(0), ctypes.c_int(0)
    for (h, w), want in {(96, 96): (5, 10), (64, 64): (7, 5), (128, 128): (3, 22), (64, 80): (6, 6), (48, 64): (7, 4), (24, 32): (12, 1)}.items():
        assert L.lpb_head_band_max_dims(h, w, ctypes.byref(r), ctypes.byref(n)) == 0
        assert (r.value, n.value) == want, (h, w)
    assert L.lpb_head_band_max_dims(95, 96, ctypes.byref(r), ctypes.byref(n)) == -1
    assert L.lpb_head_band_max_dims(96, 96, None, ctypes.byref(n)) == -1


def test_banded_decode_refusals():
    assert banded(None, 5, 10) == -1 and b"null band_max" in L.lpb_last_error()
    assert banded(ctypes.c_void_p(0x10002), 5, 10) == -1 and b"aligned" in L.lpb_last_error()
    for rows, nbands in ((5, 9), (5, 11), (4, 10), (0, 10), (48, 2)):
        assert banded(FAKE, rows, nbands) == -1 and b"do not cut" in L.lpb_last_error(), (rows, nbands)
    assert banded(FAKE, 5, 10, h=95) == -1 and b"do not cut" in L.lpb_last_error()
    assert banded(FAKE, 5, -1) == -1
    assert banded(FAKE, 5, 10, ws=ctypes.c_void_p(0x10002)) == -1 and b"workspace" in L.lpb_last_error()


def test_head_forward_band_max_refusals():
    for entry in (L.lpb_head_fwd_bf16_band_max, L.lpb_head_fwd_f16_band_max):
        args = [FAKE, 2, 2048, 12, 12, FAKE, FAKE, 17, FAKE, FAKE, 17, 0, FAKE]
        assert entry(*args, None, FAKE, FAKE, None) == -1 and b"null band_max" in L.lpb_last_error()
        assert entry(*args, ctypes.c_void_p(0x10002), FAKE, FAKE, None) == -1 and b"band_max must be 4-byte aligned" in L.lpb_last_error()
