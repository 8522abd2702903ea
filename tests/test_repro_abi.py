"""CPU: the fixed-order backward entries (lpb_convt_bwd_f32_ws, lpb_crnn_combine_bwd_ws) and their workspace queries
refuse malformed arguments with LPB_ERR_INVALID before they queue anything (the pointers below are fake, so a queued
kernel or a CUDA call would show as a different code)."""
import ctypes as C

import pytest

LPB_ERR_INVALID = -1
FAKE = 0x1000


def _lib():
    from lightning_pose_b200 import _lib

    return _lib.lib


def _convt_need(B=4, Cin=512, Hi=24, Wi=24, Cout=17):
    n = C.c_size_t(0)
    assert _lib().lpb_convt_bwd_f32_workspace_bytes(B, Cin, Hi, Wi, Cout, C.byref(n)) == 0
    return n.value


def _convt(B=4, Cin=512, Hi=24, Wi=24, shuffle=1, Cout=17, inp=FAKE, g=FAKE, w=FAKE, dw=FAKE, ws=FAKE, ws_bytes=None):
    ws_bytes = _convt_need(max(B, 0), max(Cin, 1), max(Hi, 1), max(Wi, 1), max(Cout, 1)) if ws_bytes is None else ws_bytes
    return _lib().lpb_convt_bwd_f32_ws(C.c_void_p(inp), C.c_void_p(g), B, Cin, Hi, Wi, shuffle, C.c_void_p(w), Cout, C.c_void_p(FAKE),
                                       C.c_void_p(dw), C.c_void_p(FAKE), C.c_void_p(ws), ws_bytes, None)


def test_convt_workspace_grows_with_the_partials():
    one = (512 * 17 * 9 + 17) * 4
    need = _convt_need()
    assert need % one == 0 and need // one >= 2  # several K-split slots at this size
    assert _convt_need(B=0) == 0
    n = C.c_size_t(0)
    assert _lib().lpb_convt_bwd_f32_workspace_bytes(4, 0, 24, 24, 17, C.byref(n)) == LPB_ERR_INVALID
    assert _lib().lpb_convt_bwd_f32_workspace_bytes(4, 512, 24, 24, 17, None) == LPB_ERR_INVALID


@pytest.mark.parametrize("bad", [
    {"ws": 0}, {"ws": FAKE + 2},                  # null / unaligned workspace
    {"ws_bytes": 0}, {"ws_bytes": "short"},       # too small a workspace
    {"B": -1}, {"Cin": 0}, {"Cout": 0}, {"Hi": 0}, {"Wi": 0},
    {"Hi": 23},                                   # shuffle needs even sizes
    {"inp": 0}, {"g": 0}, {"w": 0}, {"dw": 0},    # null pointers
], ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_convt_bwd_f32_ws_refuses(bad):
    if bad.get("ws_bytes") == "short":
        bad = {"ws_bytes": _convt_need() - 4}
    assert _convt(**bad) == LPB_ERR_INVALID, _lib().lpb_last_error()
    assert b"convt_bwd_f32" in _lib().lpb_last_error()


def _crnn_need(M=6, N=10, K=17, H=96, W=96):
    n = C.c_size_t(0)
    assert _lib().lpb_crnn_combine_bwd_workspace_bytes(M, N, K, H, W, C.byref(n)) == 0
    return n.value


def _crnn(M=6, N=10, K=17, H=96, W=96, wf=FAKE, idx=FAKE, g=FAKE, dwf=FAKE, ws=FAKE, ws_bytes=None):
    ws_bytes = _crnn_need() if ws_bytes is None else ws_bytes
    p = [C.c_void_p(FAKE)] * 4
    return _lib().lpb_crnn_combine_bwd_ws(C.c_void_p(wf), C.c_void_p(FAKE), C.c_void_p(idx), C.c_void_p(g), M, N, K, H, W, *p,
                                          C.c_void_p(dwf), C.c_void_p(FAKE), *p, C.c_void_p(ws), ws_bytes, None)


def test_crnn_workspace_holds_pairs_and_partials():
    # ints: start [N + 1], counts [N], pairs [5 M] (rounded to 4); floats: M * ceil(48 * 48 / 256) rows of 40 K
    assert _crnn_need() == (((2 * 10 + 1 + 30) + 3) // 4 * 4) * 4 + 6 * 9 * 40 * 17 * 4
    n = C.c_size_t(0)
    assert _lib().lpb_crnn_combine_bwd_workspace_bytes(6, 10, 17, 95, 96, C.byref(n)) == LPB_ERR_INVALID
    assert _lib().lpb_crnn_combine_bwd_workspace_bytes(6, 0, 17, 96, 96, C.byref(n)) == LPB_ERR_INVALID


@pytest.mark.parametrize("bad", [
    {"ws": 0}, {"ws": FAKE + 4},                  # null / unaligned (16 bytes) workspace
    {"ws_bytes": 0}, {"ws_bytes": "short"},       # too small a workspace
    {"M": -1}, {"N": 0}, {"K": 0}, {"H": 95}, {"W": 0},
    {"M": 4000},                                  # M * K >= 65536
    {"wf": 0}, {"idx": 0}, {"g": 0}, {"dwf": 0},  # null pointers
], ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_crnn_combine_bwd_ws_refuses(bad):
    if bad.get("ws_bytes") == "short":
        bad = {"ws_bytes": _crnn_need() - 4}
    assert _crnn(**bad) == LPB_ERR_INVALID, _lib().lpb_last_error()
    assert b"crnn_combine" in _lib().lpb_last_error()
