"""CPU: the three-deconv head's entries (lpb_head3_query / _fwd / _bwd) state which heads they serve, size their buffers and
refuse bad arguments without a GPU, and ``ops.head3_supported`` asks the same question of the library."""
import ctypes

import pytest

LAYOUTS = (0, 1)  # LPB_FEATURES_NCHW, LPB_FEATURES_NHWC
ERR_INVALID, ERR_UNSUPPORTED = -1, -3
HEAD_CLS = 20
STAGE_BYTES = 4 * 4 * 80 * 16


@pytest.fixture(scope="module")
def lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


def query(lib, b, c, h, w, ch, layout=0, train=True):
    from lightning_pose_b200._lib import Head3Sizes

    sizes = Head3Sizes()
    rc = lib.lpb_head3_query(b, c, h, w, *ch, layout, int(train), ctypes.byref(sizes))
    return rc, sizes


def row_rows(hi, wi):
    pp = wi + 1
    return (hi * pp + 2 * (pp + 1) + 7) & ~7


def bands(hi, wi):
    r = max(1, min(256 // (wi + 1), hi))
    return -(-hi // r)


COVERED = [(c, h, w, ch) for c in (512, 2048) for (h, w) in ((12, 12), (8, 8), (4, 4), (16, 16), (8, 12), (2, 4), (64, 16))
           for ch in ((17, 17, 17), (8, 8, 17), (19, 19, 20), (17, 17, 5), (1, 1, 1))]


@pytest.mark.parametrize("c,h,w,ch", COVERED)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_covered_shapes_train_and_predict(lib, c, h, w, ch, layout):
    for train in (True, False):
        rc, s = query(lib, 3, c, h, w, ch, layout, train)
        assert rc == 0, lib.lpb_last_error()
        # forward workspace: the three packs, mid (4H x 4W) and mid2 (8H x 8W) with one K stage each, the last layer's
        # split-softmax statistics
        mid = 3 * 4 * row_rows(4 * h, 4 * w) * 16
        mid2 = 3 * 4 * row_rows(8 * h, 8 * w) * 16
        part = 3 * bands(8 * h, 8 * w) * HEAD_CLS * 2 * 4
        assert s.fwd_workspace == (c // 128 + 2) * STAGE_BYTES + mid + mid2 + ((part + 255) & ~255)
        assert s.saved == 3 * (c // 32) * row_rows(2 * h, 2 * w) * 16
        plan = ctypes.c_int(-1)
        assert lib.lpb_head_bf16_plan_layout(c, h, w, ch[0], ch[1], layout, ctypes.byref(plan)) == 0
        assert s.plan == plan.value
        if layout == 1:
            assert s.plan == 0
        if train:
            # at least the three gradient row buffers G1, G2, G3 of 10 K-chunks each, and more with keypoint targets
            g = 3 * 10 * (row_rows(2 * h, 2 * w) + row_rows(4 * h, 4 * w) + row_rows(8 * h, 8 * w)) * 16
            assert s.bwd_workspace >= g
            assert s.bwd_workspace_targets > s.bwd_workspace
        else:
            assert s.bwd_workspace == 0 and s.bwd_workspace_targets == 0


def test_two_deconv_query_is_unchanged(lib):
    """The one- and two-deconv query still refuses three channels' worth of head (it has no third layer)."""
    from lightning_pose_b200 import ops

    assert not ops.head_bf16_supported((4, 2048, 12, 12), [17, 17, 17], train=True)
    assert not ops.head_bf16_supported((4, 2048, 12, 12), [17, 17, 17], train=False)


REFUSED = [  # (C, H, W, channels, train, reason)
    (2048, 12, 12, (20, 17, 17), True, "channel"),    # no room for the ones channel in mid
    (2048, 12, 12, (17, 20, 17), False, "channel"),   # ... in mid2
    (2048, 12, 12, (17, 17, 21), True, "channel"),    # wide last layer
    (2048, 12, 12, (51, 51, 51), False, "channel"),   # wide head
    (2048, 12, 24, (17, 17, 17), False, "width"),
    (2048, 12, 32, (17, 17, 17), True, "width"),
    (2048, 12, 6, (17, 17, 17), False, "width"),
    (2048, 12, 2, (17, 17, 17), False, "width"),
    (2048, 7, 8, (17, 17, 17), True, "even"),         # odd H trains nowhere
    (2048, 3, 4, (17, 17, 17), False, "multiple of 8"),
]


@pytest.mark.parametrize("c,h,w,ch,train,why", REFUSED)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_refused_shapes(lib, c, h, w, ch, train, why, layout):
    rc, s = query(lib, 2, c, h, w, ch, layout, train)
    assert rc == ERR_UNSUPPORTED and why.encode() in lib.lpb_last_error()
    assert (s.plan, s.fwd_workspace, s.saved, s.bwd_workspace, s.bwd_workspace_targets) == (0, 0, 0, 0, 0)


def test_odd_height_predicts(lib):
    rc, _ = query(lib, 2, 2048, 7, 8, (17, 17, 17), 0, train=False)
    assert rc == 0


def test_bad_arguments_are_invalid(lib):
    from lightning_pose_b200._lib import Head3Sizes

    sizes = Head3Sizes()
    assert lib.lpb_head3_query(2, 2048, 12, 12, 17, 17, 17, 0, 1, None) == ERR_INVALID
    assert lib.lpb_head3_query(2, 2048, 12, 12, 17, 17, 17, 2, 1, ctypes.byref(sizes)) == ERR_INVALID
    assert lib.lpb_head3_query(2, 2000, 12, 12, 17, 17, 17, 0, 1, ctypes.byref(sizes)) == ERR_INVALID
    assert lib.lpb_head3_query(2, 2048, 12, 12, 17, 0, 17, 0, 1, ctypes.byref(sizes)) == ERR_INVALID


def _fwd(lib, features=16, out=16, ws=16, xs=16, band_max=None, operand=1, softmax=1, w3=16):
    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731  (addresses are never dereferenced: refused first)
    return lib.lpb_head3_fwd(p(features), operand, 0, 2, 2048, 12, 12, p(16), p(16), 17, p(16), p(16), 17, p(w3), p(16), 17, softmax,
                             p(out), p(band_max), p(xs), p(ws), None)


def test_forward_refuses_null_and_misaligned_buffers(lib):
    for kw, msg in [({"features": None}, b"null pointer"), ({"out": None}, b"null pointer"), ({"ws": None}, b"null pointer"),
                    ({"w3": None}, b"w3"), ({"features": 8}, b"features must be 16-byte aligned"),
                    ({"ws": 24}, b"workspace must be 16-byte aligned"), ({"xs": 8}, b"saved_xs must be 16-byte aligned"),
                    ({"out": 4}, b"out must be 8-byte aligned"), ({"band_max": 2}, b"band_max must be 4-byte aligned"),
                    ({"operand": 0}, b"operand type"), ({"band_max": 16, "softmax": 0}, b"final_softmax")]:
        assert _fwd(lib, **kw) == ERR_INVALID, kw
        assert msg in lib.lpb_last_error(), (kw, lib.lpb_last_error())
    assert lib.lpb_head3_fwd(ctypes.c_void_p(16), 1, 0, 2, 2048, 12, 24, *[None] * 2, 17, *[None] * 2, 17, *[None] * 2, 17, 1,
                             *[None] * 5) == ERR_UNSUPPORTED


def _bwd(lib, **over):
    a = dict(g_out=16, probs=16, saved=16, fws=16, dfeat=16, ws=16, w3=16, dw3=16, db3=16, w1=16, dw1=16)
    a.update(over)
    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731
    return lib.lpb_head3_bwd(p(a["g_out"]), None, p(a["probs"]), None, None, None, p(a["saved"]), p(a["fws"]), 0, 2, 2048, 12, 12,
                             p(a["w1"]), 17, p(16), 17, p(a["w3"]), 17, p(a["dfeat"]), p(a["dw1"]), p(16), p(16), p(16), p(a["dw3"]),
                             p(a["db3"]), p(a["ws"]), None)


def test_backward_refuses_null_and_misaligned_buffers(lib):
    for kw, msg in [({"w3": None}, b"null pointer"), ({"dw3": None}, b"null pointer"), ({"db3": None}, b"null pointer"),
                    ({"saved": None}, b"null pointer"), ({"ws": None}, b"null pointer"), ({"w1": None}, b"null pointer"),
                    ({"g_out": None}, b"neither a dense gradient"), ({"g_out": 8}, b"g_out must be 16-byte aligned"),
                    ({"dfeat": 24}, b"dfeat must be 16-byte aligned"), ({"fws": 4}, b"fwd_workspace must be 16-byte aligned")]:
        assert _bwd(lib, **kw) == ERR_INVALID, kw
        assert msg in lib.lpb_last_error(), (kw, lib.lpb_last_error())


def test_ops_query_agrees_with_the_library(lib):
    from lightning_pose_b200 import ops

    for c, h, w, ch in COVERED[::3] + [(r[0], r[1], r[2], r[3]) for r in REFUSED]:
        for layout in LAYOUTS:
            for train in (True, False):
                assert ops.head3_supported((2, c, h, w), list(ch), train, layout) == (query(lib, 2, c, h, w, ch, layout, train)[0] == 0)
    assert not ops.head3_supported((2, 2048, 12, 12), [17, 17], True)
