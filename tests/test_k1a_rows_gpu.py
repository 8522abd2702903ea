"""k1a (head_bf16.cu: PixelShuffle + the first transposed convolution of a two-deconv head) works on (frame, band) items
that stage only their band's feature rows, and each item writes its own rows of the saved operand copy.  The test runs
the fast path at config 2 and at shapes on its edges (one, two and three bands, equal and unequal, W = 4 / 6 / 7 / 24 /
28) with a batch of 2S + 7 frames, so every CTA loops over several items, and checks:
  * the saved copy (filled with 0xFF bytes before the call) byte for byte against a torch construction of the padded row
    layout: every pad row is written by the kernel;
  * the mid activations in the workspace (also filled with 0xFF bytes) against the float64 reference at the bf16
    tolerance, and their pad rows and zero column as all-zero bits;
  * that a frame alone and the same frame inside the batch give identical bits."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import scale_oracle as S
from head_support import fwd_layout, gen, row_layout, softmax_split

pytestmark = pytest.mark.gpu

K = 17

# (C, H, W) -> bands as (first feature row, rows): config 2 (0,6 6,6); W = 4 (0,16 16,16 32,16); W = 6, last band shorter
# (0,12 12,12 24,8); one band in the training form with W = 6 and W = 7 (the frame's bottom edge is the only halo); H * W =
# 192 with a short last band (0,6 6,6 12,4; two channel stages); W = 24 (0,3 3,3 6,2); the widest W k1a takes, 28 (three
# bands of 2).  Band starts fall where the TMA box starts on a 16-byte boundary (head_bf16.cu make_k1a_geom).  Several of
# these shapes took the banded generic path before k1a staged bands.
SHAPES = {
    "cfg2": (2048, 12, 12), "48x4": (128, 48, 4), "32x6": (128, 32, 6), "8x6": (128, 8, 6), "8x7": (128, 8, 7),
    "16x12": (256, 16, 12), "8x24": (128, 8, 24), "6x28": (128, 6, 28),
}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


def head_call(lib, feats, w1, b1, w2, b2):
    """lpb_head_fwd_bf16 in the training form; returns (saved copy, mid activations) as int16 bit patterns."""
    b, c, h, w = feats.shape
    size = ctypes.c_size_t(0)
    assert lib.lpb_head_bf16_workspace_bytes(b, c, h, w, K, K, ctypes.byref(size)) == 0
    ws = torch.full((size.value,), 0xFF, dtype=torch.uint8, device=feats.device)
    assert lib.lpb_head_bf16_saved_bytes(b, c, h, w, ctypes.byref(size)) == 0
    xs = torch.full((size.value,), 0xFF, dtype=torch.uint8, device=feats.device)
    out = torch.empty(b, K, 8 * h, 8 * w, device=feats.device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(feats.device).cuda_stream)
    rc = lib.lpb_head_fwd_bf16(ctypes.c_void_p(feats.data_ptr()), b, c, h, w, ctypes.c_void_p(w1.data_ptr()), ctypes.c_void_p(b1.data_ptr()), K,
                               ctypes.c_void_p(w2.data_ptr()), ctypes.c_void_p(b2.data_ptr()), K, 1, ctypes.c_void_p(out.data_ptr()),
                               ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(ws.data_ptr()), stream)
    assert rc == 0, lib.lpb_last_error()
    torch.cuda.synchronize(feats.device)
    lay = fwd_layout(b, c, h, w, K, K)
    mid = ws[lay.mid_at:lay.mid_at + b * 4 * lay.nst2 * lay.mid_rows * 16]
    return xs.view(torch.int16), mid.view(torch.int16)


def saved_copy_ref(feats):
    """[B][C/32][rows][8] bf16: PixelShuffle of the features in the padded row layout (zero column, zero lead / trail rows)."""
    b, c, h, w = feats.shape
    hi, wi = 2 * h, 2 * w
    pp, lead, rows = row_layout(hi, wi)
    x = F.pixel_shuffle(feats, 2).reshape(b, c // 32, 8, hi, wi).permute(0, 1, 3, 4, 2)
    x = F.pad(x, (0, 0, 0, 1)).reshape(b, c // 32, hi * pp, 8)  # the zero column of every image row
    out = torch.zeros(b, c // 32, rows, 8, dtype=feats.dtype, device=feats.device)
    out[:, :, lead:lead + hi * pp] = x
    return out.view(torch.int16).flatten()


def mid_planes(mid, b, h, w):
    """the mid activations' [B][4][rows][8] row layout -> (B, 32, 4H, 4W) float64"""
    hi, wi = 4 * h, 4 * w
    pp, lead, rows = row_layout(hi, wi)
    m = mid.view(torch.bfloat16).reshape(b, 4, rows, 8)[:, :, lead:lead + hi * pp].reshape(b, 4, hi, pp, 8)[:, :, :, :wi]
    return m.permute(0, 1, 4, 2, 3).reshape(b, 32, hi, wi).to(torch.float64)


def mid_pads_zero(mid, b, h, w):
    """whether the mid activations' lead / trail rows and zero column (layer 2's halo) hold all-zero bits"""
    hi, wi = 4 * h, 4 * w
    pp, lead, rows = row_layout(hi, wi)
    m = mid.reshape(b, 4, rows, 8)
    zero_col = m[:, :, lead:lead + hi * pp].reshape(b, 4, hi, pp, 8)[:, :, :, wi:]
    return not (m[:, :, :lead].any() or m[:, :, lead + hi * pp:].any() or zero_col.any())


@pytest.mark.parametrize("shape", list(SHAPES))
def test_k1a_bands(lib, dev, shape):
    c, h, w = SHAPES[shape]
    plan = ctypes.c_int(-1)
    assert lib.lpb_head_bf16_plan(c, h, w, K, K, ctypes.byref(plan)) == 0 and plan.value == 1  # the fast path: k1a
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    b = 2 * sms + 7
    g = gen(11)
    feats = (torch.randn(b, c, h, w, device=dev, generator=g) * 0.5).bfloat16()
    w1 = torch.randn(c // 4, K, 3, 3, device=dev, generator=g) * (2.0 / (c // 4)) ** 0.5
    b1 = torch.rand(K, device=dev, generator=g) - 0.5
    w2 = torch.randn(K, K, 3, 3, device=dev, generator=g) * 0.3
    b2 = torch.rand(K, device=dev, generator=g) - 0.5
    with softmax_split(lib, 0):
        xs, mid = head_call(lib, feats, w1, b1, w2, b2)
        assert torch.equal(xs, saved_copy_ref(feats))

        assert mid_pads_zero(mid, b, h, w)
        got = mid_planes(mid, b, h, w)
        assert bool((got[:, K] == 1).all()) and bool((got[:, K + 1:] == 0).all())  # the constant-one channel, zero padding
        for i in range(0, b, 64):
            with torch.no_grad():
                ref = S.head_ref(feats[i:i + 64], [w1], [b1], softmax=False)  # layer 1 alone: the mid activations
            scale = float(ref.abs().max())
            err = (got[i:i + 64, :K] - ref).abs()
            assert bool((err <= 1e-2 * scale + 1e-2 * ref.abs()).all()), float(err.max())

        # a frame alone: the same bits as inside the batch (first and last frame: first and last band's CTA positions)
        _, _, rows_xs = row_layout(2 * h, 2 * w)
        _, _, rows_mid = row_layout(4 * h, 4 * w)
        nxs, nmid = c // 32 * rows_xs * 8, 4 * rows_mid * 8
        for j in (0, b - 1):
            xs1, mid1 = head_call(lib, feats[j:j + 1].contiguous(), w1, b1, w2, b2)
            assert torch.equal(xs1, xs[j * nxs:(j + 1) * nxs])
            assert torch.equal(mid1, mid[j * nmid:(j + 1) * nmid])
