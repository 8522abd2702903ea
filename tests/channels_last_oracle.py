"""numpy restatement of the PixelShuffle(2) fold into the padded row layout.  TEST INFRASTRUCTURE ONLY.

The 16-bit head's first GEMM reads X[b][kchunk][row][8]: row = lead + m * (Wi + 1) + n over the shuffled image
(Hi, Wi) = (2H, 2W), eight shuffled channels per K-chunk, zero pads.  Shuffled channel s at sub-pixel (2i + di, 2j + dj)
is source channel 4 s + q, q = 2 di + dj, at feature pixel (i, j); so a K-chunk's row entry for sub-pixel q holds source
channels q, 4 + q, ..., 28 + q of the chunk's 32.  Both packers below produce the buffer the shuffle kernels must write,
one from NCHW features and one from channels-last features."""
import numpy as np


def row_layout(hi, wi):
    pp = wi + 1
    lead = pp + 1
    return pp, lead, (hi * pp + 2 * lead + 7) & ~7


def pack_rows_nchw(feat):
    """feat (B, C, H, W) uint16 -> rows (B, C / 32, rows, 8), by the definition of PixelShuffle(2)."""
    b, c, h, w = feat.shape
    shuffled = feat.reshape(b, c // 4, 2, 2, h, w).transpose(0, 1, 4, 2, 5, 3).reshape(b, c // 4, 2 * h, 2 * w)
    pp, lead, rows = row_layout(2 * h, 2 * w)
    out = np.zeros((b, c // 32, rows, 8), feat.dtype)
    for m in range(2 * h):
        r0 = lead + m * pp
        out[:, :, r0 : r0 + 2 * w, :] = shuffled[:, :, m, :].reshape(b, c // 32, 8, 2 * w).transpose(0, 1, 3, 2)
    return out


def pack_rows_nhwc(feat_nhwc):
    """feat (B, H, W, C) uint16 -> the same rows, as the channels-last kernel forms them: each pixel's 32-channel run of a
    K-chunk de-interleaved into the four sub-pixel entries q = 2 di + dj (element k of entry q = channel 4 k + q)."""
    b, h, w, c = feat_nhwc.shape
    pp, lead, rows = row_layout(2 * h, 2 * w)
    out = np.zeros((b, c // 32, rows, 8), feat_nhwc.dtype)
    runs = feat_nhwc.reshape(b, h, w, c // 32, 8, 4)  # [..., kc, k, q]
    for i in range(h):
        for j in range(w):
            for q in range(4):
                out[:, :, lead + (2 * i + q // 2) * pp + 2 * j + q % 2, :] = runs[:, i, j, :, :, q]
    return out
