"""The 16-bit head's forward on the shapes only prediction reaches, against float64.

The forward plan (``lpb_head_bf16_plan_layout``) accepts far more shapes than the backward trains (even H, W in {4, 8,
12, 16, 24, 32}): any C that is a multiple of 128, any H x W with H * W % 8 == 0, W up to 63 (two deconvs) or 127 (one
deconv), and for NCHW features a map whose 32-channel slab fits the shuffle stage's 200 KB.  Every shape in that set is
a prediction shape (an ``image_resize_dims`` whose feature map is not a trained width), and it runs on one of two routes:

* k1a (head_bf16.cu), two-deconv NCHW maps of at most 192 pixels and W <= 31: (frame, band) items of units of
  a = 8 / gcd(W, 8) feature rows, G bands per frame as equal as possible (``urem`` of them one unit larger);
* the banded kernels (head_rows_bf16.cu), everything else: each transposed convolution cuts its Hi x Wi input into bands
  of R = 256 / (Wi + 1) image rows (two M-tiles of 128 raster rows), the last band shorter where R does not divide Hi.

``TABLE`` puts one row through each class of either route, the widest widths, the shuffle budget exactly, an NHWC map
past it, and the first shapes refused at each limit.  On the CPU, each row's route is asserted from the library's
planner, the planner is restated here and compared with the library over a grid of shapes, and every class the grid
holds must have a row (``test_table_covers_the_accepted_domain``), so a routing change cannot quietly shrink the
coverage.  On the GPU, each accepted row's heatmaps (fused, split and default softmax) and logits are held to
``head_support``'s float64 bars, its band maxima to the heatmaps' own, the decode on them to the full sweep bit for bit,
and its keypoints to the float64 decode of the float64 heatmaps; refused rows run on the fp32 kernels at their bar,
except a two-deconv map past the shuffle budget, whose heatmaps the fp32 plane softmax refuses as well."""
import collections
import ctypes
import math

import pytest
import torch

import scale_oracle as S
from head_support import (F64, STAGE_BYTES, WORST, _judge, assert_same_decode, band_dims, bits, check_heatmaps, features, forward_checks,
                          head_params, head_run, make_head, ref_forward, report_headroom, softmax_split)

NCHW, NHWC = 0, 1          # LPB_FEATURES_* (lpb200.h)
ERR_UNSUPPORTED = -3       # LPB_ERR_UNSUPPORTED
GAIN = 6.0                 # the keypoint checks' heads: peaked planes, as a trained head makes them
T = 1000.0                 # the head's soft-argmax temperature

# ------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------
Row = collections.namedtuple("Row", "deconvs c h w channels b layout route")

# The cfg rows are prediction shapes of real models: a ResNet-50 on 256 x 320 frames (8 x 10 map) and a ViT-S with
# 16-pixel patches on 448 x 448 frames (28 x 28 map).  The other rows keep C small, so the float64 reference stays cheap.
TABLE = {
    # k1a: two deconvs, NCHW.  (a, G, urem) in the comments.
    "k1a_1x8": Row(2, 128, 1, 8, (17, 17), 3, NCHW, "k1a"),          # (1, 1, 0): one feature row
    "k1a_3x16": Row(2, 256, 3, 16, (9, 13), 3, NCHW, "k1a"),         # (1, 1, 0): odd H
    "k1a_13x8": Row(2, 128, 13, 8, (17, 17), 2, NCHW, "k1a"),        # (1, 2, 1): bands of 7 and 6 rows
    "k1a_23x8": Row(2, 384, 23, 8, (17, 17), 2, NCHW, "k1a"),          # (1, 3, 2): 8, 8, 7
    "k1a_4x20": Row(2, 256, 4, 20, (17, 17), 3, NCHW, "k1a"),        # (2, 1, 0)
    "k1a_8x20": Row(2, 128, 8, 20, (17, 17), 2, NCHW, "k1a"),        # (2, 2, 0)
    "k1a_6x20": Row(2, 256, 6, 20, (19, 19), 2, NCHW, "k1a"),        # (2, 2, 1): 4, 2
    "k1a_6x28": Row(2, 128, 6, 28, (17, 17), 2, NCHW, "k1a"),        # (2, 3, 0)
    "k1a_4x10": Row(2, 512, 4, 10, (1, 1), 3, NCHW, "k1a"),          # (4, 1, 0)
    "cfg_r50_256x320": Row(2, 2048, 8, 10, (17, 17), 2, NCHW, "k1a"),  # (4, 1, 0)
    "k1a_12x10": Row(2, 128, 12, 10, (17, 17), 2, NCHW, "k1a"),      # (4, 2, 1): 8, 4
    "k1a_16x10": Row(2, 128, 16, 10, (8, 17), 2, NCHW, "k1a"),       # (4, 2, 0)
    "k1a_12x14": Row(2, 128, 12, 14, (17, 8), 2, NCHW, "k1a"),       # (4, 3, 0)
    "k1a_32x6": Row(2, 128, 32, 6, (17, 17), 2, NCHW, "k1a"),        # (4, 3, 2): 12, 12, 8
    "k1a_8x9": Row(2, 128, 8, 9, (17, 17), 3, NCHW, "k1a"),          # (8, 1, 0)
    "k1a_16x11": Row(2, 256, 16, 11, (17, 17), 2, NCHW, "k1a"),      # (8, 2, 0)
    "k1a_24x7": Row(2, 128, 24, 7, (17, 17), 2, NCHW, "k1a"),        # (8, 3, 0)
    # banded, two deconvs.  Layer 1 / layer 2 bands in the comments.
    "2d_8x1": Row(2, 128, 8, 1, (17, 17), 3, NCHW, "banded"),        # one band / one band
    "2d_8x2": Row(2, 128, 8, 2, (17, 17), 3, NCHW, "banded"),        # one / 28 + 4 rows
    "2d_8x3": Row(2, 256, 8, 3, (5, 7), 3, NCHW, "banded"),          # one / 19 + 13
    "2d_8x5": Row(2, 128, 8, 5, (17, 17), 2, NCHW, "banded"),        # one / 12, 12, 8
    "2d_8x13": Row(2, 128, 8, 13, (17, 17), 2, NCHW, "banded"),      # k1a gate passed, G = 0: 9 + 7 / 16 x 4
    "2d_4x30": Row(2, 128, 4, 30, (17, 17), 2, NCHW, "banded"),      # 2 x 4 / 8 x 2
    "2d_3x32": Row(2, 128, 3, 32, (17, 17), 2, NCHW, "banded"),      # 3 + 3 / R = 1: the widest heatmaps the decode takes
    "2d_2x40": Row(2, 128, 2, 40, (17, 17), 2, NCHW, "banded"),      # 3 + 1 / R = 1
    "2d_8x63": Row(2, 128, 8, 63, (17, 17), 2, NCHW, "banded"),        # 8 x 2 / R = 1, 253 raster rows: the widest accepted
    "2d_64x50": Row(2, 128, 64, 50, (4, 4), 1, NCHW, "banded"),      # shuffle slab exactly 200 KB; 64 x 2 / R = 1
    "2d_400x8": Row(2, 128, 400, 8, (4, 4), 1, NCHW, "banded"),      # shuffle slab exactly 200 KB; 53 x 15 + 5 / 228 x 7 + 4
    # banded, one deconv
    "1d_1x8": Row(1, 128, 1, 8, (17,), 3, NCHW, "banded"),           # one band
    "1d_4x2": Row(1, 256, 4, 2, (17,), 3, NCHW, "banded"),           # one band
    "1d_9x8": Row(1, 128, 9, 8, (20,), 2, NCHW, "banded"),           # 15 + 3
    "cfg_vit_448": Row(1, 384, 28, 28, (17,), 2, NCHW, "banded"),    # 14 x 4
    "1d_3x64": Row(1, 128, 3, 64, (17,), 2, NCHW, "banded"),         # R = 1: the widest heatmaps the decode takes
    "1d_8x127": Row(1, 128, 8, 127, (17,), 2, NCHW, "banded"),       # R = 1, 255 raster rows: the widest accepted
    "1d_24x127": Row(1, 128, 24, 127, (4,), 1, NCHW, "banded"),      # R = 1, 48 bands
    # channels-last features: always the banded kernels, no shuffle budget
    "nhwc_2d_13x8": Row(2, 128, 13, 8, (17, 17), 2, NHWC, "banded"),  # NCHW takes k1a
    "nhwc_2d_448x8": Row(2, 128, 448, 8, (4, 4), 1, NHWC, "banded"),  # NCHW refuses: 224 KB slab
    "nhwc_vit_448": Row(1, 384, 28, 28, (17,), 2, NHWC, "banded"),    # a ViT's tokens read in place
    # refused: the first shape past each limit
    "refused_2d_8x64": Row(2, 128, 8, 64, (17, 17), 2, NCHW, "refused"),   # 4 W + 1 = 257 raster rows
    "refused_1d_8x128": Row(1, 128, 8, 128, (17,), 2, NCHW, "refused"),    # 2 W + 1 = 257
    "refused_1d_401x8": Row(1, 128, 401, 8, (4,), 1, NCHW, "refused"),     # slab 200.5 KB
    "refused_2d_401x8": Row(2, 128, 401, 8, (4, 4), 1, NCHW, "refused"),   # slab 200.5 KB
}
ACCEPTED = [name for name, r in TABLE.items() if r.route != "refused"]
REFUSED = [name for name, r in TABLE.items() if r.route == "refused"]
# W = 8 is a trained width at every even H, so the exact shuffle budget along H (400 rows) and the NHWC map past it are
# shapes the backward also serves; every other row is forward-only
TRAINED_ROWS = {"2d_400x8", "nhwc_2d_448x8"}

# ------------------------------------------------------------------------------------------------
# the planner, restated (head_bf16.cu, head_rows.cuh)
# ------------------------------------------------------------------------------------------------
K1A_BAND_ROWS = 16 * 3 * 8            # raster rows of k1a's largest band: 8 MMA warps x 3 m16 tiles
K1A_STAGES, K1A_ZROWS, HEAD_KSTAGE = 2, 72, 32
CR_BAND_ROWS = 256                    # raster rows of a banded-kernel band: two M-tiles of 128
SHUFFLE_BUDGET = 200 * 1024           # HEAD_FEATURE_SMEM_BUDGET: rows_shuffle_kernel's [32][H * W] slab
PLAN_SMEM = 227 * 1024                # planning_limits(): an H100 SM's opt-in shared memory

K1aGeom = collections.namedtuple("K1aGeom", "a G ubase urem nbmax nfs box rows_alloc")


def k1a_geom(h, w):
    """make_k1a_geom: bands of units of a = 8 / gcd(W, 8) feature rows (a band's TMA box starts on 16 bytes), G the
    smallest band count whose largest band's raster (2 rows per feature row, pitch 2W + 1) fits K1A_BAND_ROWS."""
    a = 8 // math.gcd(w, 8)
    nu = -(-h // a)
    p = 2 * w + 1
    g = next((g for g in range(1, nu + 1) if 2 * min(-(-nu // g) * a, h) * p <= K1A_BAND_ROWS), 0)
    if g == 0:
        return K1aGeom(a, 0, 0, 0, 0, 0, 0, 0)
    ubase, urem = nu // g, nu % g
    nbmax = min((ubase + (urem > 0)) * a, h)
    nfs = nbmax + (g > 1)
    box = (nfs * w + 7) & ~7
    mma_rows = -(-2 * nbmax * p // 16) * 16 + p + 1
    rows_alloc = (max(mma_rows, 2 * nfs * p) + 7) & ~7
    return K1aGeom(a, g, ubase, urem, nbmax, nfs, box, rows_alloc)


def k1a_bands(h, w):
    """k1a_band: (first feature row, rows) of each band of a frame"""
    k = k1a_geom(h, w)
    out = []
    for band in range(k.G):
        f0 = k.a * (band * k.ubase + min(band, k.urem))
        out.append((f0, min(k.a * (k.ubase + (band < k.urem)), h - f0)))
    return out


def k1a_smem(k):
    return K1A_STAGES * (4 * k.rows_alloc * 16 + STAGE_BYTES) + K1A_STAGES * 4 * HEAD_KSTAGE * k.box * 2 + 128 + K1A_ZROWS * 16


def bands(hi, wi):
    """launch_convt_rows' cut of an hi x wi input: (R, band count, rows of the last band)"""
    r = max(1, min(CR_BAND_ROWS // (wi + 1), hi))
    n = -(-hi // r)
    return r, n, hi - (n - 1) * r


def band_kind(hi, wi):
    r, n, last = bands(hi, wi)
    if n == 1:
        return "one band"
    if r == 1:
        return "R = 1"
    return "short last band" if last < r else "equal bands"


def refusals(deconvs, layout, h, w):
    """the limits of the banded path a shape breaks (head_bf16.cu lpb_head_bf16_plan_layout)"""
    out = []
    if layout == NCHW and 32 * h * w * 2 > SHUFFLE_BUDGET:
        out.append("shuffle budget")
    if 2 * deconvs * w + 1 > CR_BAND_ROWS:
        out.append("width")
    return out


def plan(deconvs, layout, h, w):
    """'k1a', 'banded' or 'refused' for a narrow head (at most 20 channels per layer) and any valid C"""
    if layout == NCHW and deconvs == 2 and (w >= 7 or w in (4, 6)) and h * w <= 192 and w <= 31:
        k = k1a_geom(h, w)
        if k.G > 0 and k1a_smem(k) <= PLAN_SMEM:
            return "k1a"
    return "refused" if refusals(deconvs, layout, h, w) else "banded"


def banded_layers(deconvs, route, h, w):
    """the (Hi, Wi) inputs of the layers the banded kernel runs; the last one writes the heatmaps and band maxima"""
    if deconvs == 1:
        return [(2 * h, 2 * w)]
    return [(4 * h, 4 * w)] if route == "k1a" else [(2 * h, 2 * w), (4 * h, 4 * w)]


def classes(deconvs, layout, h, w):
    """the kernel code paths a shape selects"""
    route = plan(deconvs, layout, h, w)
    if route == "refused":
        return {("refused", deconvs, why) for why in refusals(deconvs, layout, h, w)}
    out = {("route", deconvs, layout, route)}
    if route == "k1a":
        k = k1a_geom(h, w)
        out.add(("k1a", k.a, k.G, k.urem > 0))
        if h == 1:
            out.add(("k1a", "H = 1"))
        elif h % 2:
            out.add(("k1a", "odd H"))
    layers = banded_layers(deconvs, route, h, w)
    for i, (hi, wi) in enumerate(layers):
        out.add(("band", deconvs, "last layer" if i == len(layers) - 1 else "layer 1", band_kind(hi, wi)))
    if layout == NHWC:
        nchw = plan(deconvs, NCHW, h, w)
        if nchw != "banded":
            out.add(("nhwc", "NCHW route " + nchw))
    return out


def backward_serves(h, w):
    """head_bwd_covers (head_bwd_bf16.cu) for NCHW features: the shapes test_head_shapes_gpu.py covers"""
    return h % 2 == 0 and w in (4, 8, 12, 16, 24, 32)


def lib_plan(row_or_shape):
    """the library's plan for a table row or (deconvs, C, H, W, channels, layout): (return code, plan)"""
    from lightning_pose_b200._lib import lib

    d, c, h, w, ch, layout = row_or_shape
    p = ctypes.c_int(-1)
    rc = lib.lpb_head_bf16_plan_layout(c, h, w, ch[0], ch[1] if d == 2 else 0, layout, ctypes.byref(p))
    return rc, p.value


def row_shape(r):
    return (r.deconvs, r.c, r.h, r.w, r.channels, r.layout)


# ------------------------------------------------------------------------------------------------
# CPU: routes, restated geometry, coverage
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", list(TABLE))
def test_table_routes(row):
    """Each row takes the route it states; refused rows get LPB_ERR_UNSUPPORTED and are not served by the 16-bit
    kernels at any call; no row but the two tall W = 8 maps is a shape the backward trains."""
    from lightning_pose_b200 import ops

    r = TABLE[row]
    assert len(r.channels) == r.deconvs and r.c % 128 == 0 and (r.h * r.w) % 8 == 0
    assert plan(r.deconvs, r.layout, r.h, r.w) == r.route
    rc, p = lib_plan(row_shape(r))
    shape = (r.b, r.c, r.h, r.w)
    if r.route == "refused":
        assert rc == ERR_UNSUPPORTED
        assert not ops.head_bf16_supported(shape, list(r.channels), train=False, layout=r.layout)
    else:
        assert rc == 0 and {1: "k1a", 0: "banded"}[p] == r.route
        assert ops.head_bf16_supported(shape, list(r.channels), train=False, layout=r.layout)
    trained = ops.head_bf16_supported(shape, list(r.channels), train=True, layout=r.layout)
    assert trained == (row in TRAINED_ROWS)
    assert trained == (backward_serves(r.h, r.w) and r.route != "refused")


def test_restated_k1a_geometry():
    """k1a's bands, restated: every k1a row's bands tile its frame in units of a rows (the last one clipped), the
    first ``urem`` one unit larger, each band starts on a 16-byte TMA boundary, and the largest fits K1A_BAND_ROWS
    where one band fewer would not.  The table's comments state (a, G, urem) and the band rows; they are checked here."""
    expect = {
        "k1a_1x8": (1, 1, 0, [1]), "k1a_3x16": (1, 1, 0, [3]), "k1a_13x8": (1, 2, 1, [7, 6]), "k1a_23x8": (1, 3, 2, [8, 8, 7]),
        "k1a_8x20": (2, 2, 0, [4, 4]), "k1a_6x20": (2, 2, 1, [4, 2]), "k1a_6x28": (2, 3, 0, [2, 2, 2]), "k1a_4x10": (4, 1, 0, [4]),
        "k1a_4x20": (2, 1, 0, [4]), "cfg_r50_256x320": (4, 1, 0, [8]), "k1a_12x10": (4, 2, 1, [8, 4]), "k1a_16x10": (4, 2, 0, [8, 8]),
        "k1a_12x14": (4, 3, 0, [4, 4, 4]), "k1a_32x6": (4, 3, 2, [12, 12, 8]), "k1a_8x9": (8, 1, 0, [8]),
        "k1a_16x11": (8, 2, 0, [8, 8]), "k1a_24x7": (8, 3, 0, [8, 8, 8]),
    }
    assert set(expect) == {n for n, r in TABLE.items() if r.route == "k1a"}
    for name, (a, g, urem, rows) in expect.items():
        r = TABLE[name]
        k = k1a_geom(r.h, r.w)
        assert (k.a, k.G, k.urem) == (a, g, urem), name
        bs = k1a_bands(r.h, r.w)
        assert [nb for _, nb in bs] == rows and sum(rows) == r.h, name
        assert [f0 for f0, _ in bs] == [sum(rows[:i]) for i in range(len(rows))], name
        assert all((f0 * r.w) % 8 == 0 for f0, _ in bs), name
        assert 2 * k.nbmax * (2 * r.w + 1) <= K1A_BAND_ROWS, name
        assert k.box <= r.h * r.w and k.box <= 256, name  # the TMA box stays inside the frame (make_feat_tensor_map)
        if g > 1:  # one band fewer does not fit
            assert 2 * min(-(-(-(-r.h // a)) // (g - 1)) * a, r.h) * (2 * r.w + 1) > K1A_BAND_ROWS, name
    # the one row the k1a gate passes but no band count fits
    assert k1a_geom(8, 13).G == 0 and TABLE["2d_8x13"].route == "banded"


def test_restated_bands_match_the_library():
    """The banded path's (R, bands) of every accepted row's last layer equal ``lpb_head_band_max_dims``, and the rows'
    comments state them: R = 1 rows at the widest widths (Pp = 253, 255 raster rows), one band, equal bands and a short
    last band at both depths."""
    for name in ACCEPTED:
        r = TABLE[name]
        hi, wi = banded_layers(r.deconvs, r.route, r.h, r.w)[-1]
        rr, n, _ = bands(hi, wi)
        assert band_dims(2 * hi, 2 * wi) == (rr, n), name
    assert bands(32, 252) == (1, 32, 1) and bands(16, 254) == (1, 16, 1)  # 8 x 63 layer 2, 8 x 127
    assert bands(32, 8) == (28, 2, 4) and bands(32, 12) == (19, 2, 13) and bands(32, 20) == (12, 3, 8)  # 8 x 2, 8 x 3, 8 x 5
    assert bands(16, 26) == (9, 2, 7) and bands(64, 52) == (4, 16, 4)  # 8 x 13, both layers
    assert bands(800, 16) == (15, 54, 5) and bands(1600, 32) == (7, 229, 4)  # 400 x 8
    assert bands(18, 16) == (15, 2, 3) and bands(56, 56) == (4, 14, 4)  # 9 x 8 and 28 x 28, one deconv
    # one row past each limit
    assert 32 * 64 * 50 * 2 == SHUFFLE_BUDGET == 32 * 400 * 8 * 2 < 32 * 401 * 8 * 2
    assert 4 * 63 + 1 <= CR_BAND_ROWS < 4 * 64 + 1 and 2 * 127 + 1 <= CR_BAND_ROWS < 2 * 128 + 1


GRID_H, GRID_W = range(1, 65), range(1, 129)


def test_restated_planner_matches_the_library():
    """On every shape of the grid (H <= 64, W <= 128, both depths, both layouts) the restated planner gives the
    library's answer: k1a, banded, or LPB_ERR_UNSUPPORTED."""
    code = {"k1a": (0, 1), "banded": (0, 0)}
    bad = []
    for d in (1, 2):
        for layout in (NCHW, NHWC):
            for h in GRID_H:
                for w in GRID_W:
                    if (h * w) % 8:
                        continue
                    want = plan(d, layout, h, w)
                    rc, p = lib_plan((d, 128, h, w, (17, 17), layout))
                    got = (rc, p) if rc == 0 else (rc,)
                    if got != code.get(want, (ERR_UNSUPPORTED,)):
                        bad.append((d, layout, h, w, want, got))
    assert not bad, bad[:10]


def test_table_covers_the_accepted_domain():
    """Every class of kernel path the forward-only shapes of the grid hold (k1a's (a, G, unequal bands), H = 1 and odd
    H; each banded layer's one band / equal bands / short last band / R = 1 at both depths and layouts; NHWC maps NCHW
    would route elsewhere; each refusal) has at least one table row.  The shapes the backward trains are
    test_head_shapes_gpu.py's."""
    found = set()
    for d in (1, 2):
        for layout in (NCHW, NHWC):
            for h in GRID_H:
                for w in GRID_W:
                    if (h * w) % 8 == 0 and not backward_serves(h, w):
                        found |= classes(d, layout, h, w)
    covered = set().union(*(classes(r.deconvs, r.layout, r.h, r.w) for r in TABLE.values()))
    missing = sorted(found - covered, key=str)
    assert not missing, missing
    # the table's edges: the widest accepted width at each depth, the shuffle budget exactly along W and along H, and an
    # NHWC map past it
    rows = TABLE.values()
    assert {(r.deconvs, r.w) for r in rows if r.route == "banded"} >= {(2, 63), (1, 127)}
    assert {(r.h, r.w) for r in rows if r.layout == NCHW and r.route == "banded" and 64 * r.h * r.w == SHUFFLE_BUDGET} == {(64, 50), (400, 8)}
    assert any(r.layout == NHWC and 64 * r.h * r.w > SHUFFLE_BUDGET for r in rows)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200._lib import lib

    return lib


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


def row_inputs(name, dtype=torch.bfloat16, b=None, seed=41, gain=3.0):
    """(head, features) of a row: features in the row's memory format.  Gain 3 is the head the ``head_support`` bars
    were set on; the keypoint checks take gain ``GAIN``."""
    from lightning_pose_b200 import ops

    r = TABLE[name]
    head = make_head(r.c, r.channels, seed=seed, gain=gain)
    feats = features(r.b if b is None else b, r.c, r.h, r.w, seed + 1, dtype)
    if r.layout == NHWC:
        feats = feats.contiguous(memory_format=torch.channels_last)
        assert ops.feature_layout(feats) == ops.FEATURES_NHWC, name
    return head, feats


def decode_fwd_smem(h, w, ds):
    """launch_decode_fwd's shared memory (decode.cu): the zero-padded plane tile, DEC_FWD_SCRATCH floats and 16 B"""
    r = ds + 2
    pitch = (((r + 3) & ~3) + w + r + 3) & ~3
    return ((h + 2 * r) * pitch + 880) * 4 + 16


def decode_serves(h, w, ds, dev):
    limit = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    return w <= 256 and (w << ds) <= 1024 and decode_fwd_smem(h, w, ds) <= limit


def peak_ratio(hm):
    """per plane: the second-largest 3 x 3 local maximum over the largest.  Under the heatmap bar (every pixel within
    3e-2 relative) two peaks can trade places when the ratio exceeds (1 - 3e-2) / (1 + 3e-2) = 0.94, and then the
    soft-argmax at T = 1000 legitimately jumps from one to the other."""
    b, k, h, w = hm.shape
    x = hm.reshape(b * k, 1, h, w)
    peaks = torch.where(x == torch.nn.functional.max_pool2d(x, 3, 1, 1), x, torch.zeros_like(x)).flatten(1)
    top = peaks.topk(min(2, h * w), dim=1).values
    second = top[:, 1] if top.shape[1] > 1 else torch.zeros_like(top[:, 0])
    return (second / top[:, 0]).reshape(b, k)


def keypoint_checks(head, feats, case, dev):
    """``forward_with_keypoints``: the band maxima equal the heatmaps' own per band under the fused and the split
    softmax, the decode on them equals the full sweep bit for bit, the keypoints are those of the float64 decode of
    the same heatmaps (``test_head_shapes_gpu.py::test_fused_decode``'s bar) on every plane, and within 0.5 px of the
    float64 decode of the float64 heatmaps on the planes the reference is confident in and whose largest peak no other
    peak can overtake within the heatmap bar (``peak_ratio``).  Heatmaps the decode does not take (wider than 256
    columns, or a CTA tile past shared memory) are refused with LPB_ERR_UNSUPPORTED, and nothing is returned."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200._lib import LpbError

    ws, bs = head_params(head)
    ds = head.downsample_factor
    runs = {split: head_run(feats, ws, bs, split) for split in (0, 2)}
    b, k, hh, ww = runs[0][0].shape
    if not decode_serves(hh, ww, ds, dev):
        with torch.no_grad(), pytest.raises(LpbError, match=f"error {ERR_UNSUPPORTED}: decode_fwd"):
            head.forward_with_keypoints(feats)
        return
    for split, (hm, hints) in runs.items():
        assert_same_decode(hm, hints, ds, f"{case} split={split}", T)
    with torch.no_grad():
        hm, kp, cf = head.forward_with_keypoints(feats)
        assert torch.equal(bits(hm), bits(head(feats))), case
    xy, conf, _ = ops.decode_forward(hm, ds, T)
    assert torch.equal(bits(kp), bits(xy.reshape(b, 2 * k))) and torch.equal(bits(cf), bits(conf)), case
    prefix = "fp16 " if feats.dtype == torch.float16 else ""
    kp64 = kp.to(F64)
    own, _, _, _ = S.decode_ref(hm, ds, T)
    _judge(case, {f"{prefix}keypoints vs float64 decode of their heatmaps": (kp64 - own).abs() / (2e-3 + 1e-4 * own.abs())})
    _, hm_ref = ref_forward(head, feats)
    kp_ref, cf_ref, _, _ = S.decode_ref(hm_ref, ds, T)
    d = (kp64 - kp_ref).abs().reshape(b, k, 2).amax(-1)
    held = (cf_ref > 0.5) & (peak_ratio(hm_ref) < 0.94)
    amb = d[~held]
    print(f"keypoints {case}: {int(held.sum())} of {held.numel()} planes held to 0.5 px; largest shift elsewhere "
          f"{float(amb.max()) if amb.numel() else 0.0:.3f} px")
    assert bool(held.any()), f"{case}: no plane to hold to the float64 heatmaps' keypoints"
    _judge(case, {f"{prefix}keypoints within 0.5 px of float64": d[held] / 0.5})


@pytest.mark.gpu
@pytest.mark.parametrize("row", ACCEPTED)
def test_forward(dev, row):
    """bf16: heatmaps (fused, split, the library's choice) and logits against float64, then ``keypoint_checks`` on a
    head with peaked planes."""
    head, feats = row_inputs(row)
    forward_checks(head, feats, row, splits=(0, 2, None), train=False)
    keypoint_checks(row_inputs(row, gain=GAIN)[0], feats, row, dev)


FP16_ROWS = ["k1a_13x8", "2d_8x5", "2d_8x63", "1d_9x8", "1d_8x127"]


def test_fp16_rows_cover_both_routes():
    """fp16 runs a k1a row and, at each depth, a banded row with a short last band and an R = 1 row."""
    kinds = {(TABLE[n].deconvs, TABLE[n].route, band_kind(*banded_layers(TABLE[n].deconvs, TABLE[n].route, TABLE[n].h, TABLE[n].w)[-1]))
             for n in FP16_ROWS}
    assert {(2, "k1a"), (2, "banded"), (1, "banded")} == {kd[:2] for kd in kinds}
    assert {(2, "banded", "R = 1"), (1, "banded", "R = 1"), (1, "banded", "short last band")} <= kinds


@pytest.mark.gpu
@pytest.mark.parametrize("row", FP16_ROWS)
def test_forward_fp16(dev, row):
    """fp16 features (``head_fwd<__half>``): the same checks at the fp16 bars."""
    head, feats = row_inputs(row, torch.float16)
    forward_checks(head, feats, f"{row} fp16", splits=(0, 2, None), train=False)
    keypoint_checks(row_inputs(row, gain=GAIN)[0], feats, f"{row} fp16", dev)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["k1a_23x8", "2d_8x63"])
def test_batch_invariance(dev, lib, row):
    """At B = 2S + 7 (every persistent CTA loops over several items), under the fused softmax every frame alone
    computes the batch's bits, and the batch agrees with float64."""
    b = 2 * torch.cuda.get_device_properties(dev).multi_processor_count + 7
    head, feats = row_inputs(row, b=b, seed=43)
    with torch.no_grad(), softmax_split(lib, 0):
        out = head(feats)
        alone = [i for i in range(b) if not torch.equal(bits(head(feats[i : i + 1])[0]), bits(out[i]))]
    assert not alone, f"{row}: frames {alone[:8]} differ alone"
    _, hm_ref = ref_forward(head, feats)
    check_heatmaps(out, hm_ref, f"{row} B={b}")


@pytest.mark.gpu
@pytest.mark.parametrize("row", REFUSED)
def test_refused(dev, row):
    """Refused shapes take the fp32 kernels: heatmaps within 1e-4 relative of float64, which the 16-bit route could not
    meet.  A two-deconv map past the shuffle budget has heatmaps of more than 204,800 pixels, past what the fp32 plane
    softmax holds in shared memory (58,112 on an H100), so no route serves it: the head says so instead of returning
    anything."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200._lib import LpbError

    r = TABLE[row]
    head, feats = row_inputs(row)
    assert ops.head_16_operand(feats, list(r.channels), train=False) is None
    limit = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    up = 4 * r.deconvs
    if up * r.h * up * r.w * 4 > limit:
        with torch.no_grad(), pytest.raises(LpbError, match=f"error {ERR_UNSUPPORTED}: plane_softmax_f32"):
            head(feats)
        return
    ws, bs = head_params(head)
    hm_ref = S.head_ref_chunked(feats, ws, bs, softmax=True, operands=None)
    with torch.no_grad():
        out = head(feats)
    ratio = (out.to(F64) - hm_ref).abs() / (1e-4 * hm_ref + 1e-9)
    _judge(row, {"fp32 heatmaps (1e-4 relative)": ratio.amax((-1, -2))})
