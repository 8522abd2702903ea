"""The decode on the head's band maxima (``lpb_decode_fwd_banded``) gives the full sweep's outputs, bit for bit.

The 16-bit head's softmax writes, per (frame, plane, band of its rows), the largest value each epilogue warp stored.
The banded decode sweeps only the band that holds the plane's first arg max and the bands whose maximum reaches the
hull threshold.  Checked here: the maxima equal the maxima of the written heatmaps over each band's rows, and xy,
confidence and stats equal ``ops.decode_forward``'s, on the bench's planes (trained and fresh, fused and split softmax),
other map sizes, 51 keypoints, fp16 features, and planted planes whose maxima are given in the kernel's format: ties
across and inside bands and on a band boundary, hulls across bands, peaks at the plane edges and in the short last band,
and NaN planes.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from head_support import assert_same_decode, band_dims as dims, bits, features, head_params, head_run, make_head  # noqa: E402

T = 1000.0


def slots_of(hm, rows, nbands):
    """kernel-format band maxima of arbitrary planes: slot e of band j = the maximum over its rows r with r % 8 == e"""
    b, k, h, w = hm.shape
    pad = torch.zeros((b, k, nbands * 2 * rows - h, w), device=hm.device)
    x = torch.cat([torch.nan_to_num(hm, nan=0.0), pad], dim=2).reshape(b, k, nbands, 2 * rows, w)
    out = torch.zeros((b, k, nbands, 8), device=hm.device)
    for e in range(8):
        part = x[:, :, :, e::8]
        if part.shape[3]:
            out[..., e] = part.amax(dim=(3, 4))
    return out.view(torch.int32).contiguous()


@pytest.fixture(scope="module")
def bench_problems():
    import bench

    out = {}
    for regime in ("trained", "fresh"):
        prob = bench.make_problem(16, seed=1234, device="cpu", regime=regime)
        w1, b1, w2, b2 = prob["head_params"]
        feats = prob["feats"].to(torch.bfloat16)
        out[regime] = ([w1.cuda(), w2.cuda()], [b1.cuda(), b2.cuda()], feats[:256].cuda(), feats[256:].cuda())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["trained", "fresh"])
@pytest.mark.parametrize("split", [0, 2])
def test_bench_planes(bench_problems, regime, split):
    """the bench's labeled (256) and unlabeled (512) calls, fused and split softmax"""
    weights, biases, lab, unl = bench_problems[regime]
    for name, feats in (("labeled", lab), ("unlabeled", unl)):
        hm, hints = head_run(feats, weights, biases, split)
        assert_same_decode(hm, hints, 2, f"{regime}/{name}/split={split}")


@pytest.mark.gpu
@pytest.mark.parametrize("ds", [1, 2, 3])
@pytest.mark.parametrize("case", ["cfg2_96", "vit_64", "cfg5_128", "wide51", "f16"])
def test_head_shapes(case, ds):
    """config 2's 96 x 96 maps, a one-deconv (ViT) head's 64 x 64, config 5's 128 x 128, 51 keypoints, fp16 features"""
    c, h, w, ch, b, dtype = {
        "cfg2_96": (2048, 12, 12, (17, 17), 6, torch.bfloat16),
        "vit_64": (384, 16, 16, (17,), 6, torch.bfloat16),
        "cfg5_128": (512, 16, 16, (17, 17), 4, torch.bfloat16),
        "wide51": (512, 8, 8, (51, 51), 3, torch.bfloat16),
        "f16": (2048, 12, 12, (17, 17), 4, torch.float16),
    }[case]
    head = make_head(c, ch, seed=11, gain=6.0)
    weights, biases = head_params(head)
    feats = features(b, c, h, w, 12, dtype)
    for split in (0, 2):
        hm, hints = head_run(feats, weights, biases, split)
        assert_same_decode(hm, hints, ds, f"{case}/split={split}")


def planted(h=96, w=96, n=1):
    """n planes of small noise (softmax-like: positive, tiny)"""
    g = torch.Generator().manual_seed(5)
    return (torch.rand((1, n, h, w), generator=g) * 1e-6).cuda()


def bump(p, y, x, peak, sigma=1.0):
    h, w = p.shape
    yy, xx = torch.meshgrid(torch.arange(h, device=p.device), torch.arange(w, device=p.device), indexing="ij")
    p += peak * torch.exp(-((yy - y) ** 2 + (xx - x) ** 2) / (2 * sigma**2))


def decode_planted(hm, ds=2, case=""):
    from lightning_pose_b200 import ops

    rows, nbands = dims(hm.shape[2], hm.shape[3])
    bm = ops.BandMax(slots_of(hm, rows, nbands), rows, nbands)
    return assert_same_decode(hm, bm, ds, case), bm


@pytest.mark.gpu
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_planted_ties_and_edges(ds):
    """96 x 96 planes: bands of 10 rows, the last of 6 (rows 90-95)"""
    rows, nbands = dims(96, 96)
    assert (rows, nbands) == (5, 10)
    hm = planted(n=7)
    p = hm[0]
    # 0: equal maxima in one band at two indices
    bump(p[0], 33, 50, 0.2)
    p[0, 33, 50] = p[0, 36, 52] = 0.3
    # 1: equal maxima on a band boundary (rows 19 | 20)
    bump(p[1], 19, 60, 0.1, sigma=1.3)
    p[1, 19, 60] = p[1, 20, 61] = 0.2
    # 2: a hull straddling three bands
    bump(p[2], 50, 30, 0.2, sigma=3.0)
    # 3-6: peaks at the plane's corners and edges, in the first and the short last band
    bump(p[3], 0, 0, 0.3)
    bump(p[4], 95, 95, 0.3)
    bump(p[5], 92, 0, 0.3)
    bump(p[6], 0, 95, 0.3, sigma=1.5)
    decode_planted(hm, ds, "planted")


@pytest.mark.gpu
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_tie_across_bands_takes_the_first(ds):
    """Equal maxima in bands 1 (row 17) and 2 (row 22).  The first stands alone, the second tops a flat 5 x 5 block, so
    the field's lower bound at the first is smaller, and so is the hull threshold: a plateau (rows 50-85) at a level
    between the two thresholds is a candidate only from the first peak, whose hull then overflows the window.  The planes
    sweep the plateau level; on each the banded decode equals the full sweep, and on some a decode that took the later
    band would not."""
    from lightning_pose_b200 import ops

    levels = [0.005 * i for i in range(1, 50)]
    hm = planted(n=len(levels))
    for i, lv in enumerate(levels):
        q = hm[0, i]
        q[17, 40] = 0.25
        q[20:25, 42:47] = 0.2499
        q[22, 44] = 0.25
        q[50:86, 10:86] += lv
    full, bm = decode_planted(hm, ds, "tie")
    rows, nbands = dims(96, 96)
    late = bm.bits.clone()
    b1 = late[0, :, 1]
    late[0, :, 1] = torch.where(b1 == b1.amax(dim=1, keepdim=True), b1 - 1, b1)  # band 1 one ulp below: band 2 is taken
    other = ops.decode_forward(hm, ds, T, band_max=ops.BandMax(late, rows, nbands))
    differ = [(bits(full[2][0, i]) != bits(other[2][0, i])).any().item() for i in range(len(levels))]
    assert any(differ), "no plateau level makes the band choice visible"


@pytest.mark.gpu
def test_planted_nan_planes():
    """an all-NaN plane (no positive finite maximum: the full sweeps queue it) and a single NaN away from the peak"""
    hm = planted(n=3)
    p = hm[0]
    p[0] = float("nan")
    bump(p[1], 40, 40, 0.3)
    p[1, 80, 10] = float("nan")
    bump(p[2], 70, 20, 0.3)
    full, _ = decode_planted(hm, 2, "nan")
    assert torch.isnan(full[0][0, 0]).all()


@pytest.mark.gpu
def test_other_width_short_last_band():
    """64 x 80 maps (bands of 6 rows, the last of 4) with peaks in the last band"""
    rows, nbands = dims(64, 80)
    hm = planted(64, 80, n=3)
    p = hm[0]
    bump(p[0], 63, 79, 0.3)
    bump(p[1], 61, 3, 0.3)
    bump(p[2], 59, 40, 0.2, sigma=2.0)
    assert nbands * 2 * rows > 64
    decode_planted(hm, 2, "64x80")
