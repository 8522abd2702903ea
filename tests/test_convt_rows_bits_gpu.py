"""The banded transposed-convolution kernel (convt_rows_kernel) writes the same bits in every epilogue mode.

How the accumulators reach the epilogue's "lane = row" form does not change any value: every output is the same fixed
mma.sync sequence followed by the same fp32 expressions, in the same per-lane and per-warp order.  ``tests/golden/
convt_rows_bits.npz`` holds what the kernel wrote before its epilogue moved from warp shuffles to shared memory, for
seeded heads covering each mode and instantiation: the fused two-pass softmax and its split form (the P0 launch's
per-band statistics and the P1 launch's heatmaps), 17 and a run-time count of keypoints, a keypoint-group head (softmax
and mid activations), a one-deconv head without a final softmax (raw planes), channels-last and fp16 features, and
widths whose last band is short.  Per case it keeps the shape, the SHA-256 of every element's bits and an evenly
strided sample of at most 4,096 elements (which shows where a mismatch lies).

    python tests/test_convt_rows_bits_gpu.py OUT.npz    # rewrite the vectors with the library in this tree
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from head_support import _lib, features, fwd_layout, head_params, make_head, row_layout, softmax_split  # noqa: E402

HEAD_CLS = 20

# name: (C, H, W, channels, B, dtype, channels_last, final_softmax, split, what)
#   split: the pinned softmax form (0 fused, 2 split); what: the outputs kept besides the heatmaps ("mid": layer 1's
#   activations, "partials": the split form's per-band statistics)
CASES = {
    # config 2: layer 2 (17 -> 17, 48 x 48 -> 96 x 96) with NPL = 17
    "cfg2_fused": (2048, 12, 12, (17, 17), 2, torch.bfloat16, False, True, 0, ()),
    "cfg2_split": (2048, 12, 12, (17, 17), 2, torch.bfloat16, False, True, 2, ("partials",)),
    "cfg2_fused_nhwc": (2048, 12, 12, (17, 17), 2, torch.bfloat16, True, True, 0, ()),
    "cfg2_fused_f16": (2048, 12, 12, (17, 17), 2, torch.float16, False, True, 0, ()),
    # a run-time keypoint count (NPL = 0); 16 x 16 features take the banded kernel for layer 1 too (narrow MID)
    "k12_fused": (512, 8, 8, (12, 12), 2, torch.bfloat16, False, True, 0, ()),
    "k12_split": (512, 8, 8, (12, 12), 2, torch.bfloat16, False, True, 2, ("partials",)),
    "k12_mid_16x16": (384, 16, 16, (12, 12), 1, torch.bfloat16, False, True, 0, ("mid",)),
    "k17_mid_16x16": (384, 16, 16, (17, 17), 1, torch.bfloat16, False, True, 2, ("mid", "partials")),
    # keypoint groups (WIDE): 51 keypoints, layer 1 by the group MID epilogue
    "wide51_fused": (512, 8, 8, (51, 51), 2, torch.bfloat16, False, True, 0, ("mid",)),
    "wide51_split": (512, 8, 8, (51, 51), 2, torch.bfloat16, False, True, 2, ("partials",)),
    # one deconv (ViT): 24 x 32 image rows in bands of 7 (the last has 3); raw planes and softmax
    "vit_planes_k17": (384, 12, 16, (17,), 2, torch.bfloat16, False, False, 0, ()),
    "vit_planes_k12_f16": (384, 12, 16, (12,), 2, torch.float16, False, False, 0, ()),
    "vit_softmax_k17": (384, 12, 16, (17,), 2, torch.bfloat16, False, True, 0, ()),
    "vit_softmax_k17_split_nhwc": (384, 12, 16, (17,), 2, torch.bfloat16, True, True, 2, ("partials",)),
    "vit_softmax_k5": (384, 12, 16, (5,), 1, torch.bfloat16, False, True, 0, ()),
}


def _bands(hi, wi):
    r = max(1, min(256 // (wi + 1), hi))
    return -(-hi // r)


def outputs(name):
    """{"heatmaps": ..., ["mid": ..., "partials": ...]} of the case's seeded head, as unsigned-integer bit patterns"""
    from lightning_pose_b200 import ops

    c, h, w, ch, b, dtype, nhwc, final_softmax, split, what = CASES[name]
    head = make_head(c, ch, seed=51, final_softmax=final_softmax)
    weights, biases = head_params(head)
    feats = features(b, c, h, w, 52, dtype)
    layout = ops.FEATURES_NCHW
    if nhwc:
        feats = feats.contiguous(memory_format=torch.channels_last)
        layout = ops.FEATURES_NHWC
    train = dtype == torch.bfloat16  # the training form keeps the workspace (mid activations, split statistics)
    assert ops.head_bf16_supported((b, c, h, w), list(ch), train=train, layout=layout), name
    with softmax_split(_lib(), split):
        res = ops._head_forward_16(feats, weights, biases, final_softmax, train=train, layout=layout)
        torch.cuda.synchronize()
    hm, ws = (res[0], res[1][1]) if train else (res, None)
    out = {"heatmaps": hm.contiguous().view(torch.int32).cpu().numpy().view(np.uint32)}
    c1, c2 = ch[0], (ch[1] if len(ch) == 2 else 0)
    lay = fwd_layout(b, c, h, w, c1, c2)
    if "mid" in what:
        pp, lead, rows = row_layout(4 * h, 4 * w)
        mid = ws[lay.mid_at: lay.mid_at + b * 4 * lay.nst2 * rows * 16].view(torch.int16).view(b, 4 * lay.nst2, rows, 8)
        pix = (lead + torch.arange(4 * h)[:, None] * pp + torch.arange(4 * w)[None, :]).reshape(-1).cuda()
        out["mid"] = mid[:, :, pix].cpu().numpy().view(np.uint16)
    if "partials" in what:
        hi, wi, k = (8 * h, 8 * w, c2) if c2 else (4 * h, 4 * w, c1)
        groups = -(-k // HEAD_CLS)
        part_at = lay.mid_at + (b * 4 * lay.nst2 * lay.mid_rows * 16 if c2 else 0)
        nb = _bands(hi // 2, wi // 2)
        part = ws[part_at: part_at + b * groups * nb * HEAD_CLS * 2 * 4].view(torch.int32).view(b, groups, nb, HEAD_CLS, 2)
        keep = [part[:, g, :, : min(HEAD_CLS, k - HEAD_CLS * g)].reshape(b, nb, -1) for g in range(groups)]
        out["partials"] = torch.cat(keep, dim=2).cpu().numpy().view(np.uint32)
    return out


SAMPLE = 4096


def fixture(bits):
    """{shape, sha256, sample} of an output's bits"""
    flat = bits.reshape(-1)
    digest = np.frombuffer(hashlib.sha256(flat.astype(flat.dtype.newbyteorder("<")).tobytes()).digest(), dtype=np.uint8)
    return {"shape": np.array(bits.shape, dtype=np.int64), "sha256": digest, "sample": flat[:: -(-flat.size // SAMPLE)]}


def keys(name):
    return ["heatmaps", *CASES[name][-1]]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_convt_rows_bits(golden, name):
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)

    got, want = outputs(name), golden("convt_rows_bits")
    assert sorted(got) == sorted(keys(name)), name
    for out, bits in got.items():
        fx = fixture(bits)
        for key in ("shape", "sample", "sha256"):
            assert np.array_equal(fx[key], want[f"{name}.{out}.{key}"]), (name, out, key)


if __name__ == "__main__":
    import lightning_pose_b200  # noqa: F401

    np.savez_compressed(sys.argv[1], **{f"{name}.{out}.{k}": v for name in CASES for out, bits in outputs(name).items()
                                        for k, v in fixture(bits).items()})
