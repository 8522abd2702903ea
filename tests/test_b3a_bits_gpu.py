"""The layer-1 data gradient (b3a_dgrad_kernel) computes the same d-feature bits as the kernel it replaced.

Each d-feature element is one fixed mma.sync sequence from zero (shift 0..3, K = 16 steps ascending, the all-zero steps
skipped), so which warp, fragment or column order computes it does not change its bits.  ``tests/golden/b3a_dfeat.npz``
holds the d features of the earlier kernel for seeded heads at every feature width the backward serves: BASELINE config
2's head, partial 128-channel tiles (C = 384), both epilogues (TMA and direct stores) and a keypoint-group head (the fp32
sums of the groups).  The heads end in logits, so the vectors depend on the backward's kernels and not on a softmax form.
Per case it keeps the shape, the SHA-256 of every element's bits and an evenly strided sample of at most 4,096 elements
(which shows where a mismatch lies), so the file stays small at config 2's 2048 channels.

    python tests/test_b3a_bits_gpu.py OUT.npz    # rewrite the vectors with the library in this tree
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from head_support import features, gen, grads, make_head  # noqa: E402

# name: (C, H, W, channels, B)
CASES = {
    "w4_c512_4x4": (512, 4, 4, (17, 17), 3),
    "w8_c512_8x8": (512, 8, 8, (9, 9), 2),
    "cfg2_c2048_12x12": (2048, 12, 12, (17, 17), 1),
    "w16_c384_12x16": (384, 12, 16, (17,), 1),
    "w24_c384_6x24": (384, 6, 24, (17,), 1),
    "w32_c384_8x32": (384, 8, 32, (17,), 1),
    "wide_c512_8x8_k40": (512, 8, 8, (40, 40), 2),
}


def dfeat_bits(name):
    """the d features of sum(head(feats) * gout) for the case's seeded head, as uint16 bit patterns"""
    from lightning_pose_b200 import ops

    c, h, w, ch, b = CASES[name]
    assert ops.head_bf16_supported((b, c, h, w), list(ch), train=True), name
    head = make_head(c, ch, seed=41, final_softmax=False)
    feats = features(b, c, h, w, 42, torch.bfloat16)
    up = 8 if len(ch) == 2 else 4
    gout = torch.randn(b, ch[-1], up * h, up * w, device="cuda", generator=gen(43))
    d = grads(head, feats, gout)["dfeat"]
    assert d.dtype == torch.bfloat16 and d.shape == feats.shape
    return d.view(torch.int16).cpu().numpy().view(np.uint16)


SAMPLE = 4096


def fixture(bits):
    """{shape, sha256, sample} of a case's d-feature bits"""
    flat = bits.reshape(-1)
    digest = np.frombuffer(hashlib.sha256(flat.astype("<u2").tobytes()).digest(), dtype=np.uint8)
    return {"shape": np.array(bits.shape, dtype=np.int64), "sha256": digest, "sample": flat[:: -(-flat.size // SAMPLE)]}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_dfeat_bits(golden, name):
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)

    got, want = fixture(dfeat_bits(name)), golden("b3a_dfeat")
    for key in ("shape", "sample", "sha256"):
        assert np.array_equal(got[key], want[f"{name}.{key}"]), (name, key)


if __name__ == "__main__":
    import lightning_pose_b200  # noqa: F401

    np.savez_compressed(sys.argv[1], **{f"{name}.{k}": v for name in CASES for k, v in fixture(dfeat_bits(name)).items()})
