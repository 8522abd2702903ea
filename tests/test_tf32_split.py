"""The fp32 head's convolutions run on the tensor cores in 3xTF32 (head_f32.cu).  This CPU test pins the accuracy rule
the GPU tests hold them to -- largest error over each output channel's largest |value| below 1e-5 -- by emulating the
two GEMM kinds at the head's layer shapes with ``cvt.rna.tf32.f32`` rounding and fp32 accumulation: 3xTF32 (big and
small parts, small products first) passes, and 1xTF32, what a kernel that dropped the small products computes, fails.
"""
import numpy as np
import pytest

RULE = 1e-5


def tf32_rna(x: np.ndarray) -> np.ndarray:
    """cvt.rna.tf32.f32: keep 10 mantissa bits, round to nearest with ties away from zero."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def gemm_fp32_acc(terms, k: int) -> np.ndarray:
    """sum over k of the listed (a, b) operand products, accumulated in fp32 one k at a time (tf32 x tf32 is exact)."""
    m, n = terms[0][0].shape[0], terms[0][1].shape[1]
    acc = np.zeros((m, n), dtype=np.float32)
    for kk in range(k):
        for a, b in terms:
            acc += np.outer(a[:, kk], b[kk, :]).astype(np.float32)
    return acc


def gemm_1xtf32(a, b):
    return gemm_fp32_acc([(tf32_rna(a), tf32_rna(b))], a.shape[1])


def gemm_3xtf32(a, b):
    ab, bb = tf32_rna(a), tf32_rna(b)
    as_, bs = tf32_rna(a - ab), tf32_rna(b - bb)
    return gemm_fp32_acc([(as_, bb), (ab, bs), (ab, bb)], a.shape[1])


def rule_ratio(got, a, b) -> float:
    """largest |error| over the output channel's largest |value|, against float64, in units of the rule"""
    ref = a.astype(np.float64) @ b.astype(np.float64)
    err = np.abs(got.astype(np.float64) - ref).max(0)
    return float((err / (RULE * np.abs(ref).max(0))).max())


# (M, K, N): layer 1 of a ResNet head (512 shuffled channels x 9 taps / 4 parity classes), layer 2 (17 channels)
SHAPES = {"layer1": (96, 1152, 17), "layer2": (96, 40, 17)}


@pytest.mark.parametrize("name", list(SHAPES))
def test_rule_accepts_3xtf32_and_rejects_1xtf32(name):
    m, k, n = SHAPES[name]
    rng = np.random.default_rng(7)
    a = rng.standard_normal((m, k)).astype(np.float32)
    b = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    r3, r1 = rule_ratio(gemm_3xtf32(a, b), a, b), rule_ratio(gemm_1xtf32(a, b), a, b)
    assert r3 < 0.5, (name, r3)
    assert r1 > 4.0, (name, r1)


def test_tf32_rna_rounding():
    # 1 + 2^-11 is the tie between 1 and 1 + 2^-10: away from zero; just below it rounds down; signs are symmetric
    x = np.array([1 + 2.0**-11, 1 + 2.0**-11 - 2.0**-20, -(1 + 2.0**-11), 3.0], dtype=np.float32)
    np.testing.assert_array_equal(tf32_rna(x), np.array([1 + 2.0**-10, 1.0, -(1 + 2.0**-10), 3.0], dtype=np.float32))
