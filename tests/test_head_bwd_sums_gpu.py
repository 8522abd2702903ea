"""The head backward's fixed-order sums at the benchmark's chain sizes (config 2: (B, 2048, 12, 12) -> 96x96, 17 keypoints).

lpb_head_bwd_bf16 writes per-CTA partials of dW1, dW2, db2 and db1 to the tail of its workspace and adds them in a fixed
order.  Each gradient must equal, bit for bit, the sequential float32 sum of its partials in that order (slot, then bias
class): it is what keeps a training step's gradients and Adam-updated parameters the same from build to build, not only
from run to run.  Workspace layout and slot counts as in head_bwd_bf16.cu (bwd_partials_bytes, launch_wgrad, the b2d
grid).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from head_support import head_params, make_head

WG_MAX_CTAS, B2D_MAX_CTAS, GB_CLS = 132, 264, 20
C_FEAT, H_FEAT, K_PTS = 2048, 12, 17


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    from lightning_pose_b200 import _lib

    return _lib


def wgrad_slots(nkc: int, sms: int) -> tuple[int, int]:
    """(workspace slots, slots used) of a weight-gradient layer with nkc K-chunks of 8 input channels; the frame count
    of these tests is large enough that the unit cap of launch_wgrad never binds"""
    groups = nkc // (8 if nkc % 8 == 0 else 4)
    max_slots = max(1, WG_MAX_CTAS // groups)
    return max_slots, max(1, min(sms // groups, max_slots))


def seq_sum(rows: np.ndarray) -> np.ndarray:
    """[partials, n] float32 -> the partials added one after another (np.add.accumulate adds sequentially)"""
    return np.add.accumulate(rows, axis=0, dtype=np.float32)[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("b", [256, 512])
def test_head_backward_sums_partials_in_fixed_order(lib, dev, b):
    from lightning_pose_b200 import ops

    (w1, w2), (b1, b2) = head_params(make_head(C_FEAT, (K_PTS, K_PTS), seed=101 + b))
    c4, c1, c2 = w1.shape[0], w1.shape[1], w2.shape[1]
    feats = (torch.randn(b, C_FEAT, H_FEAT, H_FEAT) * 0.5).bfloat16().to(dev)
    probs, (xs, fws) = ops._head_forward_bf16(feats, [w1, w2], [b1, b2], True, train=True)
    gout = torch.randn(probs.shape).to(dev)

    nbytes = C.c_size_t(0)
    lib.check(lib.lib.lpb_head_bwd_bf16_workspace_bytes(b, C_FEAT, H_FEAT, H_FEAT, c1, c2, C.byref(nbytes)))
    ws = torch.empty((nbytes.value,), device=dev, dtype=torch.uint8)
    dw1, db1 = torch.empty_like(w1), torch.empty((c1,), device=dev)
    dw2, db2 = torch.empty_like(w2), torch.empty((c2,), device=dev)
    p = ops._ptr
    with torch.cuda.device(dev):
        lib.check(lib.lib.lpb_head_bwd_bf16(p(gout), p(probs), None, None, None, p(xs), p(fws), b, C_FEAT, H_FEAT, H_FEAT, p(w1), c1, p(w2), c2,
                                            None, p(dw1), p(db1), p(dw2), p(db2), p(ws), ops._stream()))
    torch.cuda.synchronize(dev)

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    max1, slots1 = wgrad_slots(c4 // 8, sms)
    max2, slots2 = wgrad_slots(4, sms)
    grid = min(b, 2 * sms, B2D_MAX_CTAS)
    stride1, stride2 = c4 * c1 * 9 + 4 * c1, c1 * c2 * 9 + 4 * c2
    tail = max1 * stride1 + max2 * stride2 + B2D_MAX_CTAS * 4 * GB_CLS  # floats: [layer-1 wgrad][layer-2 wgrad][b2d bias]
    part = ws[nbytes.value - 4 * tail:].view(torch.float32).cpu().numpy()
    part1 = part[:max1 * stride1].reshape(max1, stride1)[:slots1]
    part2 = part[max1 * stride1:max1 * stride1 + max2 * stride2].reshape(max2, stride2)[:slots2]
    part_db1 = part[max1 * stride1 + max2 * stride2:].reshape(B2D_MAX_CTAS * 4, GB_CLS)[:grid * 4, :c1]

    sums = {
        "dW1": (dw1, part1[:, :c4 * c1 * 9]),
        "dW2": (dw2, part2[:, :c1 * c2 * 9]),
        "db2": (db2, part2[:, c1 * c2 * 9:c1 * c2 * 9 + 4 * c2].reshape(slots2 * 4, c2)),  # slot-major, then bias class
        "db1": (db1, part_db1),
    }
    for name, (got, rows) in sums.items():
        got = got.cpu().numpy().reshape(-1)
        assert np.isfinite(rows).all(), name
        assert np.array_equal(got, seq_sum(rows)), f"{name}: not the sequential sum of its {rows.shape[0]} partials"
        # the inputs are such that the order shows in the bits (so this test pins it)
        assert not np.array_equal(got, seq_sum(rows[::-1])), name
