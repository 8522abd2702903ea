"""Tensor-core operand self-tests (K-major / MN-major views of the row layout, row shifts; col_off has no effect)."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightning_pose_b200._lib import check, lib  # noqa: E402

dev = torch.device("cuda:0")
p = lambda t: C.c_void_p(t.data_ptr())


def to_layout(x):  # (rows, ch) -> [ch/8][rows][8] bf16
    rows, ch = x.shape
    return x.reshape(rows, ch // 8, 8).permute(1, 0, 2).contiguous().bfloat16()


def run(mode, a, b, n, k, row_shift=0, col_off=0):
    la, lb = to_layout(a).to(dev), to_layout(b).to(dev)
    d = torch.zeros(128, n, device=dev)
    check(lib.lpb_selftest_umma(p(la), la.shape[0], la.shape[1], p(lb), lb.shape[0], lb.shape[1], mode, n, k, row_shift, col_off, p(d), None))
    torch.cuda.synchronize()
    af, bf = a.bfloat16().float(), b.bfloat16().float()
    if mode == 0:
        ref = af[row_shift : row_shift + 128, :k] @ bf[:n, :k].T
    else:
        ref = af[row_shift : row_shift + k, :128].T @ bf[:k, :n]
    err = (d.cpu() - ref).abs().max().item() / ref.abs().max().item()
    return err


torch.manual_seed(0)
cases = [
    ("K-major N=80 K=32", dict(mode=0, a=torch.randn(160, 32), b=torch.randn(80, 32), n=80, k=32)),
    ("K-major row_shift=7", dict(mode=0, a=torch.randn(160, 32), b=torch.randn(80, 32), n=80, k=32, row_shift=7)),
    ("K-major N=48 col_off=32", dict(mode=0, a=torch.randn(160, 32), b=torch.randn(48, 32), n=48, k=32, col_off=32)),
    ("K-major N=48 col_off=40 (unaligned)", dict(mode=0, a=torch.randn(160, 32), b=torch.randn(48, 32), n=48, k=32, col_off=40)),
    ("MN-major M=128 N=32 K=64", dict(mode=1, a=torch.randn(64, 128), b=torch.randn(64, 32), n=32, k=64)),
    ("MN-major M=128 N=96 K=208", dict(mode=1, a=torch.randn(208, 128), b=torch.randn(208, 96), n=96, k=208)),
    ("MN-major row_shift=5", dict(mode=1, a=torch.randn(80, 128), b=torch.randn(64, 32), n=32, k=64, row_shift=5)),
]
only = os.environ.get("ST_ONLY")
for i, (name, kw) in enumerate(cases):
    if only is not None and str(i) not in only.split(","):
        continue
    err = run(**kw)
    print(f"case {i}: {name}: rel err {err:.3e} {'PASS' if err < 2e-2 else 'FAIL'}", flush=True)
