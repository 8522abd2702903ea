"""Bring-up check of the tensor-core head backward: every gradient vs torch autograd (fp32 math on bf16-rounded
operands, same mid rounding as the forward kernel).  Run on the GPU box: python scripts/test_head_bwd_bf16.py"""
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from lightning_pose_b200 import ops  # noqa: E402


def run(B, C, H, W, K, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    feat = torch.randn(B, C, H, W, device="cuda", generator=g).bfloat16()
    w1 = torch.randn(C // 4, K, 3, 3, device="cuda", generator=g) * 0.05
    b1 = torch.randn(K, device="cuda", generator=g) * 0.1
    w2 = torch.randn(K, K, 3, 3, device="cuda", generator=g) * 0.2
    b2 = torch.randn(K, device="cuda", generator=g) * 0.1
    gl = torch.randn(B, K, 8 * H, 8 * W, device="cuda", generator=g)
    out, saved = ops._head_forward_bf16(feat, [w1, w2], [b1, b2], False, train=True)
    assert saved is not None
    torch.cuda.synchronize()
    t0 = time.time()
    dfeat, dw1, db1, dw2, db2 = ops.head_backward_bf16(gl, saved, feat.shape, w1, w2)
    torch.cuda.synchronize()
    print(f"B={B} bwd first call {1e3 * (time.time() - t0):.1f} ms")
    # reference: fp32 autograd with the kernel's operand roundings (bf16 weights, bf16 mid, bf16 gradients)
    r = lambda t: t.bfloat16().float()
    f32 = feat.float().requires_grad_(True)
    w1r, w2r = r(w1).requires_grad_(True), r(w2).requires_grad_(True)
    b1r, b2r = b1.clone().requires_grad_(True), b2.clone().requires_grad_(True)
    xs = F.pixel_shuffle(f32, 2)
    mid = F.conv_transpose2d(xs, w1r, b1r, stride=2, padding=1, output_padding=1)
    mid_r = (r(mid) - mid).detach() + mid  # straight-through bf16 rounding of the stored activations
    y = F.conv_transpose2d(mid_r, w2r, b2r, stride=2, padding=1, output_padding=1)
    glr = r(gl)
    y.backward(glr)
    ok = True
    for name, got, ref in [("dfeat", dfeat.float(), f32.grad), ("dw1", dw1, w1r.grad), ("db1", db1, b1r.grad),
                           ("dw2", dw2, w2r.grad), ("db2", db2, b2r.grad)]:
        err = (got - ref).abs().max().item()
        scale = ref.abs().max().item()
        rel = err / max(scale, 1e-30)
        good = rel < 2e-2
        ok &= good
        print(f"  {name:6s} max|err| {err:.3e}  max|ref| {scale:.3e}  rel {rel:.2e}  {'ok' if good else 'FAIL'}")
    fwd_ref = y.detach()
    print(f"  fwd    rel {((out - fwd_ref).abs().max() / fwd_ref.abs().max()).item():.2e}")
    return ok


if __name__ == "__main__":
    ok = run(2, 2048, 12, 12, 17)
    ok &= run(5, 2048, 12, 12, 17, seed=1)
    ok &= run(300, 2048, 12, 12, 17, seed=2)
    if ok:
        B = 768
        feat = torch.randn(B, 2048, 12, 12, device="cuda").bfloat16()
        w1 = torch.randn(512, 17, 3, 3, device="cuda") * 0.05
        w2 = torch.randn(17, 17, 3, 3, device="cuda") * 0.2
        b = torch.zeros(17, device="cuda")
        gl = torch.randn(B, 17, 96, 96, device="cuda")
        out, saved = ops._head_forward_bf16(feat, [w1, w2], [b, b], False, train=True)
        for _ in range(3):
            ops.head_backward_bf16(gl, saved, feat.shape, w1, w2)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.head_backward_bf16(gl, saved, feat.shape, w1, w2)
        e1.record()
        torch.cuda.synchronize()
        print(f"B=768 head backward {e0.elapsed_time(e1) / 10:.3f} ms")
    print("ALL PASS" if ok else "FAILED")
    sys.exit(0 if ok else 1)
