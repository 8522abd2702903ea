"""Stand-alone check of the tensor-core head (run under `timeout`): compares the intermediate activations
(k1a) and the final heatmaps (k1b) with the oracle on identically bf16-rounded tensors."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch.nn.functional as F  # noqa: E402

from lightning_pose_b200._lib import check, lib  # noqa: E402

torch.manual_seed(0)
dev = torch.device("cuda:0")
B, Cf, H, W, K = int(os.environ.get("HB_B", 3)), 2048, 12, 12, 17
gain = 3.0
w1 = (torch.rand(Cf // 4, K, 3, 3) * 2 - 1) * gain * (6 / (K * 9 + Cf // 4 * 9)) ** 0.5
w2 = (torch.rand(K, K, 3, 3) * 2 - 1) * gain * (6 / (K * 18)) ** 0.5
b1, b2 = torch.rand(K) - 0.5, torch.rand(K) - 0.5
feats = (torch.randn(B, Cf, H, W) * 0.5).bfloat16()

r = lambda t: t.bfloat16().float()
x = F.pixel_shuffle(feats.float(), 2)
mid_ref = F.conv_transpose2d(x, r(w1), b1, stride=2, padding=1, output_padding=1)
logit_ref = F.conv_transpose2d(r(mid_ref), r(w2), b2, stride=2, padding=1, output_padding=1)
hm_ref = torch.softmax(logit_ref.reshape(B, K, -1), -1).reshape(logit_ref.shape)

nbytes = C.c_size_t(0)
check(lib.lpb_head_bf16_workspace_bytes(B, Cf, H, W, K, K, C.byref(nbytes)))
ws = torch.zeros(nbytes.value, dtype=torch.uint8, device=dev)
out = torch.zeros(B, K, 96, 96, device=dev)
args = [t.to(dev).contiguous() for t in (feats, w1, b1, w2, b2)]
p = lambda t: C.c_void_p(t.data_ptr())
for softmax in (0, 1):
    check(lib.lpb_head_fwd_bf16(p(args[0]), B, Cf, H, W, p(args[1]), p(args[2]), K, p(args[3]), p(args[4]), K, softmax, p(out), None, p(ws), None))
    torch.cuda.synchronize()
    nst = Cf // 4 // 32
    # mid lives in the padded row layout (csrc/row_layout.cuh): rows = lead + y * (Wi + 1) + x, lead = Wi + 2
    Hi, Wi = 4 * H, 4 * W
    lead, rows = Wi + 2, (Hi * (Wi + 1) + 2 * (Wi + 2) + 7) // 8 * 8
    slab = ws[(nst + 1) * 20480 :].view(torch.bfloat16).reshape(B, 4, rows, 8)
    body = slab[:, :, lead : lead + Hi * (Wi + 1)].reshape(B, 4, Hi, Wi + 1, 8)
    pads_zero = float(slab[:, :, :lead].abs().max()) == 0 and float(body[:, :, :, Wi].abs().max()) == 0 and float(slab[:, :, lead + Hi * (Wi + 1) :].abs().max()) == 0
    mid = body[:, :, :, :Wi].permute(0, 1, 4, 2, 3).reshape(B, 32, Hi, Wi).float().cpu()
    e_mid = (mid[:, :K] - mid_ref).abs().max().item()
    pad = mid[:, K + 1 :].abs().max().item()  # channel K is the constant-one channel
    ref = hm_ref if softmax else logit_ref
    o = out.cpu()
    err = (o - ref).abs().max().item()
    rel = ((o - ref).abs() / (ref.abs() + 1e-6)).max().item() if softmax else err / ref.abs().max().item()
    print(f"softmax={softmax} swap={os.environ.get('LPB_DESC_SWAP','0')}: mid max|err|={e_mid:.4g} (ref max {mid_ref.abs().max():.3g}), pad={pad:.3g}; "
          f"out max|err|={err:.4g} rel={rel:.4g} sums={o.sum((2,3)).flatten()[:3].tolist() if softmax else ''}")
    ok = e_mid < 0.05 * mid_ref.abs().max().item() and (rel < 2e-2) and pads_zero
    print("RESULT", "PASS" if ok else "FAIL")
