"""Bit-reproducible training on every route: the fp32 head's weight and bias gradients, the dense decode backward (whole
planes and queue-mode segments), the bf16 head's fused backward on fresh-init (flat) heatmaps, and the context head's
combine backward.

* The fp32 head's gradients must equal, under torch.equal, the sequential fp32 sum of the workspace's partial slots in
  slot order (the method of test_head_bwd_sums_gpu.py).
* Each route is run 20 times; every other run has unrelated kernels on a second stream, which changes how CTAs are
  scheduled.  Every run must give the same bits.
* Two training steps of each tracker, from the same seed and state, must give the same bits in every parameter gradient
  and loss scalar.

The gradients' accuracy against float64 is held by the existing tests of each route (test_f32_convt_gpu.py,
test_scale_gpu.py, test_targets_edges_gpu.py, test_context_train_gpu.py), which run the same entries.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from head_support import gen

RUNS = 20


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


def seq_sum(rows: np.ndarray) -> np.ndarray:
    """[partials, n] float32 -> the partials added one after another (np.add.accumulate adds sequentially)"""
    return np.add.accumulate(rows, axis=0, dtype=np.float32)[-1]


def repeat_under_load(fn, dev):
    """fn() -> tuple of tensors, RUNS times; odd runs with matrix products queued on a second stream first, so that
    the two streams' kernels share the SMs.  Returns the results of every run (cloned)."""
    side = torch.cuda.Stream(device=dev)
    a = torch.randn(2048, 2048, device=dev)
    torch.cuda.synchronize(dev)
    out = []
    for r in range(RUNS):
        if r % 2:
            with torch.cuda.stream(side):
                for _ in range(r % 5 + 1):
                    a = (a @ a).clamp_(-1, 1)
        out.append(tuple(t.clone() for t in fn()))
        torch.cuda.synchronize(dev)
    return out


def assert_all_equal(results, case):
    first = results[0]
    distinct = 1 + sum(any(not torch.equal(x, y) for x, y in zip(first, res)) for res in results[1:])
    assert distinct == 1, f"{case}: {distinct} of {len(results)} runs differ from the first"


# ------------------------------------------------------------------------------------------------
# fp32 head: weight / bias gradient partials summed in slot order
# ------------------------------------------------------------------------------------------------
# (case, B, Cin, Hi, Wi, Cout, shuffle): config 2's layers (ResNet-50 (B, 2048, 12, 12) -> 96x96, 17 keypoints), a ViT-S
# one-deconv layer ((B, 384, 16, 16) -> 64x64), the mirror-fish 51-keypoint layers, the third layer of a three-deconv head,
# and the first layer reading channels-last features
F32_LAYERS = [
    ("config2 L1 512->17 at 24^2", 16, 512, 24, 24, 17, 1),
    ("config2 L2 17->17 at 48^2", 16, 17, 48, 48, 17, 0),
    ("vit one-deconv 96->17 at 32^2", 16, 96, 32, 32, 17, 1),
    ("mirror-fish L1 512->51 at 24^2", 8, 512, 24, 24, 51, 1),
    ("mirror-fish L2 51->51 at 48^2", 8, 51, 48, 48, 51, 0),
    ("three-deconv L3 17->17 at 96^2", 4, 17, 96, 96, 17, 0),
    ("config2 L1 channels-last", 16, 512, 24, 24, 17, 2),
]


def _f32_inputs(b, cin, hi, wi, cout, shuffle, dev, seed):
    g = gen(seed)
    if shuffle:
        x = torch.randn(b, 4 * cin, hi // 2, wi // 2, device=dev, generator=g) * 0.5
        if shuffle == 2:
            x = x.contiguous(memory_format=torch.channels_last)
    else:
        x = torch.randn(b, cin, hi, wi, device=dev, generator=g) * 0.5
    gout = torch.randn(b, cout, 2 * hi, 2 * wi, device=dev, generator=g)
    w = torch.randn(cin, cout, 3, 3, device=dev, generator=g) * 0.05
    return x, gout, w


@pytest.mark.gpu
@pytest.mark.parametrize("case,b,cin,hi,wi,cout,shuffle", F32_LAYERS, ids=[c[0] for c in F32_LAYERS])
def test_f32_wgrad_sums_partials_in_slot_order(dev, case, b, cin, hi, wi, cout, shuffle):
    from lightning_pose_b200 import _lib

    x, gout, w = _f32_inputs(b, cin, hi, wi, cout, shuffle, dev, seed=31)
    nbytes = C.c_size_t(0)
    _lib.check(_lib.lib.lpb_convt_bwd_f32_workspace_bytes(b, cin, hi, wi, cout, C.byref(nbytes)))
    stride = cin * cout * 9 + cout
    ws = torch.full((nbytes.value // 4,), float("nan"), device=dev)  # slots the launch leaves unused stay NaN
    dw, db = torch.empty_like(w), torch.empty(cout, device=dev)
    _lib.check(_lib.lib.lpb_convt_bwd_f32_ws(x.data_ptr(), gout.data_ptr(), b, cin, hi, wi, shuffle, w.data_ptr(), cout, None,
                                             dw.data_ptr(), db.data_ptr(), ws.data_ptr(), nbytes.value,
                                             torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    part = ws.view(-1, stride).cpu().numpy()
    used = int(np.argmin(~np.isnan(part).any(axis=1))) if np.isnan(part).any() else part.shape[0]
    assert used >= 2, f"{case}: {used} K-split slot(s); the batch should give several"
    assert not np.isnan(part[:used]).any()
    nw = cin * cout * 9
    assert torch.equal(dw.cpu().reshape(-1), torch.from_numpy(seq_sum(part[:used, :nw]))), case
    assert torch.equal(db.cpu(), torch.from_numpy(seq_sum(part[:used, nw:]))), case


@pytest.mark.gpu
@pytest.mark.parametrize("case,b,cin,hi,wi,cout,shuffle", [F32_LAYERS[0], F32_LAYERS[1], F32_LAYERS[6]],
                         ids=[F32_LAYERS[i][0] for i in (0, 1, 6)])
def test_f32_head_backward_repeats(dev, case, b, cin, hi, wi, cout, shuffle):
    from lightning_pose_b200 import ops

    x, gout, w = _f32_inputs(b, cin, hi, wi, cout, shuffle, dev, seed=32)
    assert_all_equal(repeat_under_load(lambda: ops.convt_backward_f32(x, gout, w, bool(shuffle)), dev), case)


# ------------------------------------------------------------------------------------------------
# dense decode backward
# ------------------------------------------------------------------------------------------------
def _planes(n, h, w, n_flat, dev, seed):
    """n planes of softmax heatmaps: the first n_flat nearly flat (fresh-init), the rest one sharp peak each"""
    g = gen(seed)
    logits = torch.randn(n, h * w, device=dev, generator=g) * 0.01
    yy, xx = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
    cy = torch.rand(n, 1, device=dev, generator=g) * (h - 8) + 4
    cx = torch.rand(n, 1, device=dev, generator=g) * (w - 8) + 4
    peak = -((yy.reshape(1, -1) - cy) ** 2 + (xx.reshape(1, -1) - cx) ** 2) / 2.0
    logits[n_flat:] += 30.0 * peak[n_flat:].exp()
    return torch.softmax(logits, -1).reshape(1, n, h, w).contiguous()


DECODE = [(64, 64, 2), (96, 96, 2), (128, 192, 2), (64, 64, 3), (96, 96, 3), (64, 64, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,ds", DECODE, ids=[f"{h}x{w}-ds{ds}" for h, w, ds in DECODE])
@pytest.mark.parametrize("mix", ["flat", "mixed"])
def test_decode_backward_repeats(dev, h, w, ds, mix):
    """flat: every plane dense (one CTA per plane, and queue mode with the queue filling the grid); mixed: a few flat
    planes among peaked ones, so queue mode splits each over several row segments"""
    from lightning_pose_b200 import ops

    n = 272
    hm = _planes(n, h, w, n if mix == "flat" else 12, dev, seed=41 + h + ds)
    xy, conf, stats = ops.decode_forward(hm, ds, 1000.0)
    gxy = torch.randn(1, n, 2, device=dev, generator=gen(42))
    flag = None

    def run():
        nonlocal flag
        dense = ops._decode_bwd(hm, stats, gxy, ds, 1000.0)
        win, meta, ov = ops.decode_backward_windows(hm, stats, gxy, ds, 1000.0)
        flag = meta[:, 2]
        over = ov.reshape(n, h, w)[flag == 2]
        return dense, win[flag == 1], meta, over

    res = repeat_under_load(run, dev)
    n_over = int((flag == 2).sum())
    assert n_over == (n if mix == "flat" else 12), n_over
    assert_all_equal(res, f"decode {h}x{w} ds {ds} {mix}")


# ------------------------------------------------------------------------------------------------
# bf16 head fused backward on fresh-init heatmaps
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bf16_head_fresh_backward_repeats(dev):
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    torch.manual_seed(5)
    head = HeatmapHead("resnet50", 2048, 17)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=0.01)
        torch.nn.init.zeros_(layer.bias)
    head = head.to(dev)
    feats = (torch.randn(16, 2048, 12, 12, device=dev, generator=gen(51)) * 0.5).bfloat16()
    g_kp = torch.randn(16, 34, device=dev, generator=gen(52))

    def run():
        f = feats.clone().requires_grad_(True)
        head.zero_grad(set_to_none=True)
        hm, kp, cf = head.forward_with_keypoints(f)
        (kp * g_kp).sum().backward()
        return (f.grad, *[p.grad for p in head.parameters() if p.grad is not None])

    assert_all_equal(repeat_under_load(run, dev), "bf16 head, fresh init")


# ------------------------------------------------------------------------------------------------
# context combine backward
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["sequence", "call"])
def test_crnn_combine_backward_repeats(dev, form):
    from lightning_pose_b200 import ops

    k, h, w = 17, 96, 96
    g = gen(61)
    if form == "sequence":  # config 3's unlabeled chunk: 32 frames, 28 overlapping windows
        n = 32
        idx = torch.arange(n - 4, device=dev)[:, None] + torch.arange(5, device=dev)[None, :]
    else:  # reference call form on a labeled batch of 16: windows share no frames
        b = 16
        n = 5 * b
        idx = torch.arange(5, device=dev)[None, :] * b + torch.arange(b, device=dev)[:, None]
    idx = idx.to(torch.int32)
    wf = torch.randn(n, k, h, w, device=dev, generator=g)
    wb = torch.randn(n, k, h, w, device=dev, generator=g)
    ps = []
    for _ in range(2):
        ps.append((torch.randn(16 * k, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(16 * k, device=dev, generator=g) * 0.1,
                   torch.randn(16 * k, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(k, device=dev, generator=g) * 0.1))
    gout = torch.randn(idx.shape[0], k, h, w, device=dev, generator=g)

    def run():
        leaves = [t.clone().requires_grad_(True) for t in (wf, wb, *ps[0], *ps[1])]
        out = ops.crnn_combine(leaves[0], leaves[1], idx, tuple(leaves[2:6]), tuple(leaves[6:10]))
        return torch.autograd.grad(out, leaves, gout)

    assert_all_equal(repeat_under_load(run, dev), f"crnn combine, {form} form")


@pytest.mark.gpu
def test_crnn_combine_backward_any_table(dev):
    """A table with repeated frames, inside one window and across windows (the clamped edges of
    get_context_from_sequence, and a window of one frame): the fixed-order form equals the atomic form's result to
    float32 rounding, and repeats bit for bit."""
    from lightning_pose_b200 import ops

    k, h, w, n = 3, 8, 8, 6
    idx = torch.tensor([[0, 0, 0, 1, 2], [0, 0, 1, 2, 3], [1, 2, 3, 4, 5], [3, 4, 5, 5, 5], [2, 2, 2, 2, 2]], dtype=torch.int32, device=dev)
    g = gen(71)
    wf, wb = torch.randn(n, k, h, w, device=dev, generator=g), torch.randn(n, k, h, w, device=dev, generator=g)
    ps = [(torch.randn(16 * k, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(16 * k, device=dev, generator=g) * 0.1,
           torch.randn(16 * k, 1, 2, 2, device=dev, generator=g) * 0.3, torch.randn(k, device=dev, generator=g) * 0.1) for _ in range(2)]
    gout = torch.randn(idx.shape[0], k, h, w, device=dev, generator=g)

    def run():
        leaves = [t.clone().requires_grad_(True) for t in (wf, wb)]
        out = ops.crnn_combine(leaves[0], leaves[1], idx, ps[0], ps[1])
        return torch.autograd.grad(out, leaves, gout)

    res = repeat_under_load(run, dev)
    assert_all_equal(res, "crnn combine, repeated frames")
    # float64 restatement: d/dWF[f] = sum over pairs (m, s) of (L^T)^(4 - s) 0.5 g[m] (forward), mirrored backward
    from test_context_train_gpu import _block_affine, _combine_blocks  # noqa: F401  (reference helpers of the context tests)

    leaves = [t.double().requires_grad_(True) for t in (wf, wb)]
    lf, lb = _block_affine([t.double() for t in ps[0]], k), _block_affine([t.double() for t in ps[1]], k)
    ref = torch.autograd.grad(_combine_blocks(leaves[0], leaves[1], idx.long(), lf, lb), leaves, gout.double())
    for got, want in zip(res[0], ref):
        assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-5 * float(want.abs().max()))


# ------------------------------------------------------------------------------------------------
# end to end: two training steps from the same seed and state
# ------------------------------------------------------------------------------------------------
class _Backbone(torch.nn.Module):
    """Deterministic stand-in backbone: a strided convolution (its backward has no float atomics in cuDNN's
    deterministic mode, which the test sets) to (n, C, h, w) in the given dtype."""

    def __init__(self, c, patch, dtype):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, c, patch, stride=patch)
        self.dtype = dtype

    def forward(self, x):
        return self.conv(x).to(self.dtype)


def _two_steps(make, batch):
    results = []
    for _ in range(2):
        tr = make()
        tr.zero_grad(set_to_none=True)
        out = tr.training_step(batch, 0)
        out["loss"].backward()
        torch.cuda.synchronize()
        logs = [getattr(tr, name, None) for name in ("last_logs", "last_logs_unsup")]
        scalars = [out["loss"].detach().clone()] + [v.detach().clone() for v in torch.utils._pytree.tree_leaves(logs) if torch.is_tensor(v)]
        grads = [p.grad.clone() for p in tr.parameters() if p.grad is not None]
        results.append((*scalars, *grads))
    return results


@pytest.fixture
def deterministic_cudnn():
    old = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = old


@pytest.mark.gpu
def test_tracker_fp32_fresh_training_step_repeats(dev, deterministic_cudnn):
    """SemiSupervisedHeatmapTracker on fp32 features with the reference's initialiser (flat heatmaps: the dense decode
    backward on every plane), heatmap MSE + temporal + PCA-free unsupervised loss"""
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker import SemiSupervisedHeatmapTracker

    k, b, t = 17, 8, 16

    def make():
        torch.manual_seed(7)
        tr = SemiSupervisedHeatmapTracker(
            k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
            loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": 0.0, "epsilon": 1.0, "prob_threshold": 0.0}}, None),
            backbone=_Backbone(2048, 32, torch.float32), backbone_arch="resnet50", num_fc_input_features=2048, torch_seed=7).to(dev)
        return tr

    g = gen(81)
    kp = torch.rand(b, k, 2, device=dev, generator=g) * 384
    from lightning_pose_b200 import ops

    batch = {"labeled": {"images": torch.randn(b, 3, 384, 384, device=dev, generator=g), "keypoints": kp.reshape(b, 2 * k),
                         "heatmaps": ops.generate_heatmaps(kp, 384, 384, (96, 96)),
                         "bbox": torch.tensor([[0.0, 0.0, 384.0, 384.0]], device=dev).repeat(b, 1)},
             "unlabeled": {"frames": torch.randn(t, 3, 384, 384, device=dev, generator=g), "transforms": torch.tensor([-1.0], device=dev),
                           "bbox": torch.tensor([[0.0, 0.0, 384.0, 384.0]], device=dev).repeat(t, 1), "is_multiview": False}}
    assert_all_equal(_two_steps(make, batch), "SemiSupervisedHeatmapTracker fp32, fresh init")


@pytest.mark.gpu
def test_tracker_mhcrnn_training_step_repeats(dev, deterministic_cudnn):
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import SemiSupervisedHeatmapTrackerMHCRNN

    k, b, t = 17, 2, 9

    def make():
        torch.manual_seed(9)
        return SemiSupervisedHeatmapTrackerMHCRNN(
            k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
            loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": 0.5, "epsilon": 1.0, "prob_threshold": 0.0}}, None),
            backbone=_Backbone(384, 16, torch.bfloat16), backbone_arch="vits_dino", num_fc_input_features=384, torch_seed=9).to(dev)

    from lightning_pose_b200 import ops

    g = gen(91)
    kp = torch.rand(b, k, 2, device=dev, generator=g) * 256
    batch = {"labeled": {"images": torch.randn(b, 5, 3, 256, 256, device=dev, generator=g), "keypoints": kp.reshape(b, 2 * k),
                         "heatmaps": ops.generate_heatmaps(kp, 256, 256, (64, 64)),
                         "bbox": torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=dev).repeat(b, 1)},
             "unlabeled": {"frames": torch.randn(t, 3, 256, 256, device=dev, generator=g), "transforms": torch.tensor([-1.0], device=dev),
                           "bbox": torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=dev).repeat(t, 1), "is_multiview": False}}
    assert_all_equal(_two_steps(make, batch), "SemiSupervisedHeatmapTrackerMHCRNN")
