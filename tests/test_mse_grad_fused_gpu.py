"""The keypoint-target MSE's gradient stays implicit into the bf16 head's backward (lpb_head_bwd_bf16_targets): the head's
gradients are bit-identical to those of the same backward fed the dense gradient, and every other consumer of the
gradient gets exactly the dense tensor (ops.MseKeypointGrad).  The ABI test at the end needs no GPU."""
import ctypes
import os
import sys

import pytest
import torch

from head_support import features, make_head

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMG = 384.0


def labels(b, k, seed, oh, ow):
    """Keypoints in image pixels with NaN rows (dropped planes), visibility 0 / 1 / 2 (zero, uniform and Gaussian
    targets), a few far outside the image (dropped when visibility is 2)."""
    g = torch.Generator().manual_seed(seed)
    kp = torch.rand(b, k, 2, generator=g) * (IMG * 1.1) - IMG * 0.05
    kp[torch.rand(b, k, generator=g) < 0.1] = float("nan")
    vis = torch.randint(0, 3, (b, k), generator=g, dtype=torch.int32)
    return kp.cuda(), vis.cuda()


def mse(kp, vis, hm):
    from lightning_pose_b200 import ops

    return ops.heatmap_mse_from_keypoints(kp, hm, IMG, IMG, visibility=vis)


def dense_grad(kp, vis, hm, upstream=1.0):
    """The dense kernel's d loss / d hm (lpb_heatmap_mse_from_keypoints_bwd), called directly."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200._lib import check, lib

    b, k, oh, ow = hm.shape
    hm = hm.detach()
    out = torch.empty(2, device="cuda")
    ws = torch.empty(b * k * 2, device="cuda")
    gg = torch.full((1,), upstream, device="cuda")
    gp = torch.empty_like(hm)
    check(lib.lpb_heatmap_mse_from_keypoints_fwd(ops._ptr(kp), ops._ptr(vis), ops._ptr(hm), b * k, IMG, IMG, oh, ow, 1.25, ops._ptr(out), ops._ptr(ws), ops._stream()))
    check(lib.lpb_heatmap_mse_from_keypoints_bwd(ops._ptr(kp), ops._ptr(vis), ops._ptr(hm), b * k, IMG, IMG, oh, ow, 1.25, ops._ptr(out), ops._ptr(gg), ops._ptr(gp), ops._stream()))
    return gp


def head_grads(head, f, hm, g):
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    return [t.clone() for t in torch.autograd.grad(hm, [f] + params, g, retain_graph=True)]


def assert_bitwise(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape and x.stride() == y.stride(), i
        assert torch.equal(x.view(torch.int16 if x.element_size() == 2 else torch.int32), y.view(torch.int16 if y.element_size() == 2 else torch.int32)), i


CASES = [  # (C, H, W, channels, frames, channels-last features)
    (2048, 12, 12, (17, 17), 256, False),  # config 2 at the bench's labeled batch
    (2048, 12, 12, (51, 51), 32, False),   # keypoint groups
    (2048, 12, 12, (17, 17), 32, True),    # channels-last features
    (384, 16, 16, (17,), 32, False),       # one deconv
]


@pytest.mark.gpu
@pytest.mark.parametrize("c,h,w,channels,b,nhwc", CASES)
def test_implicit_gradient_matches_dense(c, h, w, channels, b, nhwc):
    from lightning_pose_b200 import ops

    head = make_head(c, channels, seed=3)
    f = features(b, c, h, w, seed=4, dtype=torch.bfloat16)
    if nhwc:
        f = f.contiguous(memory_format=torch.channels_last)
    f.requires_grad_(True)
    hm = head(f)
    kp, vis = labels(b, channels[-1], 5, hm.shape[2], hm.shape[3])
    loss = mse(kp, vis, hm)
    g = torch.autograd.grad(loss, hm, retain_graph=True)[0]
    assert isinstance(g, ops.MseKeypointGrad)
    implicit = head_grads(head, f, hm, g)
    assert g.dense is None, "the head backward materialised the gradient"
    dense = head_grads(head, f, hm, g.materialize().clone())
    assert_bitwise(implicit, dense)


@pytest.mark.gpu
def test_autograd_grad_returns_the_dense_gradient():
    head = make_head(2048, (17, 17), seed=6)
    f = features(8, 2048, 12, 12, seed=7, dtype=torch.bfloat16)
    hm = head(f)
    kp, vis = labels(8, 17, 8, 96, 96)
    loss = mse(kp, vis, hm) * 0.5
    (g,) = torch.autograd.grad(loss, hm)
    ref = dense_grad(kp, vis, hm, upstream=0.5)
    assert torch.equal(g, ref)
    assert torch.equal(g * 1, ref) and type(g * 1) is torch.Tensor
    assert torch.equal(g.cpu(), ref.cpu())


@pytest.mark.gpu
def test_second_loss_on_the_heatmaps_adds_up():
    head = make_head(2048, (17, 17), seed=9)
    f = features(16, 2048, 12, 12, seed=10, dtype=torch.bfloat16).requires_grad_(True)
    hm = head(f)
    kp, vis = labels(16, 17, 11, 96, 96)
    wt = torch.randn(hm.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12)) * 1e-3
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    got = torch.autograd.grad(mse(kp, vis, hm) + (hm * wt).sum(), [f] + params, retain_graph=True)
    want = head_grads(head, f, hm, dense_grad(kp, vis, hm) + wt)
    assert_bitwise(list(got), want)


@pytest.mark.gpu
def test_retain_graph_two_backwards():
    head = make_head(2048, (17, 17), seed=13)
    f = features(16, 2048, 12, 12, seed=14, dtype=torch.bfloat16).requires_grad_(True)
    hm = head(f)
    kp, vis = labels(16, 17, 15, 96, 96)
    loss = mse(kp, vis, hm)
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    first = torch.autograd.grad(loss, [f] + params, retain_graph=True)
    want = head_grads(head, f, hm, dense_grad(kp, vis, hm))
    second = torch.autograd.grad(loss, [f] + params)
    assert_bitwise(list(first), want)
    assert_bitwise(list(second), want)


@pytest.mark.gpu
def test_fp32_head_takes_the_dense_gradient():
    head = make_head(2048, (17, 17), seed=16)
    f = features(4, 2048, 12, 12, seed=17, dtype=torch.float32).requires_grad_(True)
    hm = head(f)
    kp, vis = labels(4, 17, 18, 96, 96)
    params = [p for d in list(head.upsampling_layers)[1:] for p in (d.weight, d.bias)]
    got = torch.autograd.grad(mse(kp, vis, hm), [f] + params, retain_graph=True)
    want = head_grads(head, f, hm, dense_grad(kp, vis, hm))
    # the data gradient is bit-identical; the fp32 route adds its weight gradients with float atomics (DESIGN.md K4), and
    # layer 2's bias gradient is zero in exact arithmetic under the softmax, so both sides hold rounding noise there
    assert_bitwise(list(got[:1]), want[:1])
    for x, y in zip(got[1:4], want[1:4]):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-5 * float(y.abs().max()))
    scale = float(want[3].abs().max())
    assert float(got[4].abs().max()) <= 1e-4 * scale and float(want[4].abs().max()) <= 1e-4 * scale


@pytest.mark.gpu
def test_labeled_step_in_a_cuda_graph():
    head = make_head(2048, (17, 17), seed=19)
    f = features(64, 2048, 12, 12, seed=20, dtype=torch.bfloat16)
    kp, vis = labels(64, 17, 21, 96, 96)

    def step():
        head.zero_grad(set_to_none=True)
        fr = f.detach().requires_grad_(True)
        hm, _, _ = head.forward_with_keypoints(fr)
        (0.5 * mse(kp, vis, hm)).backward()
        return [fr.grad] + [p.grad for p in head.parameters()]

    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert_bitwise([t.clone() for t in out], eager)


@pytest.mark.gpu
def test_bench_labeled_step_writes_no_dense_gradient():
    """The benchmark's training step (two streams): the labeled chain launches no dense MSE backward, and the only
    allocation of a labeled heatmap tensor's size is the heatmaps themselves."""
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, ROOT)
    import bench

    dev = torch.device("cuda")
    prob = bench.make_problem(16, seed=1234, device=dev)
    hp = bench.HotPath(prob, dev, fwd_only=False)
    feats = prob["feats"].to(torch.bfloat16).to(dev)
    hp.step(feats)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hp.step(feats)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not any("heatmap_mse_from_kp_bwd_kernel" in n for n in names)
    assert any("plane_dot_targets_kernel" in n for n in names)
    # the caching allocator's trace of one step: a labeled heatmap tensor's size is allocated once (the heatmaps)
    torch.cuda.memory._record_memory_history(max_entries=100000)
    try:
        hp.step(feats)
        torch.cuda.synchronize()
        snap = torch.cuda.memory._snapshot()
    finally:
        torch.cuda.memory._record_memory_history(enabled=None)
    labeled = 16 * bench.B_LABELED * bench.K_PTS * bench.HM * bench.HM * 4
    allocs = [e["size"] for trace in snap["device_traces"] for e in trace if e["action"] == "alloc"]
    assert allocs, "the allocator recorded no allocations"
    assert allocs.count(labeled) == 1, allocs.count(labeled)


def test_targets_entry_refusals_without_gpu():
    """lpb_head_bwd_bf16_targets: NULL descriptor is the _layout entry; a descriptor refuses a dense gradient beside it,
    a head without probs, null pointers and a bad geometry, all before anything is queued; the workspace grows by the
    per-plane factor rows only when targets are asked for."""
    from lightning_pose_b200._lib import MseTargets, lib

    n0, n1, n2 = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert lib.lpb_head_bwd_bf16_workspace_bytes_layout(3, 2048, 12, 12, 17, 17, 0, ctypes.byref(n0)) == 0
    assert lib.lpb_head_bwd_bf16_workspace_bytes_targets(3, 2048, 12, 12, 17, 17, 0, 0, ctypes.byref(n1)) == 0
    assert lib.lpb_head_bwd_bf16_workspace_bytes_targets(3, 2048, 12, 12, 17, 17, 0, 1, ctypes.byref(n2)) == 0
    assert n1.value == n0.value
    assert n2.value - n0.value >= 3 * 17 * (4 + 96 + 96) * 4
    assert n2.value - n0.value < 3 * 17 * (4 + 96 + 96) * 4 + 256
    assert lib.lpb_head_bwd_bf16_workspace_bytes_targets(3, 2048, 13, 12, 17, 17, 0, 1, ctypes.byref(n2)) == -3

    fake = 0x1000
    good = MseTargets(fake, None, IMG, IMG, 1.25, fake, fake)

    def call(g_out, desc, probs):
        return lib.lpb_head_bwd_bf16_targets(g_out, desc, probs, None, None, None, fake, fake, 3, 2048, 12, 12, fake, 17, fake, 17, 0,
                                             fake, fake, fake, fake, fake, fake, None)

    cases = [
        (fake, ctypes.byref(good), fake, b"g_out must be null"),
        (None, ctypes.byref(good), None, b"need the softmax head's output"),
        (None, ctypes.byref(MseTargets(None, None, IMG, IMG, 1.25, fake, fake)), fake, b"keypoint targets: null pointer"),
        (None, ctypes.byref(MseTargets(fake, None, IMG, IMG, 1.25, fake, None)), fake, b"keypoint targets: null pointer"),
        (None, ctypes.byref(MseTargets(fake, None, IMG, 0.0, 1.25, fake, fake)), fake, b"bad image size or sigma"),
        (None, ctypes.byref(MseTargets(fake, None, IMG, IMG, -1.0, fake, fake)), fake, b"bad image size or sigma"),
        (None, None, fake, b"neither a dense gradient nor decode windows"),
    ]
    for g_out, desc, probs, msg in cases:
        assert call(g_out, desc, probs) == -1, msg
        assert msg in lib.lpb_last_error(), (msg, lib.lpb_last_error())
