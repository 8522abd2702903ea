"""GPU: curriculum patch masking (csrc/patchmask.cu, lightning_pose_b200/callbacks.py) against tests/golden/patch_mask.npz
(the reference's own PatchMasker): the apply kernel bit for bit on the reference's masks, the selection's patch counts on
the reference's schedule, determinism and independence of the draws, uniformity over subsets, the no-masking cases, the
multi-view transformer's labeled step with masking and the 3-D losses replayed from a CUDA graph, and input checks."""
import numpy as np
import pytest
import torch

import patch_mask_oracle as O

pytestmark = pytest.mark.gpu

CASES = [c[0] for c in O.CASES]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lpb():
    import lightning_pose_b200  # noqa: F401  (raises if liblpb200.so is missing)
    from lightning_pose_b200 import ops

    return ops


def images_of(arr: np.ndarray, dev) -> torch.Tensor:
    if arr.dtype == np.uint16:  # bf16 bits
        return torch.from_numpy(arr.view(np.int16).copy()).view(torch.bfloat16).to(dev)
    return torch.from_numpy(arr.copy()).to(dev)


def bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().cpu()
    return t.view(torch.int16).numpy() if t.dtype == torch.bfloat16 else t.view(torch.int32).numpy()


def masker(cfg=None, seed=O.PATCH_SEED, **kw):
    from lightning_pose_b200.callbacks import PatchMasker

    return PatchMasker({**(O.CURRICULUM if cfg is None else cfg), **kw}, patch_seed=seed)


# ---- 1. apply --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_apply_reproduces_reference_masked_images_bit_for_bit(lpb, dev, golden, name):
    g = golden("patch_mask")
    x = images_of(g[f"case_{name}_in_images"], dev)
    x0 = x.clone()
    mask = torch.from_numpy(g[f"case_{name}_out_mask"]).to(dev)
    want = images_of(g[f"case_{name}_out_images"], dev)
    out = lpb.patch_mask_apply(x, mask)
    assert out.dtype == x.dtype and out.shape == x.shape and out.data_ptr() != x.data_ptr()
    np.testing.assert_array_equal(bits(out), bits(want))
    np.testing.assert_array_equal(bits(x), bits(x0))  # out of place: the input is unchanged
    # the same batch one element past a 16-byte boundary (narrower accesses)
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=dev)
    shifted = buf[1:].view(x.shape).copy_(x)
    np.testing.assert_array_equal(bits(lpb.patch_mask_apply(shifted, mask)), bits(want))


# ---- 2. selection counts ---------------------------------------------------------------------------------------------
def test_selection_masks_exactly_m_patches_on_every_schedule_row(lpb, dev, golden):
    g = golden("patch_mask")
    counts = []
    for i in range(len(g["sched_step"])):
        init_step, final_step, r0, r1 = g["sched_config"][i]
        p = int(g["sched_P"][i])
        shape_only = torch.empty((2, 3, 1, 16, 16 * p), device=dev)
        step = torch.full((1,), int(g["sched_step"][i]), dtype=torch.int64, device=dev)
        mask = lpb.patch_mask_select(shape_only, step, 5, int(init_step), int(final_step), float(r0), float(r1))
        assert mask.shape == (2, 3, p)
        counts.append((mask == 0).sum(-1))
    counts = torch.stack(counts).cpu().numpy()  # (rows, 2, 3)
    np.testing.assert_array_equal(counts, np.broadcast_to(g["sched_m"][:, None, None], counts.shape))


@pytest.mark.parametrize("name", CASES)
def test_masker_counts_match_reference_cases(lpb, dev, golden, name):
    g = golden("patch_mask")
    x = images_of(g[f"case_{name}_in_images"], dev)
    step = torch.full((1,), int(g[f"case_{name}_in_step"]), dtype=torch.int64, device=dev)
    out, mask = masker().apply_patch_masking(x, training_step=step)
    ref = g[f"case_{name}_out_mask"]
    assert mask.shape == ref.shape and mask.dtype == torch.float32
    np.testing.assert_array_equal((mask == 0).sum(-1).cpu().numpy(), (ref == 0).sum(-1))
    assert set(mask.unique().tolist()) <= {0.0, 1.0}
    np.testing.assert_array_equal(bits(out), bits(lpb.patch_mask_apply(x, mask)))


def test_selection_at_the_patch_limit(lpb, dev):
    x = torch.empty((1, 2, 1, 1024, 1024), device=dev)
    step = torch.full((1,), 30, dtype=torch.int64, device=dev)
    mask = lpb.patch_mask_select(x, step, 3, 10, 50, 0.1, 0.5)
    m = masker().patches_to_mask(30, 4096)
    assert mask.shape == (1, 2, 4096) and ((mask == 0).sum(-1) == m).all()


# ---- 3. determinism and independence -----------------------------------------------------------------------------------
def test_same_seed_and_step_same_patches_other_step_example_or_view_others(dev):
    x = torch.randn(4, 3, 3, 64, 80, device=dev)
    mk = masker()
    step = torch.full((1,), 30, dtype=torch.int64, device=dev)
    a_img, a = mk.apply_patch_masking(x, training_step=step)
    b_img, b = mk.apply_patch_masking(x, training_step=30)  # an int step is the same draw
    assert torch.equal(a, b) and torch.equal(a_img, b_img)
    flat = a.reshape(12, -1)
    assert len({tuple(r.tolist()) for r in flat}) == 12  # every (example, view) draws its own patches
    _, c = mk.apply_patch_masking(x, training_step=31)
    assert all(not torch.equal(a[i, j], c[i, j]) for i in range(4) for j in range(3))
    _, d = masker(seed=O.PATCH_SEED + 1).apply_patch_masking(x, training_step=30)
    assert all(not torch.equal(a[i, j], d[i, j]) for i in range(4) for j in range(3))
    # the reference's seed patch_seed + step + 1000 b + 100 v repeats across (step, example); these draws do not
    x2 = torch.randn(2, 1, 3, 64, 80, device=dev)
    _, e = masker(cfg={"init_step": 0, "final_step": 5000}).apply_patch_masking(x2, training_step=1000)
    _, f = masker(cfg={"init_step": 0, "final_step": 5000}).apply_patch_masking(x2, training_step=0)
    assert not torch.equal(e[0, 0], f[1, 0])


# ---- 4. uniformity ---------------------------------------------------------------------------------------------------------
def test_selection_is_uniform_over_subsets(lpb, dev):
    """P = 20, m = 5, 3200 draws (8 examples x 4 views x 100 steps): each patch is masked with probability 1/4 and each
    pair with 1/19; every frequency within 5 binomial standard deviations, and Pearson's statistic of the patch counts
    below 60 (19 degrees of freedom)."""
    x = torch.empty((8, 4, 1, 64, 80), device=dev)
    masks = []
    for s in range(100):
        step = torch.full((1,), s, dtype=torch.int64, device=dev)
        masks.append(lpb.patch_mask_select(x, step, 1234, 0, 1, 0.25, 0.25))
    z = (torch.stack(masks).reshape(-1, 20) == 0).double().cpu().numpy()  # (3200, 20), 1 = masked
    n, p = z.shape[0], 20
    assert (z.sum(1) == 5).all()
    freq = z.sum(0)
    sd = np.sqrt(n * 0.25 * 0.75)
    assert np.abs(freq - n * 0.25).max() < 5 * sd, freq
    assert (((freq - n * 0.25) ** 2) / (n * 0.25)).sum() < 60
    pair = z.T @ z
    q = 5 * 4 / (p * (p - 1))
    off = pair[~np.eye(p, dtype=bool)]
    assert np.abs(off - n * q).max() < 5 * np.sqrt(n * q * (1 - q)), off
    # distinct subsets among n uniform draws from N = C(20, 5) = 15504: mean N (1 - e^(-n / N)) = 2891, sd about 15
    big_n = 15504
    lam = n / big_n
    mean, sd_d = big_n * (1 - np.exp(-lam)), np.sqrt(big_n * np.exp(-lam) * (1 - (1 + lam) * np.exp(-lam)))
    assert abs(len({tuple(r) for r in z.astype(int)}) - mean) < 5 * sd_d


# ---- 5. no masking ------------------------------------------------------------------------------------------------------------
def test_no_masking_returns_the_input_values_and_all_ones(dev, golden):
    g = golden("patch_mask")
    x = torch.randn(2, 4, 3, 72, 88, device=dev)
    x0 = x.clone()
    same, mask = masker().apply_patch_masking(x, training_step=30, is_training=False)
    assert same is x and list(mask.shape) == g["eval_out_mask_shape"].tolist() and (mask == 1).all()
    out, mask = masker().apply_patch_masking(x, training_step=5)  # before init_step
    assert torch.equal(out, x) and out.data_ptr() != x.data_ptr() and (mask == 1).all() and mask.shape == (2, 4, 20)
    off = masker(final_ratio=0.0)
    same, mask = off.apply_masking(x, training_step=30)
    assert same is x and list(mask.shape) == g["disabled_out_mask_shape"].tolist() and (mask == 1).all()
    out, mask = masker(init_ratio=0.0, final_ratio=0.0).apply_patch_masking(x, training_step=30)
    assert torch.equal(out, x) and (mask == 1).all() and mask.shape == (2, 4, 20)
    assert torch.equal(x, x0)


# ---- 6. the multi-view transformer's training step in a CUDA graph -----------------------------------------------------------
def test_multiview_training_step_with_masking_replays_in_cuda_graph(lpb, dev):
    """Config-4 tracker (stand-in transformer), calibrated batch, heatmap MSE + both 3-D losses, patch masking from step
    0 (before init_step), 1 (init_step) and 2: three graph replays equal three eager steps."""
    from test_multiview_3d import LOSSES_3D, _calibrated_batch, _tracker

    tr, _ = _tracker(dev, LOSSES_3D)
    tr.patch_masker = masker(cfg={"init_step": 1, "final_step": 3, "init_ratio": 0.2, "final_ratio": 0.6}, seed=11)
    bd = _calibrated_batch(lpb, dev)
    images0, kp0 = bd["images"], bd["keypoints"].clone()
    params = list(tr.head.parameters()) + [tr.view_embeddings]

    def step():
        bd["images"] = images0  # training_step replaces the batch's images with the masked ones
        bd["keypoints"].copy_(kp0)  # model_to_frame_batch rewrites the targets in place
        loss = tr.training_step(bd, 0)["loss"]
        grads = torch.autograd.grad(loss, params)
        return [loss.detach(), tr.current_patch_mask, bd["images"], *grads]

    eager = [[t.clone() for t in step()] for _ in range(3)]
    assert tr.global_step.item() == 3
    assert [int((e[1] == 0).sum(-1).unique().item()) for e in eager] == [tr.patch_masker.patches_to_mask(s, 24 * 24) for s in range(3)]
    assert [tr.patch_masker.patches_to_mask(s, 24 * 24) for s in range(3)] == [0, 115, 230]
    for e in eager:
        assert torch.equal(e[2], lpb.patch_mask_apply(images0, e[1]))
        assert torch.isfinite(e[0]) and all(torch.isfinite(g_).all() and float(g_.abs().max()) > 0 for g_ in e[3:])
    assert all(not d["value"].requires_grad for d in tr.last_logs)  # no step's autograd graph outlives it

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    tr.global_step.zero_()
    for i in range(3):
        graph.replay()
        got = [t.clone() for t in out]
        for a, b in zip(eager[i][:3], got[:3]):
            assert torch.equal(a, b), i
        # gradients: the head's bias gradient is summed with float atomics (DESIGN.md), so to rounding
        for a, b in zip(eager[i][3:], got[3:]):
            assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()), i
    torch.cuda.synchronize(dev)
    assert tr.global_step.item() == 3
    assert torch.equal(images0, _calibrated_batch(lpb, dev)["images"])  # the caller's images are never written
    # the step's loss is evaluate_labeled's on the same masked batch
    bd["images"] = eager[2][2]
    bd["keypoints"].copy_(kp0)
    assert torch.equal(tr.evaluate_labeled(bd, "train").detach(), eager[2][0])


# ---- 7. malformed input -----------------------------------------------------------------------------------------------------
def test_malformed_inputs_raise(lpb, dev):
    from lightning_pose_b200._lib import LpbError

    mk = masker()
    x = torch.randn(2, 4, 3, 64, 80, device=dev)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        mk.apply_patch_masking(x.cpu(), 30)
    with pytest.raises(ValueError, match="batch, views, channels"):
        mk.apply_patch_masking(x[0], 30)
    for dt in (torch.float16, torch.float64, torch.uint8):
        with pytest.raises(ValueError, match="float32 or bfloat16"):
            mk.apply_patch_masking(x.to(dt), 30)
    with pytest.raises(ValueError, match="contiguous"):
        mk.apply_patch_masking(x.transpose(3, 4), 30)
    with pytest.raises(ValueError, match="4160 patches .* at most 4096"):
        mk.apply_patch_masking(torch.empty((1, 1, 3, 1040, 1024), device=dev), 30)
    with pytest.raises(ValueError, match="one-element int64"):
        mk.apply_patch_masking(x, torch.tensor([30], dtype=torch.int32, device=dev))
    with pytest.raises(ValueError, match="one-element int64"):
        mk.apply_patch_masking(x, torch.tensor([30]))
    with pytest.raises(ValueError, match="mask must be"):
        lpb.patch_mask_apply(x, torch.ones(2, 4, 19, device=dev))
    with pytest.raises(LpbError, match="final_step"):  # disabled maskers skip the constructor's check; the kernel does not
        masker(init_step=5, final_step=5, final_ratio=0.0).apply_patch_masking(x, 30)
