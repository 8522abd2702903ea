"""CPU pins of the float64 references in ``tests/scale_oracle.py``: each one against the CPU oracle, the golden vectors
the reference's own code wrote, and (for gradients) fp32 oracle autograd.  A wrong reference fails here, not on the GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lp_oracle as O
import scale_oracle as S

T = torch.from_numpy


def close(a, b, atol, rtol=0.0):
    a = a.detach().double().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)
    b = b.detach().double().numpy() if isinstance(b, torch.Tensor) else np.asarray(b, np.float64)
    np.testing.assert_allclose(a, b, atol=atol, rtol=rtol, equal_nan=True)


def _peaked(b, k, h, w, seed, sigma=1.6):
    g = torch.Generator().manual_seed(seed)
    cy = torch.rand(b, k, 1, 1, generator=g) * (h - 1)
    cx = torch.rand(b, k, 1, 1, generator=g) * (w - 1)
    yy = torch.arange(h).view(1, 1, h, 1).float()
    xx = torch.arange(w).view(1, 1, 1, w).float()
    logits = -((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sigma**2) + 0.05 * torch.randn(b, k, h, w, generator=g)
    return torch.softmax(logits.reshape(b, k, -1), -1).reshape(b, k, h, w)


# ------------------------------------------------------------------------------------------------
# decode
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,n,ds", [("U_n16_ds1", 16, 1), ("U_n16_ds2", 16, 2), ("U_n12_ds3", 12, 3), ("U_n96_ds2", 96, 2)])
def test_upsample_operator_matches_golden(golden, key, n, ds):
    close(S.upsample_op(n, ds, "cpu"), golden("decode")[key], atol=5e-7)  # the golden is the reference's fp32 impulse response


@pytest.mark.parametrize("name", ["peaked", "flat", "edge", "multi", "raw"])
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_ref_golden_regimes(golden, name, ds):
    g = golden("decode")
    preds, conf, pre, alt = S.decode_ref(T(g[f"{name}_in"]), ds, 1000.0)
    assert preds.dtype == torch.float64 and conf.shape == alt.shape[:2] and pre.shape[-1] == 2
    close(preds, g[f"{name}_ds{ds}_out_preds"], atol=5e-4 if name == "flat" else 5e-5)  # fp32 golden: ulp(256) = 3e-5
    close(conf, g[f"{name}_ds{ds}_out_conf"], atol=1e-6)
    close(preds.reshape(pre.shape), pre - {1: 0.5, 2: 1.5, 3: 2.5}[ds], atol=0)


def test_decode_ref_known_answers(golden):
    g = golden("decode")
    for ds in (1, 2, 3):
        p, c, _, _ = S.decode_ref(T(g[f"kat_ds{ds}_in"]), ds, 1000.0)
        close(p, g[f"kat_ds{ds}_out_preds"], atol=2e-5)
        close(c, g[f"kat_ds{ds}_out_conf"], atol=1e-6)
    for temp in (1000, 100, 10):
        p, c, _, _ = S.decode_ref(T(g["temp_in"]), 2, float(temp))
        close(p, g[f"temp{temp}_out_preds"], atol=2e-5)
        close(c, g[f"temp{temp}_out_conf"], atol=1e-6)


@pytest.mark.parametrize("shape", [(2, 3, 16, 16), (1, 2, 30, 41), (1, 2, 8, 8)])
@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_ref_vs_oracle(shape, ds):
    hm = _peaked(*shape, seed=3 + ds)
    hm[0, 0] = torch.softmax(0.01 * torch.randn(shape[2] * shape[3], generator=torch.Generator().manual_seed(ds)), 0).reshape(shape[2:])
    po, co = O.decode_softargmax(hm, ds, 1000.0)
    p, c, _, alt = S.decode_ref(hm, ds, 1000.0)
    close(p, po, atol=1e-4)
    close(c, co, atol=2e-6)
    # away from integer coordinates every alternative window is the trunc window itself
    assert torch.equal(alt[..., 0], c)


def test_decode_ref_trunc_alternatives():
    """Shifts wider than half a pixel cross an integer: conf is the trunc window, the alternatives include other windows."""
    hm = _peaked(1, 1, 8, 8, seed=1, sigma=2.0)
    _, conf, pre, alt = S.decode_ref(hm, 1, 1.0, trunc_eps=0.6)
    assert float(conf[0, 0]) == float(alt[0, 0, 0])
    assert len({round(float(v), 12) for v in alt[0, 0]}) > 1


@pytest.mark.parametrize("ds", [1, 2, 3])
def test_decode_grad_ref_vs_oracle_autograd(ds):
    hm = _peaked(2, 3, 12, 10, seed=7 + ds)
    hm[1, 2] = torch.softmax(0.3 * torch.randn(120, generator=torch.Generator().manual_seed(1)), 0).reshape(12, 10)
    gxy = torch.randn(2, 3, 2, generator=torch.Generator().manual_seed(2))
    x = hm.clone().requires_grad_(True)
    po, _ = O.decode_softargmax(x, ds, 1000.0)
    (po.reshape(2, 3, 2) * gxy).sum().backward()
    g = S.decode_grad_ref(hm, ds, 1000.0, gxy)
    # the same gradient through decode_ref's own autograd graph
    y = hm.double().requires_grad_(True)
    p, _, _, _ = S.decode_ref(y, ds, 1000.0)
    (p.reshape(2, 3, 2) * gxy.double()).sum().backward()
    close(g, y.grad, atol=1e-12 * float(y.grad.abs().max()), rtol=1e-9)
    close(g, x.grad, atol=2e-3 * float(g.abs().max()), rtol=2e-3)


# ------------------------------------------------------------------------------------------------
# head
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,nl", [("resnet", 2), ("vit", 1)])
def test_head_ref_golden(golden, tag, nl):
    g = golden("head")
    ws = [T(g[f"{tag}_w{i}"]) for i in range(nl)]
    bs = [T(g[f"{tag}_b{i}"]) for i in range(nl)]
    f = T(g[f"{tag}_in_features"])
    close(S.head_ref(f, ws, bs, True, bf16_operands=False), g[f"{tag}_out_heatmaps"], atol=1e-8, rtol=1e-5)
    close(S.head_ref(f, ws, bs, False, bf16_operands=False), g[f"{tag}_out_logits"], atol=2e-5, rtol=1e-5)
    close(S.head_ref_chunked(f, ws, bs, True, bf16_operands=False), O.head_forward(f, ws, bs), atol=1e-8, rtol=1e-5)


def _head_params(cin, c1, c2, seed):
    g = torch.Generator().manual_seed(seed)
    ws = [torch.randn(cin // 4, c1, 3, 3, generator=g) * 0.2]
    bs = [torch.rand(c1, generator=g) * 0.6 - 0.3]
    if c2:
        ws.append(torch.randn(c1, c2, 3, 3, generator=g) * 0.4)
        bs.append(torch.rand(c2, generator=g) * 0.6 - 0.3)
    return ws, bs


@pytest.mark.parametrize("c2", [0, 5])
def test_head_ref_bf16_operands(c2):
    """bf16 operands: weights and the inter-layer activations rounded exactly as the fp32 restatement of the existing
    GPU tests rounds them; the features are used as given."""
    ws, bs = _head_params(64, 5, c2, seed=4)
    feats = (torch.randn(3, 64, 3, 4, generator=torch.Generator().manual_seed(5))).bfloat16()
    r = lambda t: t.bfloat16().float()
    x = F.pixel_shuffle(feats.float(), 2)
    for i, (w, b) in enumerate(zip(ws, bs)):
        x = F.conv_transpose2d(r(x) if i else x, r(w), b, stride=2, padding=1, output_padding=1)
    got = S.head_ref(feats, ws, bs, softmax=False)
    # fp32 vs fp64 accumulation may move a mid value across a bf16 rounding boundary: compare at that scale
    close(got, x, atol=1e-2 * float(x.abs().max()), rtol=1e-2)
    assert float((got - x.double()).abs().max()) < 1e-4 * float(x.abs().max()) + 1e-2 * (c2 > 0)
    # rounded operands really differ from unrounded ones
    assert not torch.allclose(got, S.head_ref(feats, ws, bs, softmax=False, bf16_operands=False), atol=1e-9, rtol=0)
    close(S.head_ref_chunked(feats, ws, bs, True), S.head_ref(feats, ws, bs, True), atol=1e-15)


@pytest.mark.parametrize("c2,softmax", [(0, True), (5, True), (5, False)])
def test_head_grad_ref_vs_oracle_autograd(c2, softmax):
    ws, bs = _head_params(64, 5, c2, seed=6)
    feats = torch.randn(3, 64, 3, 4, generator=torch.Generator().manual_seed(7))
    out_hw = (3 * (8 if c2 else 4), 4 * (8 if c2 else 4))
    gout = torch.randn(3, c2 or 5, *out_hw, generator=torch.Generator().manual_seed(8))
    f = feats.clone().requires_grad_(True)
    wr = [w.clone().requires_grad_(True) for w in ws]
    br = [b.clone().requires_grad_(True) for b in bs]
    (O.head_forward(f, wr, br, softmax) * gout).sum().backward()
    dfeat, dws, dbs, mid_norm = S.head_grad_ref(feats, ws, bs, gout, softmax, bf16_operands=False, want_mid_grad=c2 > 0) if c2 else (
        *S.head_grad_ref(feats, ws, bs, gout, softmax, bf16_operands=False), None)
    close(dfeat, f.grad, atol=1e-6 * float(f.grad.abs().max()), rtol=1e-4)
    wscale = float(wr[-1].grad.abs().max())  # bias gradients behind a softmax cancel (the last one exactly): fp32 noise
    for a, b in zip(dws + dbs, [w.grad for w in wr] + [b.grad for b in br]):
        close(a, b, atol=1e-5 * max(float(b.abs().max()), wscale), rtol=1e-4)
    if c2:
        assert mid_norm.shape == (5,) and bool((mid_norm > 0).all())


# ------------------------------------------------------------------------------------------------
# losses
# ------------------------------------------------------------------------------------------------
def test_gaussian_targets_ref_vs_oracle(golden):
    g = golden("losses")
    kp, vis = T(g["hmb_in_kp"]), T(g["hmb_in_vis"])
    kp2 = kp.clone()
    kp2[0, 0] = float("nan")
    kp2[1, 1] = torch.tensor([-9.0, 3.0])
    kp2[2, 2] = torch.tensor([60.0, 140.0])
    for v in (None, vis):
        close(S.gaussian_targets_ref(kp2, 128, 128, (32, 32), visibility=v), O.gaussian_targets(kp2, 128, 128, (32, 32), visibility=v), atol=1e-7)


def test_heatmap_loss_ref_golden(golden):
    g = golden("losses")
    a = S.gaussian_targets_ref(T(g["hm_in_a_kp"]), 384, 384, (96, 96))
    b = S.gaussian_targets_ref(T(g["hm_in_b_kp"]), 384, 384, (96, 96))
    targ = S.gaussian_targets_ref(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"]))
    pred = T(g["hmb_in_pred"])
    for kind in ("mse", "kl", "js"):
        close(S.heatmap_loss_ref(b, a, kind), g[f"hm_{kind}_out_targb_preda"], atol=1e-7, rtol=1e-5)
        close(S.heatmap_loss_ref(a, b, kind), g[f"hm_{kind}_out_targa_predb"], atol=1e-7, rtol=1e-5)
        close(S.heatmap_loss_ref(targ, pred, kind), g[f"hmb_{kind}_out"], atol=1e-7, rtol=1e-5)
    close(S.heatmap_loss_ref(targ, pred, "mse"), g["hmb_mse_out"], atol=1e-7, rtol=1e-5)


@pytest.mark.parametrize("kind", ["mse", "kl", "js"])
def test_heatmap_loss_ref_grad_vs_oracle(golden, kind):
    g = golden("losses")
    targ = O.gaussian_targets(T(g["hmb_in_kp"]), 128, 128, (32, 32), visibility=T(g["hmb_in_vis"]))
    pred = T(g["hmb_in_pred"])
    fn = {"mse": O.heatmap_mse_loss, "kl": O.heatmap_kl_loss, "js": O.heatmap_js_loss}[kind]
    pr = pred.clone().requires_grad_(True)
    fn(targ, pr).backward()
    S._CHUNK_ELEMS, saved = 4 * 32 * 32 * 6, S._CHUNK_ELEMS  # several chunks even at this size
    try:
        v, grad = S.heatmap_loss_ref(targ, pred, kind, with_grad=True)
    finally:
        S._CHUNK_ELEMS = saved
    close(v, fn(targ, pred), atol=1e-7, rtol=1e-5)
    close(grad, pr.grad, atol=1e-9, rtol=1e-3)


def test_temporal_and_pca_refs_golden(golden):
    g = golden("losses")
    kp, conf = T(g["temporal_in_kp"]), T(g["temporal_in_conf"])
    close(S.temporal_loss_ref(kp, conf, [2.0, 20.0], 0.05), 3.8, atol=1e-6)  # tests/losses/test_losses.py:343-392
    close(S.temporal_loss_ref(kp, None, [2.0, 20.0], 0.05), 5.8, atol=1e-6)
    close(S.temporal_loss_ref(T(g["temporal2_in_kp"]), T(g["temporal2_in_conf"]), 20.0, 0.05), g["temporal2_out"], atol=1e-6)
    kseq = T(g["pca_in_kp"])
    for centering in (None, "mean", "median"):
        v = S.pca_singleview_ref(kseq, g["pca_sv_cols"].tolist(), centering, T(g["pca_sv_mean"]), T(g["pca_sv_kept"]), 2.5)
        assert v.dtype == torch.float64
        close(v, g[f"pca_sv_out_{centering}"], atol=1e-5, rtol=1e-5)
    v = S.pca_multiview_ref(kseq, g["pca_mv_mcm"].tolist(), T(g["pca_mv_mean"]), T(g["pca_mv_kept"]), 0.7)
    close(v, g["pca_mv_out"], atol=1e-5, rtol=1e-5)


def test_unsup_refs_grad_vs_oracle_autograd(golden):
    g = golden("losses")
    kseq, conf = T(g["pca_in_kp"]), torch.rand(32, 17, generator=torch.Generator().manual_seed(2))
    cols, mcm = g["pca_sv_cols"].tolist(), g["pca_mv_mcm"].tolist()
    for centering in (None, "mean", "median"):
        ref = kseq.clone().requires_grad_(True)
        (1.3 * O.temporal_loss(ref, conf, 3.0, 0.2)
         + 0.7 * O.pca_loss(O.pca_format_singleview(ref, cols, centering), T(g["pca_sv_mean"]), T(g["pca_sv_kept"]), 2.5)
         + 2.1 * O.pca_loss(O.pca_format_multiview(ref, mcm), T(g["pca_mv_mean"]), T(g["pca_mv_kept"]), 0.7)).backward()
        x = kseq.double().requires_grad_(True)
        (1.3 * S.temporal_loss_ref(x, conf, 3.0, 0.2)
         + 0.7 * S.pca_singleview_ref(x, cols, centering, T(g["pca_sv_mean"]), T(g["pca_sv_kept"]), 2.5)
         + 2.1 * S.pca_multiview_ref(x, mcm, T(g["pca_mv_mean"]), T(g["pca_mv_kept"]), 0.7)).backward()
        close(x.grad, ref.grad, atol=1e-6, rtol=1e-4)


# ------------------------------------------------------------------------------------------------
# MHCRNN
# ------------------------------------------------------------------------------------------------
def _golden_crnn_params(g, tag, uf):
    pre = f"{tag}_param_head_mf."
    c = lambda name: T(g[pre + name])
    p = {"W_f": (c("W_f.weight"), c("W_f.bias")), "W_b": (c("W_b.weight"), c("W_b.bias")),
         "H_f": tuple(c(f"H_f.{i}.{n}") for i in (0, 1) for n in ("weight", "bias")),
         "H_b": tuple(c(f"H_b.{i}.{n}") for i in (0, 1) for n in ("weight", "bias"))}
    if uf == 2:
        p["W_pre"] = (c("W_pre.weight"), c("W_pre.bias"))
    return p


@pytest.mark.parametrize("tag,uf", [("vit", 1), ("resnet", 2)])
def test_crnn_refs_golden(golden, tag, uf):
    """crnn_ref against the reference module's own outputs; the window form (crnn_combine_ref on per-frame maps) is the
    same recurrence."""
    g = golden("mhcrnn")
    p = _golden_crnn_params(g, tag, uf)
    feats = T(g[f"{tag}_in_features"]).permute(4, 0, 1, 2, 3).contiguous()  # (batch, C, h, w, frames) -> frames first
    mf = S.crnn_ref(feats, p, uf)
    assert mf.dtype == torch.float64
    close(mf, g[f"{tag}_out_mf"], atol=1e-7, rtol=1e-5)
    close(mf, O.mhcrnn_multiframe(feats, p, uf), atol=1e-7, rtol=1e-5)
    logits = S.crnn_ref(feats, p, uf, softmax=False)
    close(O.spatial_softmax2d(logits, 1.0), mf, atol=1e-12)
