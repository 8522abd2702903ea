"""Training the context (MHCRNN) head against float64: ``HeatmapMHCRNNHead`` in its sequence form (``forward_sequence``)
and its call form (``forward`` on (B, C, h, w, 5) features), and ``SemiSupervisedHeatmapTrackerMHCRNN.training_step``.

The context head combines kernels that are each tested alone: the head's logit kernels run twice on the same frames
(W_pre + W_f and W_pre + W_b, or W_f and W_b), the recurrence kernel reads their maps through a window table, the
single-frame head reads a slice of the frames, and the window gather feeds the multi-view form.  The float64 reference
is ``scale_oracle.context_ref`` (pinned on the CPU in ``test_scale_oracle.py``); every comparison goes through the
per-channel rules of ``head_support.py``, plus a per-keypoint rule for the recurrence's parameters.
``test_context_rules_reject_plausible_bugs`` shows on the CPU that the rules reject the bugs such a combination invites
(slot order, window tables, the single-frame slice, lost or doubled gradient terms)."""
import pytest
import torch

import scale_oracle as S
from head_support import (F64, WORST, _judge, check_grads, check_grads_f32, check_heatmaps, features, gen, logit_grad,
                          report_headroom)
from oracle import lp_oracle as O

BF16, F32 = torch.bfloat16, torch.float32
H_NAMES = [f"{d}.{i}.{n}" for d in ("H_f", "H_b") for i in (0, 1) for n in ("weight", "bias")]

# name: (backbone, C, h, w, upsampling_factor, keypoints).  ViT-S config 3; ResNet-50 at 384^2 (its maps take the
# whole-frame k1a kernels) and 256^2; the mirror-fish shape past 20 keypoints (keypoint groups).
ROWS = {
    "vit_c384_16x16": ("vits_dino", 384, 16, 16, 1, 17),
    "r50_c2048_12x12": ("resnet50", 2048, 12, 12, 2, 17),
    "r50_c2048_8x8": ("resnet50", 2048, 8, 8, 2, 17),
    "r50_c2048_8x12_k51": ("resnet50", 2048, 8, 12, 2, 51),
}
T_SEQ, B_CALL = 9, 3  # frames of the sequence form (5 windows), windows of the call form


@pytest.fixture(scope="module", autouse=True)
def _report_headroom():
    WORST.clear()
    yield
    report_headroom()


# ------------------------------------------------------------------------------------------------
# the head, its window tables and the float64 reference
# ------------------------------------------------------------------------------------------------
def make_context_head(arch, c, k, uf, seed, device="cuda"):
    """A HeatmapMHCRNNHead with every deconv at xavier-uniform gain 3 and biases in [-0.3, 0.3] (as ``make_head``), and
    the recurrence's weights at gain 4, so that each step moves the maps visibly, biases in [-0.1, 0.1]."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    torch.manual_seed(seed)
    head = HeatmapMHCRNNHead(arch, c, k, upsampling_factor=uf)
    mf = head.head_mf
    for layer in [*list(head.head_sf.upsampling_layers)[1:], *([mf.W_pre] if uf == 2 else []), mf.W_f, mf.W_b]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
        torch.nn.init.uniform_(layer.bias, -0.3, 0.3)
    for layer in (*mf.H_f, *mf.H_b):
        torch.nn.init.xavier_uniform_(layer.weight, gain=4.0)
        torch.nn.init.uniform_(layer.bias, -0.1, 0.1)
    return head.to(device)


def head_tensors(head):
    """(single-frame weights, biases, context parameters as ``crnn_ref`` takes them) of a HeatmapMHCRNNHead, detached."""
    deconvs = list(head.head_sf.upsampling_layers)[1:]
    mf = head.head_mf
    wb = lambda m: (m.weight.detach(), m.bias.detach())  # noqa: E731
    p = {"W_f": wb(mf.W_f), "W_b": wb(mf.W_b), "H_f": (*wb(mf.H_f[0]), *wb(mf.H_f[1])), "H_b": (*wb(mf.H_b[0]), *wb(mf.H_b[1]))}
    if mf.upsampling_factor == 2:
        p["W_pre"] = wb(mf.W_pre)
    return [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs], p


def head_grads(head):
    """The head's parameter gradients under the reference's names."""
    deconvs = list(head.head_sf.upsampling_layers)[1:]
    mf = head.head_mf
    out = {}
    for i, d in enumerate(deconvs, 1):
        out[f"dw{i}"], out[f"db{i}"] = d.weight.grad, d.bias.grad
    for key, m in (("pre", mf.W_pre if mf.upsampling_factor == 2 else None), ("f", mf.W_f), ("b", mf.W_b)):
        if m is not None:
            out[f"dw_{key}"], out[f"db_{key}"] = m.weight.grad, m.bias.grad
    for name in H_NAMES:
        d, i, n = name.split(".")
        out[name] = getattr(getattr(mf, d)[int(i)], n).grad
    return out


def sequence_table(t, device="cuda"):
    """``forward_sequence`` on t frames: window m reads frames m .. m + 4; the single-frame head frames 2 .. t - 3."""
    idx = torch.arange(t - 4, device=device)[:, None] + torch.arange(5, device=device)[None, :]
    return idx, torch.arange(2, t - 2, device=device)


def call_table(b, device="cuda"):
    """``forward`` on (b, C, h, w, 5) features, frames flattened slot-major (frame s * b + w is slot s of window w):
    window w reads s * b + w; the single-frame head the middle slot, frames 2b .. 3b - 1."""
    idx = torch.arange(5, device=device)[None, :] * b + torch.arange(b, device=device)[:, None]
    return idx, torch.arange(2 * b, 3 * b, device=device)


def _norm(g):
    return g.pow(2).sum((0, 2, 3)).sqrt()


def reference(feats, ws, bs, p, idx, sf_rows, g_sf, g_mf, operands=BF16, uf=None, wb_dfeat=True, once=False):
    """float64 autograd of sum(sf * g_sf) + sum(mf * g_mf): the single-frame head on ``feats[sf_rows]`` and the context
    head (``context_ref``) on the frames ``feats`` (N, C, h, w) through the window table ``idx``.

    Returns (sf, mf, gradients, gnorm): the gradients under ``head_grads``' names plus "dfeat" (N, C, h, w); ``gnorm``
    the per-channel L2 norm of the gradient each deconv bias sums, added over the kernel runs that sum it (one per
    head call; W_pre's is summed by both map runs), and under "H" that of the context head's logit gradient.  ``wb_dfeat=False`` and ``once=True`` build the plausible bugs of
    ``test_context_rules_reject_plausible_bugs``: W_b's d features not added, and a frame's gradient taken from one of
    the window slots that read it."""
    uf = (2 if "W_pre" in p else 1) if uf is None else uf
    f = feats.detach().to(F64).requires_grad_(True)
    sw = [w.detach().to(F64).requires_grad_(True) for w in ws]
    sb = [b.detach().to(F64).requires_grad_(True) for b in bs]
    pp = {key: tuple(t.detach().to(F64).requires_grad_(True) for t in tup) for key, tup in p.items()}
    mids_sf, mids_mf = [], []
    sf = S.head_ref(f[sf_rows], sw, sb, softmax=True, operands=operands, mids=mids_sf)
    if once:  # every window slot its own frame; a frame's gradient read back from the first slot that holds it
        flat = idx.reshape(-1)
        f_win = f.detach()[flat].requires_grad_(True)
        mf, wf, wb = S.context_ref(f_win, pp, uf, torch.arange(flat.numel(), device=f.device).reshape(idx.shape), operands, mids=mids_mf)
    else:
        mf, wf, wb = S.context_ref(f, pp, uf, idx, operands, mids=mids_mf)
    ((sf * g_sf.to(F64)).sum() + (mf * g_mf.to(F64)).sum()).backward()
    dfeat = f.grad.clone()
    if once:
        first = {}
        for j, fr in enumerate(flat.tolist()):
            first.setdefault(fr, j)
        for fr, j in first.items():
            dfeat[fr] += f_win.grad[j]
    if not wb_dfeat:  # d features of the W_b run: its maps' gradient back through W_pre + W_b
        layers = ([pp["W_pre"]] if uf == 2 else []) + [pp["W_b"]]
        f2 = f.detach().requires_grad_(True)
        m = S.head_ref(f2, [w for w, _ in layers], [b for _, b in layers], softmax=False, operands=operands)
        (dw_b,) = torch.autograd.grad((m * wb.grad).sum(), f2)
        dfeat -= dw_b
    grads = {"dfeat": dfeat}
    for i, (w, b) in enumerate(zip(sw, sb), 1):
        grads[f"dw{i}"], grads[f"db{i}"] = w.grad, b.grad
    for key, name in (("W_pre", "pre"), ("W_f", "f"), ("W_b", "b")):
        if key in pp:
            grads[f"dw_{name}"], grads[f"db_{name}"] = pp[key][0].grad, pp[key][1].grad
    for name in H_NAMES:
        d, i, n = name.split(".")
        grads[name] = pp[d][2 * int(i) + (n == "bias")].grad
    gnorm = {f"db{len(sw)}": _norm(logit_grad(g_sf, sf.detach())), "db_f": _norm(wf.grad), "db_b": _norm(wb.grad),
             "H": _norm(logit_grad(g_mf, mf.detach()))}
    if len(sw) == 2:
        gnorm["db1"] = _norm(mids_sf[0].grad)
    if uf == 2:
        gnorm["db_pre"] = _norm(mids_mf[0].grad) + _norm(mids_mf[1].grad)
    return sf.detach(), mf.detach(), grads, gnorm


def check_recurrence(got, ref, gnorm, k, case, rel, sums, prefix=""):
    """H_f / H_b: each keypoint's slice of each tensor (its 16 hidden filters) within ``rel`` of that slice's largest
    entry.  The output bias (one entry per keypoint) sums the chain's gradient over every block and step; behind the
    softmax the first step's sum cancels exactly (a logit gradient sums to 0 over its plane), so the entry itself is no
    scale for its error.  It is held, as ``check_grads`` / ``check_grads_f32`` hold a deconv bias, to ``rel`` of itself
    plus ``sums`` (4 x 2^-8 after bf16 operands, 2^-14 in fp32) of what it sums: four steps of the keypoint's logit
    gradient, of L2 norm ``gnorm["H"][k]`` each."""
    ratios = {}
    for name in H_NAMES:
        g, r = got[name].detach().to(F64).reshape(k, -1), ref[name].to(F64).reshape(k, -1)
        err = (g - r).abs().amax(1)
        if name.endswith("1.bias"):
            ratios[prefix + name] = err / (rel * r.abs().amax(1) + 4 * sums * gnorm["H"].to(F64) + 1e-12)
        else:
            ratios[prefix + name] = err / (rel * r.abs().amax(1) + 1e-12)
    _judge(case, ratios)


def check_context_grads(got, ref, gnorm, k, case, fp32=False, rel=1e-2, global_scale=()):
    """The deconvs and d features by ``check_grads`` (bf16, ``rel``, ``global_scale``) or ``check_grads_f32``; the
    recurrence per keypoint within ``rel`` (bf16) or 1e-3 (fp32)."""
    deconv = {n: v for n, v in ref.items() if n not in H_NAMES}
    if fp32:
        check_grads_f32(got, deconv, gnorm, case)
        check_recurrence(got, ref, gnorm, k, case, 1e-3, 2.0**-14, prefix="fp32 ")
    else:
        check_grads(got, deconv, gnorm, case, rel=rel, global_scale=global_scale)
        check_recurrence(got, ref, gnorm, k, case, rel, 4 * 2.0**-8)


def check_heatmaps_f32(out, ref, case, key):
    """fp32 features: every pixel within 1e-4 relative (+1e-9) of float64 (``test_fp32_fallback``'s bar)."""
    out, ref = out.detach().to(F64), ref.to(F64)
    _judge(case, {f"fp32 {key}: relative error": ((out - ref).abs() / (1e-4 * ref + 1e-9)).amax((-1, -2))})


def check_forward(sf, mf, sf_ref, mf_ref, case, dtype):
    if dtype == F32:
        check_heatmaps_f32(sf, sf_ref, case, "sf heatmaps")
        check_heatmaps_f32(mf, mf_ref, case, "mf heatmaps")
    else:
        check_heatmaps(sf, sf_ref, case, key="sf heatmaps")
        check_heatmaps(mf, mf_ref, case, key="mf heatmaps")


# ------------------------------------------------------------------------------------------------
# CPU: the rules reject plausible bugs
# ------------------------------------------------------------------------------------------------
def _hidden_params(k, seed):
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: (torch.rand(*s, generator=g, dtype=F64) * 2 - 1)  # noqa: E731
    return (0.4 * u(16 * k, 1, 2, 2), 0.1 * u(16 * k), 0.4 * u(16 * k, 1, 2, 2), 0.1 * u(k))


def _block_affine(hp, k):
    """(L (K, 4, 4), h (K, 4)) of a hidden layer: H(x)[2x2 block] = L x + h (csrc/crnn.cu)."""
    cw, tw = hp[0].reshape(k, 16, 4), hp[2].reshape(k, 16, 4)
    return torch.einsum("kfo,kfi->koi", tw, cw), hp[3][:, None] + torch.einsum("kfo,kf->ko", tw, hp[1].reshape(k, 16))


def _combine_blocks(wf, wb, idx, lf, lb):
    """crnn_combine_ref with the hidden layers as block-affine maps (L, h)."""
    def hidden(z, lh):
        m, k, hh, ww = z.shape
        zb = z.reshape(m, k, hh // 2, 2, ww // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(m, k, hh // 2, ww // 2, 4)
        y = torch.einsum("koi,mkyxi->mkyxo", lh[0], zb) + lh[1][None, :, None, None, :]
        return y.reshape(m, k, hh // 2, ww // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(m, k, hh, ww)

    xf = wf[idx[:, 0]]
    for t in range(1, 5):
        xf = wf[idx[:, t]] + hidden(xf, lf)
    xb = wb[idx[:, 4]]
    for t in range(3, -1, -1):
        xb = wb[idx[:, t]] + hidden(xb, lb)
    return (xf + xb) / 2


def test_context_rules_reject_plausible_bugs():
    """On a small float64 context head (two-deconv maps, bf16 operand roundings), the gradients of each plausible bug
    are rejected by the rules the GPU tests apply, and the unchanged reference passes them."""
    torch.manual_seed(5)
    c, h, w, k, t, b = 128, 4, 4, 3, 10, 2
    ws = [torch.nn.init.xavier_uniform_(torch.empty(c // 4, k, 3, 3, dtype=F64), gain=3.0),
          torch.nn.init.xavier_uniform_(torch.empty(k, k, 3, 3, dtype=F64), gain=3.0)]
    bs = [torch.empty(k, dtype=F64).uniform_(-0.3, 0.3), torch.empty(k, dtype=F64).uniform_(-0.3, 0.3)]
    dc = lambda cin: (torch.nn.init.xavier_uniform_(torch.empty(cin, k, 3, 3, dtype=F64), gain=3.0), torch.empty(k, dtype=F64).uniform_(-0.3, 0.3))  # noqa: E731
    p = {"W_pre": dc(c // 4), "W_f": dc(k), "W_b": dc(k), "H_f": _hidden_params(k, 1), "H_b": _hidden_params(k, 2)}
    feats = (torch.randn(t, c, h, w, dtype=F64) * 0.5).bfloat16()
    idx, rows = sequence_table(t, "cpu")
    g_sf = torch.randn(t - 4, k, 8 * h, 8 * w, dtype=F64)
    g_mf = torch.randn(t - 4, k, 8 * h, 8 * w, dtype=F64)
    def run(idx=idx, rows=rows, g_mf=g_mf, **kw):
        return reference(feats, ws, bs, p, idx, rows, g_sf, g_mf, **kw)

    sf, mf, ref, gnorm = run()

    def passes(got, sf_got=sf, mf_got=mf, case="reference"):
        check_heatmaps(sf_got, sf, case, key="sf heatmaps")
        check_heatmaps(mf_got, mf, case, key="mf heatmaps")
        check_context_grads(got, ref, gnorm, k, case)

    def rejects(res):
        with pytest.raises(AssertionError):
            passes(res[2], res[0], res[1], case="mutated")

    passes({n: v.clone() for n, v in ref.items()})
    # the recurrence with its hidden layers as block-affine maps is the same function: its (L, h) gradients map back
    # onto the parameters' (the kernel's prepare_bwd), and a transposed dL does not
    maps = [S.head_ref(feats, [p["W_pre"][0], p[key][0]], [p["W_pre"][1], p[key][1]], softmax=False) for key in ("W_f", "W_b")]
    hp = {d: tuple(x.clone().requires_grad_(True) for x in p[d]) for d in ("H_f", "H_b")}
    lh = {d: _block_affine(hp[d], k) for d in hp}
    leaves = {d: tuple(x.detach().requires_grad_(True) for x in lh[d]) for d in lh}
    logits = _combine_blocks(maps[0], maps[1], idx, leaves["H_f"], leaves["H_b"])
    torch.testing.assert_close(logits, S.crnn_combine_ref(maps[0], maps[1], idx, p["H_f"], p["H_b"]), rtol=1e-12, atol=1e-12)
    mf_l = torch.softmax(logits.flatten(2), -1).reshape(logits.shape)
    (mf_l * g_mf).sum().backward()
    for transpose in (False, True):
        got = dict(ref)
        for d in ("H_f", "H_b"):
            dl, dh = leaves[d][0].grad, leaves[d][1].grad
            pg = torch.autograd.grad(lh[d], hp[d], (dl.transpose(1, 2) if transpose else dl, dh), retain_graph=True)
            for i, n in enumerate(("0.weight", "0.bias", "1.weight", "1.bias")):
                got[f"{d}.{n}"] = pg[i]
        if transpose:
            rejects((sf, mf, got))
        else:
            passes(got)
    # the backward chain's slot order reversed (and with it the forward)
    rejects(run(idx=idx.flip(1)))
    # the combine's 0.5 dropped in the backward
    rejects((sf, mf, run(g_mf=2 * g_mf)[2]))
    # W_b's d features not added
    rejects((sf, mf, run(wb_dfeat=False)[2]))
    # the single-frame head on frames shifted by one
    rejects(run(rows=rows + 1))
    # a frame read by several windows given the gradient of one of them
    rejects((sf, mf, run(once=True)[2]))
    # the call form: its window table frame-major (window w reads 5 w + s) instead of slot-major
    idx_c, rows_c = call_table(b, "cpu")
    feats_c = feats[: 5 * b]
    g_sf_c, g_mf_c = g_sf[:b], g_mf[:b]
    sf_c, mf_c, ref_c, gnorm_c = reference(feats_c, ws, bs, p, idx_c, rows_c, g_sf_c, g_mf_c)
    check_context_grads(ref_c, ref_c, gnorm_c, k, "call form reference")
    bad_sf, bad_mf, bad, _ = reference(feats_c, ws, bs, p, torch.arange(5 * b).reshape(b, 5), rows_c, g_sf_c, g_mf_c)
    with pytest.raises(AssertionError):
        check_heatmaps(bad_mf, mf_c, "mutated", key="mf heatmaps")
    with pytest.raises(AssertionError):
        check_context_grads(bad, ref_c, gnorm_c, k, "mutated")
    WORST.clear()


# ------------------------------------------------------------------------------------------------
# GPU: the window gather's gradient
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n,ctx", [(1, 5), (2, 5), (3, 5), (8, 5), (8, 3)])
def test_context_gather_gradient(n, ctx, dtype):
    """get_context_from_sequence is differentiable: a frame's gradient is the sum of the window slots that read it, the
    repeated edge frames included, against float64 autograd of the reference's window loop.  The slots are summed in
    fp32: within 2^-21 of the sum of their magnitudes, and rounded once to bf16 for bf16 frames."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import get_context_from_sequence

    seq = torch.randn(n, 8, 4, 6, device="cuda", generator=gen(n)).to(dtype)
    gout = torch.randn(n, ctx, 8, 4, 6, device="cuda", generator=gen(n + ctx)).to(dtype)
    x = seq.clone().requires_grad_(True)
    win = get_context_from_sequence(x, ctx)
    assert win.grad_fn is not None
    assert torch.equal(win.detach().cpu().float(), O.context_windows(seq.cpu().float(), ctx))
    win.backward(gout)

    def ref(g):
        s = seq.cpu().to(F64).requires_grad_(True)
        (O.context_windows(s, ctx).to(F64) * g.cpu().to(F64)).sum().backward()
        return s.grad

    want, mag = ref(gout), ref(gout.abs())
    err = (x.grad.cpu().to(F64) - want).abs()
    allowed = 2.0**-21 * mag + (2.0**-8 * want.abs() if dtype == BF16 else 0.0) + 1e-30
    assert x.grad.dtype == dtype and bool((err <= allowed).all()), float((err / allowed).max())


# ------------------------------------------------------------------------------------------------
# GPU: the head in both forms
# ------------------------------------------------------------------------------------------------
def _run_sequence(head, x, g_seed=7):
    leaf = x.clone().requires_grad_(True)
    sf, mf = head.forward_sequence(leaf)
    g_sf = torch.randn(sf.shape, device="cuda", generator=gen(g_seed))
    g_mf = torch.randn(mf.shape, device="cuda", generator=gen(g_seed + 1))
    head.zero_grad(set_to_none=True)
    ((sf * g_sf).sum() + (mf * g_mf).sum()).backward()
    return sf.detach(), mf.detach(), {"dfeat": leaf.grad, **head_grads(head)}, g_sf, g_mf


def _check_case(head, frames, got, sf, mf, idx, rows, g_sf, g_mf, k, case, dtype):
    ws, bs, p = head_tensors(head)
    sf_ref, mf_ref, ref, gnorm = reference(frames, ws, bs, p, idx, rows, g_sf, g_mf, operands=BF16 if dtype == BF16 else None)
    check_forward(sf, mf, sf_ref, mf_ref, case, dtype)
    check_context_grads(got, ref, gnorm, k, case, fp32=dtype == F32)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("form", ["sequence", "call"])
@pytest.mark.parametrize("row", list(ROWS))
def test_context_head(row, form, dtype):
    """sf / mf heatmaps, every parameter gradient and d features of random dense output gradients, against float64."""
    arch, c, h, w, uf, k = ROWS[row]
    head = make_context_head(arch, c, k, uf, seed=11)
    case = f"{row} {form} {'bf16' if dtype == BF16 else 'fp32'}"
    if form == "sequence":
        x = features(T_SEQ, c, h, w, 3, dtype)
        sf, mf, got, g_sf, g_mf = _run_sequence(head, x)
        frames = x
        idx, rows = sequence_table(T_SEQ)
    else:
        frames = features(5 * B_CALL, c, h, w, 3, dtype)  # slot-major, as forward flattens them
        x = frames.reshape(5, B_CALL, c, h, w).permute(1, 2, 3, 4, 0).contiguous()
        leaf = x.clone().requires_grad_(True)
        sf, mf = head(leaf, torch.Size([B_CALL, 5, 3, 16 * h, 16 * w]), False)
        g_sf = torch.randn(sf.shape, device="cuda", generator=gen(7))
        g_mf = torch.randn(mf.shape, device="cuda", generator=gen(8))
        head.zero_grad(set_to_none=True)
        ((sf * g_sf).sum() + (mf * g_mf).sum()).backward()
        got = {"dfeat": leaf.grad.permute(4, 0, 1, 2, 3).reshape(frames.shape), **head_grads(head)}
        sf, mf = sf.detach(), mf.detach()
        idx, rows = call_table(B_CALL)
    assert got["dfeat"].dtype == dtype and sf.shape == mf.shape == (idx.shape[0], k, 4 * uf * h, 4 * uf * w)
    _check_case(head, frames, got, sf, mf, idx, rows, g_sf, g_mf, k, case, dtype)


@pytest.mark.gpu
def test_context_head_channels_last():
    """The ViT row's sequence form on channels-last features (a transformer's tokens): its maps take the banded kernels
    as the NCHW call does, so the heatmaps are the same bits, and so are the single-frame head's gradients.  The rest of
    the backward passes through the recurrence's backward, which sums shared frames' map gradients and the hidden
    layers' gradients with float atomics: it is held to float64 by the same rules."""
    arch, c, h, w, uf, k = ROWS["vit_c384_16x16"]
    head = make_context_head(arch, c, k, uf, seed=12)
    x = features(T_SEQ, c, h, w, 4, BF16)
    xc = x.contiguous(memory_format=torch.channels_last)
    assert not xc.is_contiguous()
    sf, mf, got, g_sf, g_mf = _run_sequence(head, x)
    sf_c, mf_c, got_c, _, _ = _run_sequence(head, xc)
    assert torch.equal(sf_c, sf) and torch.equal(mf_c, mf)
    for name in ("dw1", "db1"):
        assert torch.equal(got_c[name], got[name]), name
    idx, rows = sequence_table(T_SEQ)
    _check_case(head, x, got_c, sf_c, mf_c, idx, rows, g_sf, g_mf, k, "vit channels-last sequence bf16", BF16)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["vit_c384_16x16", "r50_c2048_12x12"])
def test_context_head_past_one_wave(row):
    """One sequence of 2 S + 11 frames (S read from the device): the head's persistent launches loop over frames."""
    arch, c, h, w, uf, k = ROWS[row]
    t = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 11
    head = make_context_head(arch, c, k, uf, seed=13)
    x = features(t, c, h, w, 5, BF16)
    sf, mf, got, g_sf, g_mf = _run_sequence(head, x, g_seed=9)
    idx, rows = sequence_table(t)
    _check_case(head, x, got, sf, mf, idx, rows, g_sf, g_mf, k, f"{row} sequence of {t} frames", BF16)


# ------------------------------------------------------------------------------------------------
# GPU: a semi-supervised training step
# ------------------------------------------------------------------------------------------------
class _Backbone(torch.nn.Module):
    """Stands in for ViT-S: (n, 3, 256, 256) -> (n, 384, 16, 16) bf16; keeps each output, with its gradient."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 384, 16, stride=16)
        self.outs = []

    def forward(self, x):
        y = self.conv(x).bfloat16()
        y.retain_grad()
        self.outs.append(y)
        return y


def remap_ref(kp, bbox, model_h, model_w, views):
    """model pixels -> frame pixels, bbox (x, y, h, w) per view (rows 2 .. n + 1 of a context batch's n + 4), float64."""
    n = kp.shape[0]
    bb = bbox.to(F64)
    bb = (bb if bb.shape[0] == n else bb[2:-2]).reshape(n, views, 1, 4)
    p = kp.reshape(n, views, -1, 2)
    return torch.stack([p[..., 0] / model_w * bb[..., 3] + bb[..., 0], p[..., 1] / model_h * bb[..., 2] + bb[..., 1]], -1).reshape(n, -1)


def _bbox(n, views, seed):
    g = gen(seed)
    xy = torch.rand(n, views, 2, device="cuda", generator=g) * 40
    hw = 200 + torch.rand(n, views, 2, device="cuda", generator=g) * 150
    return torch.cat([xy, hw], -1).reshape(n, 4 * views)


@pytest.mark.gpu
@pytest.mark.parametrize("unlabeled", ["single-view", "multi-view"])
def test_tracker_training_step(unlabeled):
    """One training_step on a labeled context batch (B, 5, 3, H, W) and an unlabeled video, single-view (T, 3, H, W) or
    multi-view (T, V, 3, H, W).  The float64 reference is staged: the losses' gradient with respect to both heads'
    heatmaps, taken at the kernels' heatmaps (heatmap MSE; the temporal loss through the remap and the soft-argmax),
    then back through the single-frame head and ``context_ref``.  The head's parameter gradients (summed over both
    batches) and the gradient at the backbone's output of each batch are held to it, and to the kernels' own heatmap
    gradients taken back through the same reference, with the 2e-2 bar and the rules of the other tests that chain the
    decode gradient (``test_head_shapes_gpu.py::test_fused_decode``)."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.losses.factory import LossFactory
    from lightning_pose_b200.models.heatmap_tracker_mhcrnn import SemiSupervisedHeatmapTrackerMHCRNN

    k, b, views = 17, 2, (2 if unlabeled == "multi-view" else 1)
    t = 7 if views == 2 else 9
    eps, thr, log_w = 1.0, 0.0, 0.5  # no confidence mask: an untrained head's confidences can all lie under one
    torch.manual_seed(0)
    tr = SemiSupervisedHeatmapTrackerMHCRNN(
        k, loss_factory=LossFactory({"heatmap_mse": {"log_weight": 0.0}}, None),
        loss_factory_unsupervised=LossFactory({"temporal": {"log_weight": log_w, "epsilon": eps, "prob_threshold": thr}}, None),
        backbone=_Backbone(), backbone_arch="vits_dino", num_fc_input_features=384).cuda()
    tr.head = make_context_head("vits_dino", 384, k, 1, seed=21)
    calls = []
    forward = tr.forward

    def recorded(images, is_multiview=False):
        calls.append(forward(images, is_multiview=is_multiview))
        for hm in calls[-1]:
            hm.retain_grad()
        return calls[-1]

    tr.forward = recorded
    g = gen(22)
    kp_lab = torch.rand(b, k, 2, device="cuda", generator=g) * 256
    labeled = {"images": torch.randn(b, 5, 3, 256, 256, device="cuda", generator=g), "keypoints": kp_lab.reshape(b, 2 * k),
               "heatmaps": S.gaussian_targets_ref(kp_lab, 256, 256, (64, 64)).float(), "bbox": _bbox(b, 1, 23)}
    shape = (t, views, 3, 256, 256) if views == 2 else (t, 3, 256, 256)
    unlab = {"frames": torch.randn(shape, device="cuda", generator=g), "transforms": torch.tensor([-1.0], device="cuda"),
             "bbox": _bbox(t, views, 24), "is_multiview": views == 2}
    tr.zero_grad(set_to_none=True)
    tr.training_step({"labeled": labeled, "unlabeled": unlab}, 0)["loss"].backward()
    case = f"training_step, {unlabeled} unlabeled video"

    # the losses' gradient at the kernels' heatmaps
    (sf_l, mf_l), (sf_u, mf_u) = [(s.detach(), m.detach()) for s, m in calls]
    hm = torch.cat([sf_l, mf_l])
    _, g_l = S.heatmap_loss_ref(torch.cat([labeled["heatmaps"]] * 2), hm, "mse", with_grad=True)
    g_l = 0.5 * g_l  # weight 1 / (2 exp(0)); the heatmap loss is not annealed
    hm_u = torch.cat([sf_u, mf_u])
    n_u = t - 4
    preds, _, _, _ = S.decode_ref(hm_u, 2)
    conf = torch.cat([ops.decode_softargmax(sf_u, 2)[1], ops.decode_softargmax(mf_u, 2)[1]])
    kp = preds.detach().requires_grad_(True)
    kp_frame = torch.cat([remap_ref(kp[:n_u], unlab["bbox"], 256, 256, views), remap_ref(kp[n_u:], unlab["bbox"], 256, 256, views)])
    loss_t = S.temporal_loss_ref(kp_frame, conf, eps, thr) / (2 * torch.exp(torch.tensor(log_w, dtype=F64)))
    (g_kp,) = torch.autograd.grad(loss_t, kp)
    g_u = S.decode_grad_ref(hm_u, 2, 1000.0, g_kp)

    # back through the heads, on the backbone's output rows
    ws, bs, p = head_tensors(tr.head)
    feats_l, feats_u = tr.backbone.outs
    idx_l = torch.arange(b, device="cuda")[:, None] * 5 + torch.arange(5, device="cuda")[None, :]  # window w: rows 5 w + s
    r_l = reference(feats_l, ws, bs, p, idx_l, idx_l[:, 2], g_l[:b], g_l[b:])
    # unlabeled rows t * V + v; window (t', v) reads frames t' .. t' + 4 of view v, its single frame t' + 2
    idx_u = (torch.arange(n_u, device="cuda")[:, None, None] + torch.arange(5, device="cuda")[None, None, :]) * views + torch.arange(views, device="cuda")[None, :, None]
    idx_u = idx_u.reshape(n_u * views, 5)
    r_u = reference(feats_u, ws, bs, p, idx_u, idx_u[:, 2], g_u[:n_u].reshape(n_u * views, k, 64, 64), g_u[n_u:].reshape(n_u * views, k, 64, 64))
    for (sf, mf), r, name in (((sf_l, mf_l), r_l, "labeled"), ((sf_u, mf_u), r_u, unlabeled)):
        check_forward(sf.reshape(r[0].shape), mf.reshape(r[1].shape), r[0], r[1], f"{case}: {name} batch", BF16)
    # the kernels' own heatmap gradients, back through the reference: every gradient per channel.  Against the float64
    # loss gradient the single-frame head's last weight gradient is held to its largest entry instead: at T = 1000 the
    # softmax backward of a peaked plane cancels all but a sliver of its decode gradient, and what is left of a small
    # keypoint's plane lies below the decode kernel's fp32 gradient error (test_head_shapes_gpu.py::test_fused_decode)
    (gsf_l, gmf_l), (gsf_u, gmf_u) = [(s.grad, m.grad) for s, m in calls]
    r_lk = reference(feats_l, ws, bs, p, idx_l, idx_l[:, 2], gsf_l, gmf_l)
    r_uk = reference(feats_u, ws, bs, p, idx_u, idx_u[:, 2], gsf_u.reshape(n_u * views, k, 64, 64), gmf_u.reshape(n_u * views, k, 64, 64))
    got = head_grads(tr.head)
    for (ra, rb), what, scale in (((r_lk, r_uk), "kernel heatmap gradients", ()), ((r_l, r_u), "float64 loss gradient", (f"dw{len(ws)}",))):
        ref = {n: ra[2][n] + rb[2][n] for n in got}
        gnorm = {n: ra[3][n] + rb[3][n] for n in ra[3]}
        check_context_grads(got, ref, gnorm, k, f"{case}, {what}", rel=2e-2, global_scale=scale)
        for out, r, name in ((feats_l, ra, "labeled"), (feats_u, rb, unlabeled)):
            assert out.grad is not None and bool(out.grad.abs().max() > 0), f"{case}: no gradient reached the backbone's output ({name} batch)"
            check_grads({"dfeat": out.grad}, {"dfeat": r[2]["dfeat"]}, {}, f"{case}, {what}: backbone output, {name} batch", rel=2e-2)
