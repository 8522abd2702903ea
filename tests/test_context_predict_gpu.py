"""GPU: BatchedPredictor's context mode (MHCRNN models; csrc/predict.cu lpb_pack_context_predictions) against
tests/golden/context_predict.npz, which holds the reference's own final tables, and against the eager composition of
the existing parts run window by window the way the reference's reader and predict_step do."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import context_predict_oracle as CO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN_CASES = [f"{tag}_{c[0]}" for tag, *_ in CO.HEADS for c in CO.CASES if not (tag == "uf2" and c[0] == "issue_example")]


def n_windows(n, s):
    """PrepareDALI.num_iters for a context predict reader (step S - 4)."""
    t = s - 4
    return n if t == 1 else -(-(n - s) // t) + 1


def golden_head(g, tag):
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

    arch, uf = {h[0]: (h[1], h[2]) for h in CO.HEADS}[tag]
    head = HeatmapMHCRNNHead(arch, CO.C, CO.K, upsampling_factor=uf)
    sd = {k[len(tag) + 7 :]: torch.from_numpy(g[k]) for k in g.files if k.startswith(f"{tag}_param_")}
    missing, unexpected = head.load_state_dict(sd, strict=False)
    assert not unexpected and all(".layers." in m for m in missing), (missing, unexpected)
    return head.to(DEV).eval()


def padded(x, total, fill):
    """x (N, ...) extended to ``total`` rows with ``fill``."""
    if total <= x.shape[0]:
        return x[:total]
    return torch.cat([x, fill.expand(total - x.shape[0], *x.shape[1:])])


def run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=True, sub_chunk=None, features_of=None):
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    t = s - 4
    chunks = math.ceil(n / t)
    f_all = padded(feats, chunks * t, pad[None])
    b_all = padded(bbox, chunks * t, bbox[-1:])
    bp = BatchedPredictor(head, head.head_sf.out_channels, n, t, image_hw, use_graph=use_graph, sub_chunk=sub_chunk,
                          features_of=features_of)
    bp.run((f_all[i : i + t], b_all[i : i + t]) for i in range(0, chunks * t, t))
    torch.cuda.synchronize()
    assert int(bp.cursor) == chunks * t
    return bp


def eager_windows(head, feats, pad, bbox, n, s, image_hw, decode=None, windows=None):
    """Per-window tuples of the reference's reader + predict_step, composed from existing parts: forward_sequence on each
    window of S frames (step S - 4, padded with ``pad``), decode, the strict-greater selection, remap_keypoints with the
    window's box rows (the middle S - 4 are used).  ``windows``: how many (default: the reader's count for n frames)."""
    from lightning_pose_b200 import ops

    t, k = s - 4, head.head_sf.out_channels
    decode = decode or head.run_subpixelmaxima
    out = []
    with torch.no_grad():
        for j in range(n_windows(n, s) if windows is None else windows):
            idx = torch.arange(j * t, j * t + s)
            win = torch.stack([feats[i] if i < n else pad for i in idx.tolist()])
            rows = bbox[idx.clamp(max=n - 1)]
            sf, mf = head.forward_sequence(win)
            kp_sf, cf_sf = decode(sf)
            kp_mf, cf_mf = decode(mf)
            kp_sf, cf_sf, kp_mf, cf_mf = (x.to(DEV) for x in (kp_sf, cf_sf, kp_mf, cf_mf))
            pick = torch.gt(cf_mf, cf_sf)
            kp = torch.where(pick[..., None], kp_mf.reshape(-1, k, 2), kp_sf.reshape(-1, k, 2)).reshape(-1, 2 * k)
            cf = torch.where(pick, cf_mf, cf_sf)
            out.append((ops.remap_keypoints(kp, None, rows, image_hw[0], image_hw[1]), cf))
    return out


def fixed_table(windows, n, k):
    """The host form: vstack, trim, fix_context_preds_confs, interleave -> (N, 3K)."""
    from lightning_pose_b200.utils.predictions import PredictionHandler

    ph = PredictionHandler([f"bp{i}" for i in range(k)], n, model_type="heatmap_mhcrnn")
    kp = ph.fix_context_preds_confs(torch.vstack([w[0] for w in windows])[:n])
    cf = ph.fix_context_preds_confs(torch.vstack([w[1] for w in windows])[:n])
    return torch.from_numpy(ph.make_pred_arr_undo_resize(kp.cpu().numpy(), cf.cpu().numpy()))


def golden_inputs(g, p):
    n, s, _, ih, iw = (int(v) for v in g[f"{p}_meta"])
    t = lambda name: torch.from_numpy(g[f"{p}_{name}"]).to(DEV)
    return t("features"), t("pad"), t("bbox"), n, s, (ih, iw)


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_context_predictor_matches_reference_golden(golden, case, use_graph):
    g = golden("context_predict")
    head = golden_head(g, case.split("_")[0])
    feats, pad, bbox, n, s, image_hw = golden_inputs(g, case)
    bp = run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=use_graph)
    kp, cf = bp.results()
    np.testing.assert_allclose(kp.cpu().numpy(), g[f"{case}_kp"], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(cf.cpu().numpy(), g[f"{case}_conf"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("case", ["uf1_r_n_minus_1", "uf2_r_lt_n", "uf1_issue_example"])
def test_context_predictor_graph_equals_eager_and_reruns(golden, case):
    g = golden("context_predict")
    head = golden_head(g, case.split("_")[0])
    feats, pad, bbox, n, s, image_hw = golden_inputs(g, case)
    graph = run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=True)
    again = run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=True)
    eager = run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=False)
    assert torch.equal(graph.table, eager.table) and torch.equal(graph.table, again.table)
    assert graph.launches_per_chunk is not None and graph.launches_per_chunk >= 8
    sub = run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=True, sub_chunk=5)  # sub-chunks, same table
    assert torch.equal(sub.table, graph.table)


@pytest.mark.parametrize("case", ["uf1_r_ge_n", "uf1_r_lt_n", "uf2_r_n_minus_1", "uf2_n5", "uf2_n_lt_s"])
def test_context_predictor_matches_eager_composition(golden, case):
    from lightning_pose_b200.utils.predictions import PredictionHandler

    g = golden("context_predict")
    head = golden_head(g, case.split("_")[0])
    feats, pad, bbox, n, s, image_hw = golden_inputs(g, case)
    bp = run_predictor(head, feats, pad, bbox, n, s, image_hw)
    windows = eager_windows(head, feats, pad, bbox, n, s, image_hw)
    want = fixed_table(windows, n, CO.K)
    np.testing.assert_allclose(bp.table.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
    # the final table's DataFrame equals the reference call form on the per-window tuples
    names = [f"bp{i}" for i in range(CO.K)]
    ph = PredictionHandler(names, n, model_type="heatmap_mhcrnn")
    np.testing.assert_allclose(ph.dataframe(bp.table, frame_aligned=True).to_numpy(), ph(windows).to_numpy(), rtol=1e-5, atol=1e-5)


def test_context_predictor_computes_each_frame_once(golden):
    g = golden("context_predict")
    head = golden_head(g, "uf1")
    feats, pad, bbox, n, s, image_hw = golden_inputs(g, "uf1_issue_example")
    seen = []

    def features_of(x):
        seen.append(x.shape[0])
        return x

    run_predictor(head, feats, pad, bbox, n, s, image_hw, use_graph=False, features_of=features_of)
    assert seen == [s - 4] * math.ceil(n / (s - 4))


def test_pack_context_kernel_selection_nan_and_edges():
    """The kernel alone: strict-greater selection (NaN keeps sf), the remap, and the rows one call fills."""
    from lightning_pose_b200 import ops

    n, t, k = 9, 8, 3  # S = 12: R = 8 < N = 9, rows 0, 1 and 8 hold frame 2
    kp_sf = torch.arange(t * 2 * k, dtype=torch.float32, device=DEV).reshape(t, 2 * k)
    kp_mf = kp_sf + 1000.0
    cf_sf = torch.full((t, k), 0.5, device=DEV)
    cf_mf = torch.tensor([[0.6, 0.5, float("nan")]], device=DEV).repeat(t, 1)
    bbox = torch.tensor([[10.0, 20.0, 32.0, 64.0]], device=DEV).repeat(t, 1)
    table = torch.full((n, 3 * k), -1.0, device=DEV)
    cursor = torch.full((1,), 4, dtype=torch.int64, device=DEV)  # output frames 2 .. 9
    ops.pack_context_predictions(kp_sf, cf_sf, kp_mf, cf_mf, bbox, 64, 32, table, t, cursor=cursor)
    assert int(cursor) == 4 + t
    tab = table.cpu().reshape(n, k, 3)
    sel = torch.where(torch.tensor([True, False, False])[None, :, None], kp_mf.cpu().reshape(t, k, 2), kp_sf.cpu().reshape(t, k, 2))
    x = sel[..., 0] / 32 * 64 + 10  # model -> frame: x / model_width * w + x0
    y = sel[..., 1] / 64 * 32 + 20
    for row, frame in [(0, 2), (1, 2), (2, 2), (7, 7), (8, 2)]:
        o = frame - 2
        np.testing.assert_allclose(tab[row, :, 0].numpy(), x[o].numpy(), rtol=1e-6)
        np.testing.assert_allclose(tab[row, :, 1].numpy(), y[o].numpy(), rtol=1e-6)
        np.testing.assert_array_equal(tab[row, :, 2].numpy(), np.array([0.6, 0.5, 0.5], np.float32))


def test_context_predictor_bf16_config3_shape():
    """vits_dino features (., 384, 16, 16) bf16 -> 64 x 64 heatmaps, upsampling_factor 1: the table's keypoints agree with
    the oracle's decode of the same heatmaps to sub-pixel level."""
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from oracle import lp_oracle as O

    torch.manual_seed(7)
    k, n, s, img = 17, 70, 36, (256, 256)
    head = HeatmapMHCRNNHead("vits_dino", 384, k, upsampling_factor=1)
    for layer in list(head.head_sf.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    head = head.to(DEV).eval()
    feats = (torch.randn(n, 384, 16, 16, device=DEV) * 0.5).bfloat16()
    pad = torch.zeros(384, 16, 16, device=DEV, dtype=torch.bfloat16)
    bbox = torch.tensor([[0.0, 0.0, 256.0, 256.0]], device=DEV).repeat(n, 1)
    bp = run_predictor(head, feats, pad, bbox, n, s, img)
    oracle_decode = lambda hm: O.decode_softargmax(hm.cpu(), 2, 1000.0)
    want = fixed_table(eager_windows(head, feats, pad, bbox, n, s, img, decode=oracle_decode), n, k).float().reshape(n, k, 3)
    got = bp.table.cpu().reshape(n, k, 3)
    ok = want[..., 2] > 0.5
    assert int(ok.sum()) >= 10  # enough confident keypoints for a meaningful comparison
    assert float((got[..., :2] - want[..., :2]).abs().amax(-1)[ok].max()) < 0.5
    np.testing.assert_allclose(got[..., 2].numpy(), want[..., 2].numpy(), atol=2e-3)


def test_context_predictor_crop_mode():
    """uint8 frames + a box table: crop inside the chunk, against crop -> forward_sequence -> ... composed eagerly."""
    from lightning_pose_b200 import ops
    from lightning_pose_b200.data.bboxes import crop_and_resize_frames
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    torch.manual_seed(11)
    k, c, img, n, s, fh, fw = 7, 128, 64, 23, 12, 120, 160
    head = HeatmapMHCRNNHead("vits_dino", c, k, upsampling_factor=1)
    for prm in head.head_sf.parameters():
        torch.nn.init.normal_(prm, std=0.3)
    head = head.to(DEV).eval()
    channel, scale = torch.arange(c, device=DEV) % 3, torch.randn(c, device=DEV)[None, :, None, None]

    def features_of(frames):  # stand-in backbone of elementwise ops: (T, 3, 64, 64) -> (T, 128, 4, 4)
        return (F.avg_pool2d(frames.float(), 16)[:, channel] * scale).contiguous()

    gen = torch.Generator(device=DEV).manual_seed(5)
    video = torch.randint(0, 256, (n, fh, fw, 3), dtype=torch.uint8, device=DEV, generator=gen)
    xy = torch.rand(n, 2, device=DEV, generator=gen) * 60
    boxes = torch.cat([xy.floor(), torch.full((n, 2), 50.0, device=DEV) + torch.arange(n, device=DEV)[:, None]], 1)
    t = s - 4
    chunks = math.ceil(n / t)
    frames = padded(video, chunks * t, torch.zeros(1, fh, fw, 3, dtype=torch.uint8, device=DEV))
    tables = {}
    for use_graph in (True, False):
        bp = BatchedPredictor(head, k, n, t, (img, img), features_of=features_of, use_graph=use_graph, bboxes=boxes, frame_hw=(fh, fw))
        bp.run(frames[i : i + t] for i in range(0, chunks * t, t))
        torch.cuda.synchronize()
        tables[use_graph] = bp.table.clone()
    assert torch.equal(tables[True], tables[False])
    # eager: crop every frame of the padded stream to its row (rows past the end repeat the last), then the reference form
    total = (n_windows(n, s) - 1) * t + s
    stream = padded(video, total, torch.zeros(1, fh, fw, 3, dtype=torch.uint8, device=DEV))
    rows = padded(boxes, total, boxes[-1:])
    with torch.no_grad():
        crops, clamped = crop_and_resize_frames(ops.frames_normalize(stream), rows, [img, img])
        feats = features_of(crops)
    want = fixed_table(eager_windows(head, feats, feats[-1], clamped, total, s, (img, img), windows=n_windows(n, s)), n, k)
    np.testing.assert_allclose(tables[False].cpu().numpy(), want.numpy(), rtol=1e-4, atol=2e-3)
