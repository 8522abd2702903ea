"""Batched inference driver (SURVEY 8f-1): table schema / context fix-up on the CPU, the CUDA-graph chunk loop on the GPU."""
import numpy as np
import pytest
import torch

from lightning_pose_b200.utils.predictions import PredictionHandler, frame_range_for_rank, make_dlc_pandas_index


def test_frame_ranges_cover_the_video_once():
    assert frame_range_for_rank(100_000, 0, 8) == (0, 12_500) and frame_range_for_rank(100_000, 7, 8) == (87_500, 100_000)
    for n, w in ((10, 4), (7, 8), (96, 1), (1001, 3)):
        spans = [frame_range_for_rank(n, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_prediction_table_schema_matches_reference_columns():
    # reference utils/predictions.py:180-206: cols are (bp0_x, bp0_y, bp0_likelihood, bp1_x, ...)
    kp = np.arange(12, dtype=np.float64).reshape(2, 6)
    cf = np.array([[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]])
    arr = PredictionHandler.make_pred_arr_undo_resize(kp, cf)
    assert arr.shape == (2, 9)
    np.testing.assert_array_equal(arr[0], [0, 1, 0.1, 2, 3, 0.2, 4, 5, 0.3])
    idx = make_dlc_pandas_index("heatmap", ["nose", "tail", "paw"])
    assert idx.names == ["scorer", "bodyparts", "coords"]
    assert list(idx[:4]) == [("heatmap_tracker", "nose", "x"), ("heatmap_tracker", "nose", "y"), ("heatmap_tracker", "nose", "likelihood"), ("heatmap_tracker", "tail", "x")]
    h = PredictionHandler(["nose", "tail", "paw"], frame_count=2)
    df = h([(torch.from_numpy(kp[:1]), torch.from_numpy(cf[:1])), (torch.from_numpy(kp[1:]), torch.from_numpy(cf[1:]))])
    assert df.shape == (2, 9) and float(df.iloc[1, 5]) == 0.5
    # the device-table route gives the same frame
    df2 = h.dataframe(torch.from_numpy(arr))
    assert df2.equals(df)


def test_context_shift_fixup_matches_reference_rule():
    # reference :146-178: row i of a context model is frame i+2; pad the first two with row 0, last two with row -3
    h = PredictionHandler(["a"], frame_count=6, model_type="heatmap_mhcrnn")
    stacked = torch.arange(6, dtype=torch.float32).reshape(6, 1) * 10  # rows for frames 2..7 (last two are junk)
    fixed = h.fix_context_preds_confs(stacked.clone())
    assert fixed.flatten().tolist() == [0.0, 0.0, 0.0, 10.0, 10.0, 10.0]
    z = h.fix_context_preds_confs(stacked.clone(), zero_pad_confidence=True)
    assert z.flatten().tolist() == [0.0, 0.0, 0.0, 10.0, 0.0, 0.0]
    h2 = PredictionHandler(["a"], frame_count=8, model_type="heatmap_mhcrnn")  # fewer rows than frames: pad with row 0
    assert h2.fix_context_preds_confs(stacked.clone()).flatten().tolist() == [0.0, 0.0, 0.0, 10.0, 20.0, 30.0, 0.0, 0.0]


def test_batched_predictor_refuses_bad_single_view_chunks():
    """One view takes the tensor form's checks of several: the chunk's length, the view count of (T, V, 3, h, w) frames
    and the (T, 4) box, all refused before anything is enqueued (the head stays on the CPU)."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    bp = BatchedPredictor(HeatmapHead("vits_dino", 64, 5), 5, 20, 4, (32, 32))
    with pytest.raises(ValueError, match="fixed-size"):
        bp.feed(torch.zeros(3, 64, 2, 2))
    with pytest.raises(ValueError, match=r"expected \(T, 1, 3, h, w\)"):
        bp.feed(torch.zeros(4, 2, 3, 32, 32))
    with pytest.raises(ValueError, match=r"bbox must be \(4, 4\)"):
        bp.feed(torch.zeros(4, 64, 2, 2), torch.zeros(4, 8))
    with pytest.raises(ValueError, match=r"bbox must be \(4, 4\)"):
        bp.feed(torch.zeros(4, 64, 2, 2), torch.zeros(3, 4))


def test_context_predictor_refuses_a_chunk_of_the_wrong_length():
    from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    bp = BatchedPredictor(HeatmapMHCRNNHead("vits_dino", 64, 5), 5, 20, 4, (32, 32))
    with pytest.raises(ValueError, match="fixed-size"):
        bp.feed(torch.zeros(5, 64, 2, 2))


@pytest.mark.gpu
def test_batched_predictor_graph_refuses_a_chunk_unlike_its_capture():
    """A replay copies the chunk into the captured input, which would cast fp32 features to the bf16 of the capture, so
    graph mode refuses the chunk and names both forms; eager mode takes either."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor

    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    head = HeatmapHead("resnet50", 512, 17).to(dev).eval()
    feats = torch.randn(8, 512, 4, 4, device=dev) * 0.5
    graph = BatchedPredictor(head, 17, 16, 8, (128, 128))
    graph.feed(feats.bfloat16())
    with pytest.raises(ValueError, match=r"captured for tensor \(8, 512, 4, 4\) torch.bfloat16, .*; this chunk is tensor \(8, 512, 4, 4\) torch.float32"):
        graph.feed(feats)
    assert int(graph.cursor) == 8
    eager = BatchedPredictor(head, 17, 16, 8, (128, 128), use_graph=False)
    eager.feed(feats.bfloat16())
    eager.feed(feats)
    assert int(eager.cursor) == 16


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [True, False])
def test_batched_predictor_matches_oracle(use_graph):
    """cfg-5 style chunk loop (here 20 frames in chunks of 8, the last one padded) against the CPU oracle."""
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead
    from lightning_pose_b200.utils.predictions import BatchedPredictor
    from oracle import lp_oracle as O

    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    k, n, chunk, c, fh, fw, img = 17, 20, 8, 512, 4, 4, 128
    head = HeatmapHead("resnet50", c, k)
    for layer in list(head.upsampling_layers)[1:]:
        torch.nn.init.xavier_uniform_(layer.weight, gain=3.0)
    feats = torch.randn(n, c, fh, fw) * 0.5
    bbox = torch.tensor([[3.0, 5.0, 200.0, 260.0]]).repeat(n, 1) + torch.arange(n)[:, None]
    deconvs = list(head.upsampling_layers)[1:]
    hm = O.head_forward(feats, [d.weight.detach() for d in deconvs], [d.bias.detach() for d in deconvs])
    kp_ref, cf_ref = O.decode_softargmax(hm, 2, 1000.0)
    kp_ref = O.model_to_frame(kp_ref, bbox, img, img)
    head = head.to(dev).eval()
    bp = BatchedPredictor(head, k, n, chunk, (img, img), use_graph=use_graph)
    pad = (-n) % chunk
    f_dev = torch.cat([feats, feats[-1:].repeat(pad, 1, 1, 1)]).to(dev)
    b_dev = torch.cat([bbox, bbox[-1:].repeat(pad, 1)]).to(dev)
    bp.run((f_dev[i : i + chunk], b_dev[i : i + chunk]) for i in range(0, n + pad, chunk))
    kp, cf = bp.results()
    np.testing.assert_allclose(kp.cpu().numpy(), kp_ref.numpy(), rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(cf.cpu().numpy(), cf_ref.numpy(), rtol=1e-4, atol=1e-5)
    assert int(bp.cursor) == n + pad
    df = PredictionHandler([f"bp{i}" for i in range(k)], n)(iter([(kp, cf)]))
    assert df.shape == (n, 3 * k)
    np.testing.assert_allclose(df.to_numpy(), PredictionHandler([f"bp{i}" for i in range(k)], n).dataframe(bp.table).to_numpy())
