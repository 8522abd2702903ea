"""Batched inference: the ``predict_new_vids`` path of the reference on one GPU per frame range (SURVEY 8f-1).

Reference flow (``lightning_pose/utils/predictions.py``): ``pl.Trainer.predict`` over a DALI loader returns a Python
list of per-batch ``(keypoints, confidences)`` tuples (:472-521); ``PredictionHandler`` stacks them on the host
(:97-144), trims the padded tail, fixes the two-frame shift of context models (:146-178), interleaves into
``(x, y, likelihood)`` columns with numpy (:180-206) and labels them with a DLC-style MultiIndex (:551-570).  It always
runs with ``devices=1`` (:352, :474).

Here one *chunk* of ``T`` frames is one CUDA-graph replay: head -> soft-argmax decode -> model->frame remap ->
rows of a preallocated ``(N, 3K)`` device table at a device-resident cursor (``lpb_pack_predictions``).  Nothing
returns to the host until the video is done; then ONE device->host copy of the table.  The table's column order is the
reference's, so ``PredictionHandler.make_pred_arr_undo_resize`` / ``make_dlc_pandas_index`` below produce the same CSV.
Multi-GPU (the reference itself never predicts on more than one device): ``BatchedPredictor(..., shard=(rank, world))``
predicts rank ``rank``'s contiguous rows ``frame_range_for_rank(N, rank, world)`` into a full-length table at global rows,
feeding ``feed_range``: its own frames, plus for a context model a 2-frame halo at each edge.  ``gather()`` is one
all-gather of every rank's rows into the full table on every rank, then the context edge fill
(``fill_context_edges``): each edge row whose source frame lies in another shard is copied from that frame's own row.
The gathered table equals the one-GPU table bit for bit.
"""
from __future__ import annotations

import operator
from typing import Callable, Iterable, Sequence

import numpy as np
import torch

from lightning_pose_b200 import ops

__all__ = ["BatchedPredictor", "FramePredictor", "PredictionHandler", "make_dlc_pandas_index", "frame_range_for_rank",
           "shard_feed_range", "context_edge_fill", "fill_context_edges"]


def frame_range_for_rank(n_frames: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, near-equal frame ranges: [start, stop) of ``rank`` (cfg 5: 100,000 frames -> 12,500 per GPU)."""
    per = -(-n_frames // max(world, 1))
    return min(rank * per, n_frames), min((rank + 1) * per, n_frames)


def _context_rows(n_frames: int, chunk: int) -> int:
    """R, the rows the reference's context reader produces for windows of S = T + 4 frames with step T (one window per
    frame when T = 1): ``context_source_row`` in csrc/predict.cu."""
    t = chunk
    return n_frames if t == 1 else t * (-(-(n_frames - t - 4) // t) + 1)


def _context_source(row: int, n_frames: int, r_rows: int) -> int:
    """The frame whose prediction row ``row`` of the final context table holds (the rule of ``pack_context_kernel``)."""
    if r_rows >= n_frames:
        return min(max(row, 2), n_frames - 3)
    return row if 2 <= row <= r_rows - 1 else 2


def shard_feed_range(n_frames: int, chunk: int, rank: int, world: int, context: bool = False) -> tuple[int, int]:
    """[lo, hi): the frames shard ``rank`` of ``world`` feeds, in chunks of ``chunk`` from frame lo, the last chunk padded
    past hi as the one-GPU caller pads the video's end.  A frame model feeds its own rows' frames.  A context model's
    row f needs frames f - 2 .. f + 2, so its shard feeds a 2-frame halo on each side, clamped to the video.  When
    R = N - 1, row N - 2 reads the first padding frame N: a shard that owns that row starts one frame earlier if its
    chunks would otherwise end exactly at frame N, so that frame N is fed and frame N - 2 is predicted."""
    a, b = frame_range_for_rank(n_frames, rank, world)
    if not context or a == b:
        return a, b
    lo, hi = max(a - 2, 0), min(b + 2, n_frames)
    if _context_rows(n_frames, chunk) == n_frames - 1 and a <= n_frames - 2 < b and (n_frames - lo) % chunk == 0:
        lo -= 1  # lo >= 1 here: lo = 0 would need N = 0 and N = 1 (mod T), so T = 1, where R = N
    return lo, hi


def context_edge_fill(n_frames: int, chunk: int, world: int) -> list[tuple[int, int]]:
    """(row, source row) pairs that complete a context table gathered from ``world`` shards: every edge row (0, 1, the
    last four) whose source frame's own row belongs to another shard.  The kernel writes a frame's prediction to all
    its rows, but only the shard that owns the frame's row computes it from the right window; another shard's rows
    hold a halo frame's prediction (or none) there.  Empty for one shard."""
    n, per = n_frames, -(-n_frames // max(world, 1))
    r_rows = _context_rows(n, chunk)
    pairs = []
    for row in sorted({0, 1, *range(max(n - 4, 0), n)}):
        src = _context_source(row, n, r_rows)
        if row // per != src // per:
            pairs.append((row, src))
    return pairs


def fill_context_edges(table: torch.Tensor, chunk: int, world: int) -> torch.Tensor:
    """Apply ``context_edge_fill`` to an (N, 3K) context table on its device, in place (one gather, one scatter)."""
    pairs = context_edge_fill(table.shape[0], chunk, world)
    if pairs:
        dst, src = (torch.tensor(rows, dtype=torch.int64, device=table.device) for rows in zip(*pairs))
        table.index_copy_(0, dst, table.index_select(0, src))
    return table


def make_dlc_pandas_index(model_type: str, keypoint_names: Sequence[str]):
    """``[scorer, bodyparts, coords]`` MultiIndex with coords (x, y, likelihood) (reference :551-570)."""
    import pandas as pd

    return pd.MultiIndex.from_product([[f"{model_type}_tracker"], list(keypoint_names), ["x", "y", "likelihood"]],
                                      names=["scorer", "bodyparts", "coords"])


class PredictionHandler:
    """Video-side mirror of the reference's ``PredictionHandler`` (:41-329): same column schema, same context fix-up.

    ``frame_count`` is given directly (the reference counts the video's frames with OpenCV; video I/O is out of scope).
    ``view_names`` (the reference's ``cfg.data.view_names``) names the views of a multi-view video, in the order of the
    prediction columns: view v owns keypoint columns ``[v K, (v + 1) K)`` (reference :296-315).
    """

    def __init__(self, keypoint_names: Sequence[str], frame_count: int, model_type: str = "heatmap",
                 view_names: Sequence[str] | None = None) -> None:
        if keypoint_names is None:
            raise ValueError("must include `keypoint_names`")
        self.keypoint_names = list(keypoint_names)
        self.frame_count = int(frame_count)
        self.model_type = model_type
        self.view_names = list(view_names) if view_names is not None else None

    def _views(self) -> list[str]:
        if not self.view_names:
            raise ValueError("multi-view predictions need `view_names`")
        return self.view_names

    @property
    def do_context(self) -> bool:
        return self.model_type == "heatmap_mhcrnn"

    def fix_context_preds_confs(self, stacked: torch.Tensor, zero_pad_confidence: bool = False) -> torch.Tensor:
        """Context models predict frame i+2 at row i: shift by two and replicate the edges (reference :146-178)."""
        first = stacked[0:1].repeat(2, 1)
        combined = torch.cat([first, stacked[:-2]], dim=0)
        if combined.shape[0] == self.frame_count:
            combined[-2:, :] = combined[-3, :]
        else:
            n_pad = self.frame_count - combined.shape[0]
            combined = torch.cat([combined, combined[0:1].repeat(n_pad, 1)], dim=0)
        if zero_pad_confidence:
            combined[:2, :] = 0.0
            combined[-2:, :] = 0.0
        return combined

    @staticmethod
    def make_pred_arr_undo_resize(keypoints_np: np.ndarray, confidence_np: np.ndarray) -> np.ndarray:
        """(n, 2K) keypoints + (n, K) confidences -> (n, 3K) columns bp0_x, bp0_y, bp0_likelihood, ... (:180-206)."""
        assert keypoints_np.shape[0] == confidence_np.shape[0]
        assert keypoints_np.shape[1] == confidence_np.shape[1] * 2
        k = confidence_np.shape[-1]
        out = np.zeros((keypoints_np.shape[0], 3 * k))
        out[:, 0::3] = keypoints_np[:, 0::2]
        out[:, 1::3] = keypoints_np[:, 1::2]
        out[:, 2::3] = confidence_np
        return out

    def dataframe(self, table: torch.Tensor | np.ndarray, frame_aligned: bool = False):
        """(N, 3K) prediction table (device or host) -> DataFrame with the reference's columns.  ``frame_aligned``: the
        table is already final (row f is frame f, as a context-mode ``BatchedPredictor`` writes it), so the context
        shift-and-fill is skipped."""
        import pandas as pd

        arr = table.detach().cpu().numpy() if isinstance(table, torch.Tensor) else np.asarray(table)
        arr = arr[: self.frame_count]
        if self.do_context and not frame_aligned:
            k = len(self.keypoint_names)
            t = torch.from_numpy(arr)
            kp = self.fix_context_preds_confs(t.reshape(-1, k, 3)[:, :, :2].reshape(-1, 2 * k).clone())
            cf = self.fix_context_preds_confs(t.reshape(-1, k, 3)[:, :, 2].clone(), zero_pad_confidence=False)
            arr = self.make_pred_arr_undo_resize(kp.numpy(), cf.numpy())
        return pd.DataFrame(arr, columns=make_dlc_pandas_index(self.model_type, self.keypoint_names))

    def dataframes(self, table: torch.Tensor | np.ndarray, frame_aligned: bool = False) -> dict:
        """(N, 3 V K) multi-view prediction table -> ``{view_name: DataFrame}``, view v from columns [3 K v, 3 K (v + 1))."""
        w = 3 * len(self.keypoint_names)
        if table.shape[1] != w * len(self._views()):
            raise ValueError(f"table has {table.shape[1]} columns; {len(self._views())} views of {w} expected")
        return {name: self.dataframe(table[:, w * v : w * (v + 1)], frame_aligned) for v, name in enumerate(self._views())}

    def __call__(self, preds: Iterable[tuple[torch.Tensor, torch.Tensor]], is_multiview_video: bool = False):
        """Reference call form: a list of per-batch (keypoints, confidences) tuples -> DataFrame, or with
        ``is_multiview_video`` the (N, 2 V K) / (N, V K) stack split into ``{view_name: DataFrame}`` (:287-315)."""
        preds = list(preds)
        kp = torch.vstack([p[0] for p in preds])[: self.frame_count]
        cf = torch.vstack([p[1] for p in preds])[: self.frame_count]
        if self.do_context:
            kp = self.fix_context_preds_confs(kp)
            cf = self.fix_context_preds_confs(cf, zero_pad_confidence=False)
        import pandas as pd

        columns = make_dlc_pandas_index(self.model_type, self.keypoint_names)
        if not is_multiview_video:
            return pd.DataFrame(self.make_pred_arr_undo_resize(kp.cpu().numpy(), cf.cpu().numpy()), columns=columns)
        k = len(self.keypoint_names)
        if cf.shape[1] != k * len(self._views()):
            raise ValueError(f"predictions have {cf.shape[1]} keypoints; {len(self._views())} views of {k} expected")
        kp_np, cf_np = kp.cpu().numpy(), cf.cpu().numpy()
        return {name: pd.DataFrame(self.make_pred_arr_undo_resize(kp_np[:, 2 * k * v : 2 * k * (v + 1)], cf_np[:, k * v : k * (v + 1)]),
                                   columns=columns)
                for v, name in enumerate(self._views())}


def _graph_kernel_count(graph: torch.cuda.CUDAGraph) -> int:
    """Kernel nodes of a captured graph (driver API: cuGraphGetNodes / cuGraphNodeGetType)."""
    import ctypes as C

    cu = C.CDLL("libcuda.so.1")
    g = C.c_void_p(graph.raw_cuda_graph())
    n = C.c_size_t(0)
    if cu.cuGraphGetNodes(g, None, C.byref(n)) != 0:
        raise RuntimeError("cuGraphGetNodes failed")
    nodes = (C.c_void_p * n.value)()
    if cu.cuGraphGetNodes(g, nodes, C.byref(n)) != 0:
        raise RuntimeError("cuGraphGetNodes failed")
    kind = C.c_int(0)
    count = 0
    for node in nodes:
        if cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(kind)) != 0:
            raise RuntimeError("cuGraphNodeGetType failed")
        count += kind.value == 0  # CU_GRAPH_NODE_TYPE_KERNEL
    return count


class BatchedPredictor:
    """CUDA-graph chunk loop writing straight into a preallocated (N, 3 V K) device table, V = ``num_views``.

    ``head``: a ``HeatmapHead`` or ``HeatmapMHCRNNHead`` on the device, in eval mode.  Each ``feed`` is a chunk of
    exactly T = ``chunk`` video frames (``dali.base.predict.sequence_length`` = 96 in the reference config): the caller
    pads the last one and the table writer drops the surplus rows, at ``cursor``, a device int64 that each chunk
    advances, so nothing returns to the host until the video is done.  ``features_of`` maps the chunk's T V frames (frame-major,
    view-minor) to backbone features: None when the caller streams features, else a backbone, captured into the same
    graph.  With ``use_graph`` the first chunk is captured (``launches_per_chunk`` counts its kernels) and every chunk
    replays it, so every chunk must have the first one's form, shapes and dtypes.  The input forms:

    Tensor: (T V, ...) frames or features, or (T, V, 3, h, w) frames, and an optional (T, 4 V) ``bbox``, [x, y, h, w]
    per view, that maps keypoints back to the frame (default: the whole model image ``image_hw``).

    Views (reference ``predict_video(video_file=[one per view])``, ``utils/predictions.py:416-540``): V uint8
    (T, H_v, W_v, 3) views in a list or tuple, sizes fixed by the first chunk, normalised by one launch inside the chunk
    (``ops.frames_normalize_views``); each view's box is its whole frame.

    Crop (crop-zoom models, reference ``predict_video(..., bbox_file=...)``, ``utils/predictions.py:455-470`` and
    ``data/video/dali.py:332-380``): with ``bboxes``, the video's (N, 4) device table (``compute_bboxes`` /
    ``smooth_bboxes``), and ``frame_hw``, uint8 (T, H, W, 3) full frames and no ``bbox``.  One launch inside the chunk
    crops each frame to its row at the cursor (rows past the end repeat the last) and resizes it; the clamped boxes it
    writes map the keypoints back.  Both ingests write ``crop_dtype`` (float32, bfloat16 or float16), channels-last if
    ``crop_channels_last``.  Features of the backbone's dtype pick the head's kernels: bf16, and fp16 (the reference's
    ``precision="fp16"``, ``torch.autocast(float16)``) run on the 16-bit tensor-core head, fp32 on the 3xTF32 one.

    The body runs ``sub_chunk`` frames at a time.  Frame body (``HeatmapHead``; for V > 1 the multi-view transformer's,
    ``features_of=model.forward_vit``, or a tracker's that folds views into the batch): head -> decode -> remap ->
    ``lpb_pack_predictions``; view v owns columns [3 K v, 3 K (v + 1)), the reference's per-view split
    (``view_tables``, ``PredictionHandler.dataframes``).

    Regression body (``LinearRegressionHead``, one view; reference ``RegressionTracker.predict_step``): head ->
    ``lpb_pack_predictions`` with a likelihood of 0.0, the reference's zeros, and the keypoints in model pixels as
    ``predict_step`` returns them (it has no model -> frame remap).  A ``bbox``, crop mode and more than one view raise.

    Context body (``HeatmapMHCRNNHead``, one view; reference ``HeatmapTrackerMHCRNN.predict_step`` over windows of
    S = T + 4 frames with step T, ``dali.context.predict.sequence_length``): T counts NEW frames; chunk j yields frames
    j T - 2 .. j T + T - 3.  The two / four frames before a chunk stay on the device (their single-frame decode, boxes
    and W_f / W_b maps), so every frame passes through ``features_of``, ``head_sf`` and the maps once.
    ``lpb_pack_context_predictions`` writes each frame's selected, remapped prediction to every row the reference's
    ``fix_context_preds_confs`` gives it: after the last chunk ``table`` is the reference's final table
    (``PredictionHandler.dataframe(table, frame_aligned=True)``).  With R = T (ceil((N - S) / T) + 1): R >= N: row f is
    frame clamp(f, 2, N - 3); R < N: row f is frame f for 2 <= f <= R - 1 and frame 2 otherwise (the reference pads the
    tail with its first row).  Only when R = N - 1 does a row (N - 2) depend on frame N, the first padding frame of the
    last chunk; the reference reads the zero-filled frame its reader pads with there, so the caller's padding matters in
    that case only.  N < 5 raises (the reference has no window to predict from).

    Shards (``shard=(rank, world)``; the default (0, 1) is the whole video): the predictor owns rows
    ``rows = frame_range_for_rank(N, rank, world)`` of the full-length table and is fed ``feed_range``
    (``shard_feed_range``), in chunks starting at its first frame, the last one padded as above.  The device cursor
    starts there, so every writer and the crop ingest work in global rows unchanged.  A context shard's first two output
    frames come from the zero halo.  They land in rows of other shards, which the gather overwrites, and in edge rows
    whose source frame lies in another shard (when R < N frame 2's tail rows [R, N) may be the shard's own), which
    the edge fill overwrites: the fill, not row ownership, is what discards them.  ``gather()`` assembles the table on
    every rank.
    """

    def __init__(self, head, num_keypoints: int, n_frames: int, chunk: int, image_hw: tuple[int, int],
                 features_of: Callable[[torch.Tensor], torch.Tensor] | None = None, device=None, use_graph: bool = True,
                 sub_chunk: int | None = None, bboxes: torch.Tensor | None = None, frame_hw: tuple[int, int] | None = None,
                 crop_dtype: torch.dtype = torch.float32, crop_channels_last: bool = False, num_views: int = 1,
                 shard: tuple[int, int] = (0, 1)) -> None:
        from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
        from lightning_pose_b200.models.heads.regression import LinearRegressionHead

        self.head, self.k, self.n_frames, self.chunk = head, int(num_keypoints), int(n_frames), int(chunk)
        self.context = isinstance(head, HeatmapMHCRNNHead)
        self.regression = isinstance(head, LinearRegressionHead)
        self.num_views = int(num_views)
        if self.regression and self.num_views > 1:
            raise ValueError("multiview prediction is not supported for regression models")
        if self.regression and bboxes is not None:
            raise ValueError("bbox cropping is not supported for regression models")
        if self.context and self.num_views > 1:
            raise ValueError("context prediction is not supported for multiview models")
        if self.context and self.n_frames < 5:
            raise ValueError(f"a context model needs at least 5 frames to predict from; the video has {self.n_frames}")
        if self.chunk < 1:
            raise ValueError(f"chunk must be >= 1; got {self.chunk}")
        if self.num_views < 1:
            raise ValueError(f"num_views must be >= 1; got {self.num_views}")
        rank, world = (int(v) for v in shard)
        if world < 1 or not 0 <= rank < world:
            raise ValueError(f"shard must be (rank, world) with 0 <= rank < world; got {tuple(shard)}")
        self.shard = (rank, world)
        self.rows = frame_range_for_rank(self.n_frames, rank, world)
        self.feed_range = shard_feed_range(self.n_frames, self.chunk, rank, world, self.context)
        # frames per head / decode call inside a chunk: small enough that the heatmaps written by the head are still in
        # the 126 MB L2 when the decode reads them (None: the whole chunk at once)
        self.sub_chunk = int(sub_chunk) if sub_chunk else self.chunk
        self.image_hw = (int(image_hw[0]), int(image_hw[1]))
        self.features_of = features_of
        self.device = torch.device(device) if device is not None else next(head.parameters()).device
        self.crop_dtype, self.crop_channels_last = crop_dtype, bool(crop_channels_last)
        # the table is the first N rows of ``world`` equal blocks, the all-gather's outputs (the last one padded)
        per = -(-self.n_frames // world)
        self._blocks = torch.zeros((per * world, 3 * self.k * self.num_views), dtype=torch.float32, device=self.device)
        self.table = self._blocks[: self.n_frames]
        self.cursor = torch.full((1,), self.feed_range[0], dtype=torch.int64, device=self.device)
        self.use_graph = use_graph
        self._graph = self._static = self._captured = None
        self.launches_per_chunk = None
        self._image_bbox = self._whole_frames([self.image_hw] * self.num_views)
        self._view_hw = self._view_bbox = None  # uint8 views: their frame sizes and boxes, fixed by the first chunk
        self.bboxes = None
        if bboxes is not None:
            if self.num_views > 1:
                raise ValueError("bbox cropping is not supported for multiview models")
            if frame_hw is None or features_of is None:
                raise ValueError("crop mode needs frame_hw (the full frame size) and features_of (frames -> features)")
            self.bboxes = ops._bbox_table(bboxes, "bboxes")
            if self.bboxes.shape[0] != self.n_frames:
                raise ValueError(f"bboxes has {self.bboxes.shape[0]} rows but the video has {self.n_frames} frames")
            self.frame_hw = (int(frame_hw[0]), int(frame_hw[1]))
        if self.regression:  # the likelihood column
            self._zero_conf = torch.zeros((self.chunk, self.k), dtype=torch.float32, device=self.device)
        if self.context:  # the halo buffers; the maps' are sized by the first chunk's maps
            t, k, dev = self.chunk, self.k, self.device
            self._wf = self._wb = None
            self._kp_sf = torch.zeros((t + 2, 2 * k), dtype=torch.float32, device=dev)
            self._cf_sf = torch.zeros((t + 2, k), dtype=torch.float32, device=dev)
            self._box = torch.zeros((t + 2, 4), dtype=torch.float32, device=dev)
            self._idx = (torch.arange(t, device=dev)[:, None] + torch.arange(5, device=dev)[None, :]).to(torch.int32)

    def _whole_frames(self, sizes: list[tuple[int, int]]) -> torch.Tensor:
        """(T, 4 V) boxes [0, 0, h, w] of whole frames of the views' ``sizes``."""
        row = [float(s) for h, w in sizes for s in (0, 0, h, w)]
        return torch.tensor([row], dtype=torch.float32, device=self.device).repeat(self.chunk, 1)

    def _halo(self) -> tuple[tuple[torch.Tensor, int], ...]:
        """The context buffers and their halo rows: row b of the maps holds frame cursor - 4 + b, of the others frame
        cursor - 2 + b."""
        return ((self._wf, 4), (self._wb, 4), (self._kp_sf, 2), (self._cf_sf, 2), (self._box, 2))

    def _reset(self) -> None:
        self.cursor.fill_(self.feed_range[0])
        self.table.zero_()
        if self.context:
            for buf, _ in self._halo():
                buf.zero_()

    def _inputs(self, x, bbox) -> tuple[str, tuple[torch.Tensor, ...]]:
        """A chunk as fed -> (its form, its checked tensors): "crop" (frames,), "views" (*views, boxes) or
        "tensor" (x, boxes)."""
        t, v = self.chunk, self.num_views
        if self.bboxes is not None:
            if bbox is not None:
                raise ValueError("crop mode takes its boxes from the `bboxes` table given at construction")
            if x.dtype != torch.uint8 or tuple(x.shape) != (t, *self.frame_hw, 3):
                raise ValueError(f"crop mode expects uint8 ({t}, {self.frame_hw[0]}, {self.frame_hw[1]}, 3) frames; got {tuple(x.shape)} {x.dtype}")
            return "crop", (x,)
        if isinstance(x, (list, tuple)):
            if bbox is not None:
                raise ValueError("uint8 views take their boxes from the views' frame sizes")
            if len(x) != v:
                raise ValueError(f"expected {v} views; got {len(x)}")
            if self.features_of is None:
                raise ValueError("uint8 views need features_of (frames -> features)")
            for view in x:
                if view.dtype != torch.uint8 or view.dim() != 4 or view.shape[-1] != 3:
                    raise ValueError(f"each view must be uint8 (T, H, W, 3); got {tuple(view.shape)} {view.dtype}")
            counts = [view.shape[0] for view in x]
            if len(set(counts)) != 1:
                raise ValueError(f"all views must have the same frame count; got {counts}")
            if counts[0] != t:
                raise ValueError(f"chunks are fixed-size ({t} frames); pad the last one (got {counts[0]})")
            hw = [tuple(int(s) for s in view.shape[1:3]) for view in x]
            if self._view_hw is None:
                self._view_hw, self._view_bbox = hw, self._whole_frames(hw)
            elif hw != self._view_hw:
                raise ValueError(f"view sizes {hw} differ from the first chunk's {self._view_hw}")
            return "views", (*x, self._view_bbox)
        if x.dim() == 5 and x.shape[1] != v:
            raise ValueError(f"expected (T, {v}, 3, h, w) frames; got {tuple(x.shape)}")
        if x.shape[0] != (t if x.dim() == 5 else t * v):
            raise ValueError(f"chunks are fixed-size, ({t * v}, ...) or ({t}, {v}, ...); pad the last one (got {tuple(x.shape)})")
        if bbox is None:
            bbox = self._image_bbox
        elif self.regression:
            raise ValueError("a regression model predicts in model pixels (RegressionTracker.predict_step has no bbox remap)")
        elif tuple(bbox.shape) != (t, 4 * v):
            raise ValueError(f"bbox must be ({t}, {4 * v}); got {tuple(bbox.shape)}")
        return "tensor", (x, bbox)

    def _ingest(self, form: str, xs) -> tuple[torch.Tensor, torch.Tensor]:
        """A chunk's tensors -> (the (T V, ...) batch for ``features_of``, the (T, 4 V) boxes)."""
        if form == "crop":  # crop to the rows at the cursor BEFORE the table writer advances it
            x, bbox = ops.frames_crop_normalize(xs[0], self.bboxes, self.image_hw, cursor=self.cursor,
                                                channels_last=self.crop_channels_last, dtype=self.crop_dtype)
        elif form == "views":
            x = ops.frames_normalize_views(xs[:-1], self.image_hw, channels_last=self.crop_channels_last, dtype=self.crop_dtype)
            bbox = xs[-1]
        else:
            x, bbox = xs
        return (x.reshape(-1, *x.shape[2:]) if x.dim() == 5 else x), bbox

    @torch.no_grad()
    def _chunk(self, form: str, xs) -> None:
        """One chunk, enqueued on the current stream with no host sync: ingest, features, the body per sub-chunk."""
        x, bbox = self._ingest(form, xs)
        feats = self.features_of(x) if self.features_of is not None else x
        emit = self._emit_context if self.context else self._emit_regression if self.regression else self._emit_frames
        for i in range(0, self.chunk, self.sub_chunk):
            emit(feats, bbox, i, min(self.sub_chunk, self.chunk - i))

    def _emit_frames(self, feats: torch.Tensor, bbox: torch.Tensor, i: int, n: int) -> None:
        """Frames [i, i + n) of the chunk: head -> decode -> model->frame remap (bboxes.py:222-288) -> table rows."""
        v = self.num_views
        kp, cf = self.head.run_subpixelmaxima(self.head(feats[i * v : (i + n) * v]))
        # (n V, 2K) -> (n, 2 V K): the views of a frame side by side, as the trackers fold them
        kp = ops.remap_keypoints(kp.reshape(n, 2 * self.k * v), None, bbox[i : i + n], *self.image_hw, num_views=v)
        ops.pack_predictions(kp, cf.reshape(n, self.k * v), self.table, cursor=self.cursor)

    def _emit_regression(self, feats: torch.Tensor, bbox: torch.Tensor, i: int, n: int) -> None:
        """Frames [i, i + n) of a regression chunk: pooled linear head -> table rows, likelihood 0.0."""
        ops.pack_predictions(self.head(feats[i : i + n]), self._zero_conf[:n], self.table, cursor=self.cursor)

    def _emit_context(self, feats: torch.Tensor, bbox: torch.Tensor, i: int, n: int) -> None:
        """Frames [i, i + n) of a context chunk: the single-frame head and the W_f / W_b maps into the halo buffers, then
        the predictions of frames cursor - 2 + i .. cursor - 3 + i + n.  The first sub-chunk stores the chunk's boxes,
        the last one makes the chunk's final frames the next chunk's halo."""
        head, mf, t = self.head, self.head.head_mf, self.chunk
        if i == 0:
            self._box[2:].copy_(bbox)
        f = feats[i : i + n]
        kp, cf = head.run_subpixelmaxima(head.head_sf(f))  # single-frame head, once per frame
        self._kp_sf[2 + i : 2 + i + n].copy_(kp)
        self._cf_sf[2 + i : 2 + i + n].copy_(cf)
        wf, wb = mf._maps(f)  # W_f / W_b, once per frame
        if self._wf is None:
            self._wf = torch.zeros((t + 4, *wf.shape[1:]), dtype=torch.float32, device=self.device)
            self._wb = torch.zeros_like(self._wf)
        self._wf[4 + i : 4 + i + n].copy_(wf)
        self._wb[4 + i : 4 + i + n].copy_(wb)
        hf = (mf.H_f[0].weight, mf.H_f[0].bias, mf.H_f[1].weight, mf.H_f[1].bias)
        hb = (mf.H_b[0].weight, mf.H_b[0].bias, mf.H_b[1].weight, mf.H_b[1].bias)
        kp_mf, cf_mf = head.run_subpixelmaxima(ops.plane_softmax(ops.crnn_combine(self._wf, self._wb, self._idx[i : i + n], hf, hb)))
        ops.pack_context_predictions(self._kp_sf[i : i + n], self._cf_sf[i : i + n], kp_mf, cf_mf, self._box[i : i + n],
                                     *self.image_hw, self.table, t, cursor=self.cursor)
        if i + n == t:
            for buf, halo in self._halo():
                tail = buf[t : t + halo]
                buf[:halo].copy_(tail.clone() if t < halo else tail)

    def _capture(self, form: str, xs) -> None:
        self._static = [x.clone() for x in xs]
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):  # warm-up (per-shape tables, allocator pools); rewind the cursor afterwards
                self._chunk(form, self._static)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self._reset()
        self._graph = torch.cuda.CUDAGraph(keep_graph=True)  # kept so that its kernel nodes can be counted
        with torch.cuda.graph(self._graph):
            self._chunk(form, self._static)
        self.launches_per_chunk = _graph_kernel_count(self._graph)
        self._graph.instantiate()
        self.cursor.fill_(self.feed_range[0])  # the capture itself does not execute, but keep the invariant explicit

    def feed(self, x: torch.Tensor | Sequence[torch.Tensor], bbox: torch.Tensor | None = None) -> None:
        """Process the next chunk: a tensor with an optional ``bbox``, V uint8 views, or in crop mode uint8 full frames
        (the forms of the class docstring)."""
        form, xs = self._inputs(x, bbox)
        if not self.use_graph:
            self._chunk(form, xs)
            return
        got = f"{form} " + ", ".join(f"{tuple(t.shape)} {t.dtype}" for t in xs)
        if self._graph is None:
            self._capture(form, xs)
            self._captured = got
        if got != self._captured:  # a replay would cast or mis-read it
            raise ValueError(f"the chunk's graph was captured for {self._captured}; this chunk is {got}")
        for dst, src in zip(self._static, xs):
            dst.copy_(src, non_blocking=True)
        self._graph.replay()

    def run(self, chunks: Iterable[torch.Tensor | tuple[torch.Tensor, torch.Tensor] | Sequence[torch.Tensor]]) -> torch.Tensor:
        """Feed every chunk of an iterable, return the (N, 3 V K) table (still on the device).  An item is a chunk, a
        (chunk, bbox) pair, or a chunk's uint8 views."""
        for item in chunks:
            if isinstance(item, tuple) and not all(isinstance(t, torch.Tensor) and t.dtype == torch.uint8 for t in item):
                self.feed(*item)
            else:
                self.feed(item)
        return self.table

    def gather(self) -> torch.Tensor:
        """The full (N, 3 V K) table on every rank, equal to the one-GPU table: one ``all_gather`` of each rank's block
        of ``ceil(N / world)`` rows (its own rows, padded), then ``fill_context_edges`` on the device.  Every rank of
        the default process group calls it, those without rows too; one shard needs no collective."""
        rank, world = self.shard
        if world > 1:
            import torch.distributed as dist

            if dist.get_world_size() != world or dist.get_rank() != rank:
                raise ValueError(f"shard {self.shard} does not match the process group (rank {dist.get_rank()} of "
                                 f"{dist.get_world_size()})")
            blocks = list(self._blocks.split(self._blocks.shape[0] // world))
            dist.all_gather(blocks, blocks[rank].clone())
        if self.context:
            fill_context_edges(self.table, self.chunk, world)
        return self.table

    def results(self) -> tuple[torch.Tensor, torch.Tensor]:
        """(keypoints (N, 2K'), confidences (N, K')) views of the table - the reference's ``(preds, confs)`` pair, with
        K' = V K in multi-view mode."""
        kk = self.k * self.num_views
        t = self.table.reshape(self.n_frames, kk, 3)
        return t[:, :, :2].reshape(self.n_frames, 2 * kk), t[:, :, 2]

    def view_tables(self) -> list[torch.Tensor]:
        """The V (N, 3K) column blocks of the table, one per view (views, not copies)."""
        w = 3 * self.k
        return [self.table[:, w * v : w * (v + 1)] for v in range(self.num_views)]


class FramePredictor:
    """One frame in, its keypoints out, with one CUDA-graph replay per call: the reference's ``Model.predict_frame``
    (``lightning_pose/api/model.py:298-509``) for loops that need each answer before the next camera frame.

    ``head``: a ``HeatmapHead``, ``HeatmapMHCRNNHead`` or ``LinearRegressionHead`` on the device, in eval mode;
    ``features_of`` maps the ingested
    (F, 3, h, w) images (channels-last memory with ``channels_last``) to backbone features, e.g. the tracker's
    ``backbone``.  ``image_hw`` is the model's input size (``image_resize_dims``); ``dtype`` / ``channels_last`` the
    ingest's output, what ``features_of`` takes; ``mean`` / ``std`` the normalisation.

    ``predict_frame(frame_rgb, bbox=None)`` keeps the reference's contract: ``frame_rgb`` is uint8 (H, W, 3), or
    (5, H, W, 3) for a context model (the T = 5 frames its labeled batches use; other T raise), as a host numpy array or
    a CUDA tensor already on the device; ``bbox`` an optional (x, y, w, h) crop, cut as ``frame[y:y+h, x:x+w]`` (the far
    edges clip to the frame).  Returns ``{"keypoints": (K, 2), "confidence": (K,)}`` float32 numpy arrays in
    original-frame pixels, and raises ``ValueError`` where the reference does.

    Body: ``ops.frames_crop_resize_cv2`` (the reference's cv2 resize and numpy normalisation, bit for bit, with the box
    read on the device) -> ``features_of`` -> head -> soft-argmax decode -> model -> frame remap -> one (K, 3) row.  A
    context head runs ``HeatmapTrackerMHCRNN``'s labeled form on (1, 5, 3, h, w) and keeps, per keypoint, the
    multi-frame prediction where its confidence is greater than the single-frame one (a NaN keeps single-frame).  A
    regression head maps its model-pixel keypoints to the frame and reports a confidence of 1.0, as the reference's
    ``predict_frame`` does for regression models (``api/model.py:495-500``; its ``predict_step`` gives zeros instead).

    With ``use_graph`` the first call of each input form (host or device frame, frame shape) is captured; a new form
    captures anew and replaces the old graph.  The images' dtype, and with it the features', is fixed per predictor.
    The box changes on every call without a capture.  A host frame and the box are written to pinned staging buffers whose
    host -> device copies are nodes of the graph, and the result comes back by a device -> host copy inside it; a
    device frame is copied into the graph's input buffer on the device.  A call is: write the staging buffers, replay,
    synchronise once, return copies.  ``launches_per_call`` counts the captured kernels.  ``use_graph=False`` runs the
    same body eagerly.
    """

    CONTEXT_FRAMES = 5

    def __init__(self, head, num_keypoints: int, image_hw: tuple[int, int], features_of: Callable[[torch.Tensor], torch.Tensor],
                 device=None, use_graph: bool = True, dtype: torch.dtype = torch.float32, channels_last: bool = False,
                 mean: Sequence[float] = ops.IMAGENET_MEAN, std: Sequence[float] = ops.IMAGENET_STD) -> None:
        from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead
        from lightning_pose_b200.models.heads.regression import LinearRegressionHead

        if features_of is None:
            raise ValueError("features_of (images -> backbone features) is required")
        ops._out_format(dtype)
        self.head, self.k = head, int(num_keypoints)
        self.context = isinstance(head, HeatmapMHCRNNHead)
        self.regression = isinstance(head, LinearRegressionHead)
        self.image_hw = (int(image_hw[0]), int(image_hw[1]))
        self.features_of = features_of
        self.device = torch.device(device) if device is not None else next(head.parameters()).device
        self.use_graph = bool(use_graph)
        self.dtype, self.channels_last = dtype, bool(channels_last)
        self.mean, self.std = tuple(float(v) for v in mean), tuple(float(v) for v in std)
        # the (K, 3) result: a context call writes the one frame of a five-row window to all five rows
        # (lpb_pack_context_predictions with frame0 = 4, step 1), a frame call writes row 0
        self._table = torch.zeros((self.CONTEXT_FRAMES if self.context else 1, 3 * self.k), dtype=torch.float32, device=self.device)
        self._ones = torch.ones((1, self.k), dtype=torch.float32, device=self.device)  # a regression head's confidence
        self._box = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._pin_box = torch.zeros(4, dtype=torch.int32).pin_memory()
        self._pin_out = torch.zeros((self.k, 3), dtype=torch.float32).pin_memory()
        self._key = self._graph = self._frames = self._pin_frames = None
        self.launches_per_call = None

    def _check(self, frame_rgb, bbox) -> tuple[np.ndarray | torch.Tensor, tuple[int, int, int, int]]:
        """The reference's input checks (api/model.py:353-407) -> (frames (F, H, W, 3), box [x, y, w, h])."""
        if isinstance(frame_rgb, torch.Tensor):
            if frame_rgb.dtype != torch.uint8:
                raise ValueError(f"frame_rgb must be uint8, got {frame_rgb.dtype}")
            if not frame_rgb.is_cuda:
                frame_rgb = frame_rgb.numpy()
            elif frame_rgb.device != self.device:
                raise ValueError(f"frame_rgb is on {frame_rgb.device}; the model is on {self.device}")
        else:
            frame_rgb = np.asarray(frame_rgb)
            if frame_rgb.dtype != np.uint8:
                raise ValueError(f"frame_rgb must be uint8, got {frame_rgb.dtype}")
        shape = tuple(frame_rgb.shape)
        if len(shape) not in (3, 4) or shape[-1] != 3:
            raise ValueError(f"frame_rgb must be (H, W, 3) or (T, H, W, 3), got shape {shape}")
        if int(np.prod(shape)) == 0:
            raise ValueError("frame_rgb is empty")
        if self.context and len(shape) == 3:
            raise ValueError(f"a context model requires frame_rgb of shape ({self.CONTEXT_FRAMES}, H, W, 3); got a single frame "
                             f"{shape}. Use BatchedPredictor for video input.")
        if self.context and shape[0] != self.CONTEXT_FRAMES:
            raise ValueError(f"a context model takes {self.CONTEXT_FRAMES} frames, the context length of its labeled batches; "
                             f"got {shape[0]}")
        if not self.context and len(shape) == 4:
            raise ValueError(f"a single-frame model takes one (H, W, 3) frame; got shape {shape}")
        h, w = shape[-3], shape[-2]
        if bbox is None:
            return frame_rgb, (0, 0, w, h)
        bx, by, bw, bh = (operator.index(v) for v in bbox)
        if bx < 0 or by < 0:
            raise ValueError(f"bbox origin must be non-negative, got x={bx}, y={by}")
        if bw <= 0 or bh <= 0:
            raise ValueError(f"bbox width and height must be positive, got w={bw}, h={bh}")
        if bx >= w or by >= h:
            raise ValueError(f"bbox (x={bx}, y={by}, w={bw}, h={bh}) produces an empty crop on frame of shape {shape}")
        return frame_rgb, (bx, by, min(bw, w), min(bh, h))  # sizes past the frame clip as the numpy slice does

    def _body(self) -> torch.Tensor:
        """Ingest -> features -> head -> decode -> remap into ``_table``; returns the (K, 3) result row (device)."""
        head, (mh, mw) = self.head, self.image_hw
        x, bbox = ops.frames_crop_resize_cv2(self._frames, self.image_hw, self._box, self.mean, self.std,
                                             channels_last=self.channels_last, dtype=self.dtype)
        if self.channels_last:
            x = x.permute(0, 3, 1, 2)
        feats = self.features_of(x)
        if self.regression:
            ops.pack_predictions(ops.remap_keypoints(head(feats), None, bbox, mh, mw), self._ones, self._table, row0=0)
            return self._table.view(self.k, 3)
        if not self.context:
            _, kp, cf = head.forward_with_keypoints(feats)
            kp = ops.remap_keypoints(kp, None, bbox, mh, mw)
            ops.pack_predictions(kp, cf, self._table, row0=0)
            return self._table.view(self.k, 3)
        t = self.CONTEXT_FRAMES
        # HeatmapTrackerMHCRNN.forward on a (1, 5, 3, h, w) labeled batch
        reps = torch.permute(feats.reshape(1, t, *feats.shape[1:]), (0, 2, 3, 4, 1))
        sf, mf = head(reps, (1, t, 3, mh, mw), False)
        kp_sf, cf_sf = head.run_subpixelmaxima(sf)
        kp_mf, cf_mf = head.run_subpixelmaxima(mf)
        # a table of five rows, fed frame0 = 4: output frame 2, which is every row's source
        ops.pack_context_predictions(kp_sf, cf_sf, kp_mf, cf_mf, bbox, mh, mw, self._table, 1, frame0=t - 1)
        return self._table[2].view(self.k, 3)

    @torch.no_grad()
    def _call(self, from_host: bool) -> None:
        """One call's device work on the current stream: staging -> device, the body, result -> pinned buffer."""
        if from_host:
            self._frames.copy_(self._pin_frames, non_blocking=True)
        self._box.copy_(self._pin_box, non_blocking=True)
        self._pin_out.copy_(self._body(), non_blocking=True)

    def _prepare(self, key) -> None:
        """Buffers (and with ``use_graph`` the graph) of an input form: (host?, frame shape)."""
        self._key, self._graph = key, None
        from_host, shape = key
        self._frames = torch.zeros(shape, dtype=torch.uint8, device=self.device)
        self._pin_frames = torch.zeros(shape, dtype=torch.uint8).pin_memory() if from_host else None
        if not self.use_graph:
            return
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):  # warm-up: per-shape tables, allocator pools
                self._call(from_host)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph(keep_graph=True)  # kept so that its kernel nodes can be counted
        with torch.cuda.graph(graph):
            self._call(from_host)
        self.launches_per_call = _graph_kernel_count(graph)
        graph.instantiate()
        self._graph = graph

    def predict_frame(self, frame_rgb, bbox: tuple[int, int, int, int] | None = None) -> dict[str, np.ndarray]:
        """The reference's ``predict_frame``: ``{"keypoints": (K, 2), "confidence": (K,)}`` float32, frame pixels."""
        frames, box = self._check(frame_rgb, bbox)
        from_host = not isinstance(frames, torch.Tensor)
        shape = tuple(frames.shape) if frames.ndim == 4 else (1, *frames.shape)
        if self._key != (from_host, shape):
            self._prepare((from_host, shape))
        self._pin_box.numpy()[:] = box
        if from_host:
            np.copyto(self._pin_frames.numpy(), frames.reshape(shape))
        else:
            self._frames.copy_(frames.reshape(shape))
        if self._graph is not None:
            self._graph.replay()
        else:
            self._call(from_host)
        torch.cuda.current_stream(self.device).synchronize()
        out = self._pin_out.numpy()
        return {"keypoints": out[:, :2].copy(), "confidence": out[:, 2].copy()}
