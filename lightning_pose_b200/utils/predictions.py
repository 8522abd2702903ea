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
Multi-GPU: replicas over contiguous frame ranges (``frame_range_for_rank``), no communication (the reference itself
never predicts on more than one device).
"""
from __future__ import annotations

from typing import Callable, Iterable, Sequence

import numpy as np
import torch

from lightning_pose_b200 import ops

__all__ = ["BatchedPredictor", "PredictionHandler", "make_dlc_pandas_index", "frame_range_for_rank"]


def frame_range_for_rank(n_frames: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, near-equal frame ranges: [start, stop) of ``rank`` (cfg 5: 100,000 frames -> 12,500 per GPU)."""
    per = -(-n_frames // max(world, 1))
    return min(rank * per, n_frames), min((rank + 1) * per, n_frames)


def make_dlc_pandas_index(model_type: str, keypoint_names: Sequence[str]):
    """``[scorer, bodyparts, coords]`` MultiIndex with coords (x, y, likelihood) (reference :551-570)."""
    import pandas as pd

    return pd.MultiIndex.from_product([[f"{model_type}_tracker"], list(keypoint_names), ["x", "y", "likelihood"]],
                                      names=["scorer", "bodyparts", "coords"])


class PredictionHandler:
    """Video-side mirror of the reference's ``PredictionHandler`` (:41-329): same column schema, same context fix-up.

    ``frame_count`` is given directly (the reference counts the video's frames with OpenCV; video I/O is out of scope).
    """

    def __init__(self, keypoint_names: Sequence[str], frame_count: int, model_type: str = "heatmap") -> None:
        if keypoint_names is None:
            raise ValueError("must include `keypoint_names`")
        self.keypoint_names = list(keypoint_names)
        self.frame_count = int(frame_count)
        self.model_type = model_type

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

    def __call__(self, preds: Iterable[tuple[torch.Tensor, torch.Tensor]]):
        """Reference call form: a list of per-batch (keypoints, confidences) tuples -> DataFrame."""
        preds = list(preds)
        kp = torch.vstack([p[0] for p in preds])[: self.frame_count]
        cf = torch.vstack([p[1] for p in preds])[: self.frame_count]
        if self.do_context:
            kp = self.fix_context_preds_confs(kp)
            cf = self.fix_context_preds_confs(cf, zero_pad_confidence=False)
        import pandas as pd

        arr = self.make_pred_arr_undo_resize(kp.cpu().numpy(), cf.cpu().numpy())
        return pd.DataFrame(arr, columns=make_dlc_pandas_index(self.model_type, self.keypoint_names))


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
    """CUDA-graph chunk loop writing straight into a preallocated (N, 3K) device table.

    ``head``: a ``HeatmapHead`` (already on the device, eval).  ``features_of``: callable mapping a chunk's input (frames
    or precomputed features) to backbone features ``(T, C, h, w)`` - identity when the caller streams features; a backbone
    module otherwise (library convolutions; its kernels are captured into the same graph).  Chunks are fixed-size ``T``
    (``dali.base.predict.sequence_length`` = 96 in the reference config); the last chunk is padded by the caller and its
    surplus rows are dropped by the table writer.

    Crop mode (crop-zoom pose models, reference ``predict_video(..., bbox_file=...)``, ``utils/predictions.py:455-470``
    and ``data/video/dali.py:332-380``): ``bboxes`` is the video's (N, 4) [x, y, h, w] device table (``compute_bboxes``
    / ``smooth_bboxes``) and ``frame_hw`` the full frame size.  ``feed`` then takes uint8 (T, H, W, 3) decoded frames;
    inside the chunk (and its graph) one launch crops each frame to its box row at the table's device cursor (rows past
    the end repeat the last), resizes the crop to ``image_hw`` and normalises it into ``crop_dtype`` (channels-last if
    ``crop_channels_last``) for ``features_of``, and the clamped boxes it writes map the keypoints back to the frame.
    ``launches_per_chunk``: kernel launches in one captured chunk (set at capture).

    Context mode (``head`` a ``HeatmapMHCRNNHead``, reference ``HeatmapTrackerMHCRNN.predict_step`` over a reader of
    windows of ``S = chunk + 4`` frames with step ``chunk``, ``dali.context.predict.sequence_length``): ``chunk`` is the
    number of NEW frames per call, the caller feeds ``ceil(N / chunk)`` non-overlapping chunks (the last one padded) and
    chunk j yields the predictions of frames ``j * chunk - 2 .. j * chunk + chunk - 3``.  The two / four frames before a
    chunk stay on the device between calls (their single-frame decode, their boxes and their W_f / W_b maps), so every
    frame passes through ``features_of``, ``head_sf`` and the maps once.  ``lpb_pack_context_predictions`` writes each
    frame's selected, remapped prediction to every row the reference's ``fix_context_preds_confs`` gives it, so after
    the last chunk ``table`` is the reference's final table for ``sequence_length = chunk + 4`` with no host fix-up (use
    ``PredictionHandler.dataframe(table, frame_aligned=True)``).  With R = chunk * (ceil((N - S) / chunk) + 1):
    R >= N: row f is frame clamp(f, 2, N - 3); R < N: row f is frame f for 2 <= f <= R - 1 and frame 2 otherwise (the
    reference pads the tail with its first row).  Only when R = N - 1 does a row (N - 2) depend on frame N, the first
    padding frame of the last chunk; the reference reads the zero-filled frame its reader pads with there, so the
    caller's padding matters in that case only.  N < 5 raises (the reference has no window to predict from).
    """

    def __init__(self, head, num_keypoints: int, n_frames: int, chunk: int, image_hw: tuple[int, int],
                 features_of: Callable[[torch.Tensor], torch.Tensor] | None = None, device=None, use_graph: bool = True,
                 sub_chunk: int | None = None, bboxes: torch.Tensor | None = None, frame_hw: tuple[int, int] | None = None,
                 crop_dtype: torch.dtype = torch.float32, crop_channels_last: bool = False, num_views: int = 1) -> None:
        from lightning_pose_b200.models.heads.heatmap_mhcrnn import HeatmapMHCRNNHead

        self.head, self.k, self.n_frames, self.chunk = head, int(num_keypoints), int(n_frames), int(chunk)
        self.context = isinstance(head, HeatmapMHCRNNHead)
        if self.context and int(num_views) > 1:
            raise ValueError("context prediction is not supported for multiview models")
        if self.context and self.n_frames < 5:
            raise ValueError(f"a context model needs at least 5 frames to predict from; the video has {self.n_frames}")
        if self.chunk < 1:
            raise ValueError(f"chunk must be >= 1; got {self.chunk}")
        # frames per head / decode call inside a chunk: small enough that the heatmaps written by the head are still in
        # the 126 MB L2 when the decode reads them (None: the whole chunk at once)
        self.sub_chunk = int(sub_chunk) if sub_chunk else self.chunk
        self.image_hw = (int(image_hw[0]), int(image_hw[1]))
        self.features_of = features_of
        self.device = torch.device(device) if device is not None else next(head.parameters()).device
        self.table = torch.zeros((self.n_frames, 3 * self.k), dtype=torch.float32, device=self.device)
        self.cursor = torch.zeros((1,), dtype=torch.int64, device=self.device)
        self.use_graph = use_graph
        self._graph = None
        self._static_in = None
        self._static_bbox = None
        self.launches_per_chunk = None
        self.bboxes = None
        if bboxes is not None:
            if int(num_views) > 1:
                raise ValueError("bbox cropping is not supported for multiview models")
            if frame_hw is None or features_of is None:
                raise ValueError("crop mode needs frame_hw (the full frame size) and features_of (frames -> features)")
            self.bboxes = ops._bbox_table(bboxes, "bboxes")
            if self.bboxes.shape[0] != self.n_frames:
                raise ValueError(f"bboxes has {self.bboxes.shape[0]} rows but the video has {self.n_frames} frames")
            self.frame_hw = (int(frame_hw[0]), int(frame_hw[1]))
            self.crop_dtype, self.crop_channels_last = crop_dtype, bool(crop_channels_last)
        if self.context:
            # halo + chunk buffers: index b of the maps holds frame cursor - 4 + b, of the others frame cursor - 2 + b; the
            # maps' buffers are sized by the first chunk's maps
            t, k, dev = self.chunk, self.k, self.device
            self._wf = self._wb = None
            self._kp_sf = torch.zeros((t + 2, 2 * k), dtype=torch.float32, device=dev)
            self._cf_sf = torch.zeros((t + 2, k), dtype=torch.float32, device=dev)
            self._box = torch.zeros((t + 2, 4), dtype=torch.float32, device=dev)
            self._idx = (torch.arange(t, device=dev)[:, None] + torch.arange(5, device=dev)[None, :]).to(torch.int32)

    def _reset(self) -> None:
        self.cursor.zero_()
        self.table.zero_()
        if self.context:
            for buf in (self._wf, self._wb, self._kp_sf, self._cf_sf, self._box):
                if buf is not None:
                    buf.zero_()

    def _context_chunk(self, x: torch.Tensor, bbox: torch.Tensor) -> None:
        """One context chunk, eager: T new frames -> the predictions of frames cursor - 2 .. cursor + T - 3."""
        head, mf = self.head, self.head.head_mf
        hf = (mf.H_f[0].weight, mf.H_f[0].bias, mf.H_f[1].weight, mf.H_f[1].bias)
        hb = (mf.H_b[0].weight, mf.H_b[0].bias, mf.H_b[1].weight, mf.H_b[1].bias)
        t = self.chunk
        with torch.no_grad():
            feats = self.features_of(x) if self.features_of is not None else x
            self._box[2:].copy_(bbox)
            for i in range(0, t, self.sub_chunk):
                n = min(self.sub_chunk, t - i)
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
                kp_mf, cf_mf = head.run_subpixelmaxima(ops.plane_softmax(ops.crnn_combine(self._wf, self._wb, self._idx[i : i + n], hf, hb)))
                ops.pack_context_predictions(self._kp_sf[i : i + n], self._cf_sf[i : i + n], kp_mf, cf_mf, self._box[i : i + n],
                                             self.image_hw[0], self.image_hw[1], self.table, t, cursor=self.cursor)
            for buf, halo in ((self._wf, 4), (self._wb, 4), (self._kp_sf, 2), (self._cf_sf, 2), (self._box, 2)):
                tail = buf[t : t + halo]
                buf[:halo].copy_(tail.clone() if t < halo else tail)  # the last frames become the next chunk's halo

    # one chunk, eager: everything below is enqueued on the current stream; no host sync
    def _chunk(self, x: torch.Tensor, bbox: torch.Tensor | None) -> None:
        if self.bboxes is not None:  # crop to the rows at the cursor BEFORE the table writer advances it
            x, bbox = ops.frames_crop_normalize(x, self.bboxes, self.image_hw, cursor=self.cursor, channels_last=self.crop_channels_last,
                                                dtype=self.crop_dtype)
        if self.context:
            self._context_chunk(x, bbox)
            return
        feats = self.features_of(x) if self.features_of is not None else x
        with torch.no_grad():
            for i in range(0, self.chunk, self.sub_chunk):
                heatmaps = self.head(feats[i : i + self.sub_chunk])
                kp, cf = self.head.run_subpixelmaxima(heatmaps)
                kp = ops.remap_keypoints(kp, None, bbox[i : i + self.sub_chunk], self.image_hw[0], self.image_hw[1])  # model -> frame (bboxes.py:222-288)
                ops.pack_predictions(kp, cf, self.table, cursor=self.cursor)

    def _capture(self, x: torch.Tensor, bbox: torch.Tensor) -> None:
        self._static_in = torch.empty_like(x)
        self._static_in.copy_(x)
        if bbox is not None:
            self._static_bbox = torch.empty_like(bbox)
            self._static_bbox.copy_(bbox)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):  # warm-up (per-shape tables, allocator pools); rewind the cursor afterwards
                self._chunk(self._static_in, self._static_bbox)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self._reset()
        self._graph = torch.cuda.CUDAGraph(keep_graph=True)  # kept so that its kernel nodes can be counted
        with torch.cuda.graph(self._graph):
            self._chunk(self._static_in, self._static_bbox)
        self.launches_per_chunk = _graph_kernel_count(self._graph)
        self._graph.instantiate()
        self.cursor.zero_()  # the capture itself does not execute, but keep the invariant explicit

    def feed(self, x: torch.Tensor, bbox: torch.Tensor | None = None) -> None:
        """Process the next chunk (``x``: (T, ...) frames or features on the device; in crop mode uint8 (T, H, W, 3)
        frames, and ``bbox`` must be None: the boxes come from the predictor's table)."""
        if x.shape[0] != self.chunk:
            raise ValueError(f"chunks are fixed-size ({self.chunk} frames); pad the last one (got {x.shape[0]})")
        if self.bboxes is not None:
            if bbox is not None:
                raise ValueError("crop mode takes its boxes from the `bboxes` table given at construction")
            if x.dtype != torch.uint8 or tuple(x.shape[1:]) != (*self.frame_hw, 3):
                raise ValueError(f"crop mode expects uint8 ({self.chunk}, {self.frame_hw[0]}, {self.frame_hw[1]}, 3) frames; got {tuple(x.shape)} {x.dtype}")
        elif bbox is None:
            bbox = torch.tensor([[0.0, 0.0, float(self.image_hw[0]), float(self.image_hw[1])]], device=self.device).repeat(self.chunk, 1)
        if not self.use_graph:
            self._chunk(x, bbox)
            return
        if self._graph is None:
            self._capture(x, bbox)
        self._static_in.copy_(x, non_blocking=True)
        if bbox is not None:
            self._static_bbox.copy_(bbox, non_blocking=True)
        self._graph.replay()

    def run(self, chunks: Iterable[torch.Tensor | tuple[torch.Tensor, torch.Tensor]]) -> torch.Tensor:
        """Feed every chunk of an iterable, return the (N, 3K) table (still on the device)."""
        for item in chunks:
            if isinstance(item, tuple):
                self.feed(item[0], item[1])
            else:
                self.feed(item)
        return self.table

    def results(self) -> tuple[torch.Tensor, torch.Tensor]:
        """(keypoints (N, 2K), confidences (N, K)) views of the table - the reference's ``(preds, confs)`` pair."""
        t = self.table.reshape(self.n_frames, self.k, 3)
        return t[:, :, :2].reshape(self.n_frames, 2 * self.k), t[:, :, 2]
