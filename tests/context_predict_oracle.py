"""Golden generator for video prediction with context (MHCRNN) models.  TEST INFRASTRUCTURE ONLY.

``python tests/context_predict_oracle.py`` writes ``tests/golden/context_predict.npz``.  It runs the reference's own
``HeatmapMHCRNNHead``, ``run_subpixelmaxima`` and ``model_to_frame_batch`` (loaded unmodified through
``oracle/ref_loader.py``).  The pieces whose files need Lightning, DALI or omegaconf to import are executed from their
source text with the type annotations stripped:
  * ``get_context_from_sequence``             lightning_pose/models/base.py:159-196
  * ``HeatmapTrackerMHCRNN.predict_step``     lightning_pose/models/heatmap_tracker_mhcrnn.py:180-229
  * ``PrepareDALI.num_iters``                 lightning_pose/data/video/dali.py:494-534
  * ``PredictionHandler.unpack_preds`` and ``fix_context_preds_confs``  lightning_pose/utils/predictions.py:97-177
The reader is modelled as the reference configures it for context prediction (dali.py:600-619): windows of S frames
with step S - 4, ``num_iters`` of them, frames past the end replaced by one fixed padding feature (the backbone's output
for the reader's zero-filled frame); the backbone is the identity on seeded features.  Box rows follow the crop-mode
cursor (dali.py:332-372): rows [jT, jT + S), padded with the last row.

Cases (``{tag}_{case}``): ``features`` (N, C, h, w), ``pad`` (C, h, w), ``bbox`` (N, 4) x y h w, ``meta`` [N, S,
upsampling_factor, image height, image width]; the reference's final ``kp`` (N, 2K) and ``conf`` (N, K); ``rows`` (N,)
the frame whose prediction each row holds (the same functions run on frame-index labels).  Head parameters are stored
once per tag (``{tag}_param_<state-dict key>``).  Needs the reference tree; the GPU tests only read the committed npz.
"""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "context_predict.npz")
K, C, FH, FW = 5, 32, 4, 4

# (name, N, S): R = T * (ceil((N - S) / T) + 1) with T = S - 4
CASES = [
    ("r_ge_n", 30, 12),   # R = 32 >= N
    ("r_lt_n", 27, 12),   # R = 24 < N: rows 24-26 hold pred(2)
    ("r_n_minus_1", 25, 12),  # R = 24 = N - 1: row 23 reads the padding frame 25
    ("n5", 5, 12),        # the shortest video
    ("n_lt_s", 9, 16),    # one window, shorter than S
    ("issue_example", 100, 16),  # R = 96: frames 96-99 hold pred(2)
]
# (tag, backbone_arch, upsampling_factor, image (h, w)); features are (C, 4, 4)
HEADS = [("uf1", "vits_dino", 1, (64, 64)), ("uf2", "resnet50", 2, (128, 128))]


def _ref():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_loader as R

    return R


def reference_tree_available() -> bool:
    R = _ref()
    need = ("models/base.py", "models/heatmap_tracker_mhcrnn.py", "data/video/dali.py", "utils/predictions.py")
    return all(os.path.isfile(os.path.join(R.REF_ROOT, "lightning_pose", p)) for p in need)


def _function(path: str, name: str, cls: str | None = None):
    """Source text of a reference function (or method of ``cls``), decorators and annotations stripped."""
    tree = ast.parse(open(path).read())
    body = tree.body
    if cls is not None:
        body = next(n for n in body if isinstance(n, ast.ClassDef) and n.name == cls).body
    fn = next(n for n in body if isinstance(n, ast.FunctionDef) and n.name == name)
    fn.decorator_list, fn.returns = [], None
    for a in fn.args.args + fn.args.kwonlyargs:
        a.annotation = None
    return ast.unparse(fn)


def source_functions() -> dict:
    """The reference functions executed from their source text."""
    R = _ref()
    lp = os.path.join(R.REF_ROOT, "lightning_pose")
    ns = {"torch": torch, "np": np}
    for path, name, cls in (("models/base.py", "get_context_from_sequence", None),
                            ("models/heatmap_tracker_mhcrnn.py", "predict_step", "HeatmapTrackerMHCRNN"),
                            ("data/video/dali.py", "num_iters", "PrepareDALI"),
                            ("utils/predictions.py", "unpack_preds", "PredictionHandler"),
                            ("utils/predictions.py", "fix_context_preds_confs", "PredictionHandler")):
        exec(_function(os.path.join(lp, path), name, cls), ns)
    return ns


def num_iters(fns: dict, n: int, s: int) -> int:
    pipe = {"sequence_length": s, "step": s - 4, "batch_size": 1}
    self = types.SimpleNamespace(_pipe_dict={"predict": {"context": pipe}}, train_stage="predict", model_type="context",
                                 frame_count=n)
    return fns["num_iters"](self)


def unpack(fns: dict, preds: list, n: int):
    """PredictionHandler.unpack_preds for a video of n frames and a heatmap_mhcrnn model."""
    self = types.SimpleNamespace(video_file="video.mp4", frame_count=n, do_context=True,
                                 cfg=types.SimpleNamespace(model=types.SimpleNamespace(model_type="heatmap_mhcrnn")))
    self.fix_context_preds_confs = types.MethodType(fns["fix_context_preds_confs"], self)
    return fns["unpack_preds"](self, preds)


def reference_row_map(fns: dict, n: int, s: int) -> np.ndarray:
    """Frame whose prediction each row of the reference's final table holds: the reader's windows carry their valid
    frames' indices through unpack_preds (an empty list of windows raises there, as in the reference)."""
    t = s - 4
    preds = []
    for j in range(num_iters(fns, n, s)):
        f = torch.arange(j * t + 2, j * t + s - 2, dtype=torch.float64)[:, None]
        preds.append((f, f.clone()))
    rows, _ = unpack(fns, preds, n)
    return rows[:, 0].numpy().astype(np.int64)


def row_rule(n: int, s: int) -> np.ndarray:
    """The row rule lpb_pack_context_predictions implements."""
    t = s - 4
    r = n if t == 1 else t * (-(-(n - s) // t) + 1)  # step 1: one window per frame (num_iters' first branch)
    f = np.arange(n)
    if r >= n:
        return np.clip(f, 2, n - 3)
    return np.where((f >= 2) & (f <= r - 1), f, 2)


def _head(mh, arch: str, uf: int, seed: int):
    torch.manual_seed(seed)
    head = mh.HeatmapMHCRNNHead(arch, C, K, upsampling_factor=uf)
    for prm in head.head_sf.parameters():  # peaked, non-degenerate maps
        torch.nn.init.normal_(prm, std=0.3)
    return head.eval()


def reference_table(fns: dict, db, head, feats, pad, bbox, s: int, image_hw):
    """The reference's final (kp (N, 2K), conf (N, K)) for a video of per-frame features ``feats``."""
    n, t = feats.shape[0], s - 4

    def forward(images):  # identity backbone on the window's features, then get_representations + the head
        reps = fns["get_context_from_sequence"](img_seq=window["feats"], context_length=5)
        if reps.shape[0] < 5:
            raise RuntimeError("Not enough valid frames to make a context representation.")
        reps = torch.permute(reps[2:-2], (0, 2, 3, 4, 1))
        return head(reps, images.shape, False)

    tracker = types.SimpleNamespace(forward=forward, head=head)
    fns["model_to_frame_batch"] = db.model_to_frame_batch
    preds = []
    for j in range(num_iters(fns, n, s)):
        idx = list(range(j * t, j * t + s))
        window = {"feats": torch.stack([feats[i] if i < n else pad for i in idx])}
        rows = bbox[[min(i, n - 1) for i in idx]]
        batch = {"frames": torch.zeros(1).expand(s, 3, *image_hw), "bbox": rows.clone()}
        kp, cf = fns["predict_step"](tracker, batch, j)
        preds.append((kp, cf))
    return unpack(fns, preds, n)


def main(path: str = GOLDEN_PATH) -> None:
    assert reference_tree_available(), "needs the full reference tree"
    R = _ref()
    mh = R.load("lightning_pose.models.heads.heatmap_mhcrnn")
    db = R.load("lightning_pose.data.bboxes")
    fns = source_functions()
    out = {}
    with torch.no_grad():
        for hi, (tag, arch, uf, image_hw) in enumerate(HEADS):
            head = _head(mh, arch, uf, 60 + hi)
            for name, tns in head.state_dict().items():
                if ".layers." not in name:  # ModuleList aliases of the same tensors
                    out[f"{tag}_param_{name}"] = tns.numpy().copy()
            for ci, (case, n, s) in enumerate(CASES):
                if uf == 2 and case == "issue_example":
                    continue
                gen = torch.Generator().manual_seed(1000 * hi + ci)
                feats = torch.randn(n, C, FH, FW, generator=gen)
                pad = torch.randn(C, FH, FW, generator=gen)
                xy = torch.cumsum(torch.randn(n, 2, generator=gen) * 3, 0) + 40
                hw = torch.randint(60, 120, (n, 2), generator=gen).float()
                bbox = torch.cat([xy.round(), hw], 1)
                kp, cf = reference_table(fns, db, head, feats, pad, bbox, s, image_hw)
                rows = reference_row_map(fns, n, s)
                assert np.array_equal(rows, row_rule(n, s)), (case, n, s)
                p = f"{tag}_{case}"
                out[f"{p}_features"], out[f"{p}_pad"], out[f"{p}_bbox"] = feats.numpy(), pad.numpy(), bbox.numpy()
                out[f"{p}_meta"] = np.asarray([n, s, uf, *image_hw], np.int64)
                out[f"{p}_kp"], out[f"{p}_conf"], out[f"{p}_rows"] = kp.numpy(), cf.numpy(), rows
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main(*sys.argv[1:])
