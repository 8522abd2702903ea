"""lightning_pose_b200 - H100-native (sm_90a) hot path of lightning-pose.

Mirrors the reference's module layout for the one path it accelerates, so that
``lightning_pose.models.heads.heatmap`` -> ``lightning_pose_b200.models.heads.heatmap`` etc.:

    models/heads/heatmap.py   HeatmapHead, run_subpixelmaxima, upsample, make_upsampling_layers
    data/heatmaps.py          generate_heatmaps, evaluate_heatmaps_at_location
    data/utils.py, bboxes.py  undo_affine_transform_batch, model_to_frame_batch
    losses/losses.py          the 12 loss classes;  losses/factory.py  get_loss_classes, LossFactory
    utils/pca.py              KeypointPCA (device-side reproject / reprojection error)

All numerics run in ``liblpb200.so`` (hand-written CUDA behind the C-ABI of ``include/lpb200.h``).
Importing this package without the built library raises: there is no CPU fallback.
"""
from . import _lib  # noqa: F401  (fails loudly when liblpb200.so is missing)
from . import ops  # noqa: F401

__version__ = "0.1.0"
