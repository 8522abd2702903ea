"""CPU: the surface of ``SemiSupervisedHeatmapTrackerMultiviewTransformer`` (reference
``models/heatmap_tracker_multiview.py:370-484``), its transform-shape rule, and the package's independence of the
test oracle."""
import ast
import inspect
import os

import pytest
import torch

from lightning_pose_b200.models.heatmap_tracker_multiview import (HeatmapTrackerMultiviewTransformer,
                                                                  SemiSupervisedHeatmapTrackerMultiviewTransformer,
                                                                  view_transforms)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the reference constructor's keywords (:376-394); the backbone, head, optimizer and image-size ones configure parts
# that are the caller's modules or out of scope here and are accepted through **kwargs
REFERENCE_KEYWORDS = ["num_keypoints", "num_views", "loss_factory", "loss_factory_unsupervised", "backbone", "pretrained",
                      "head", "downsample_factor", "torch_seed", "optimizer", "optimizer_params", "lr_scheduler",
                      "lr_scheduler_params", "image_size"]


def _model(**kw):
    return SemiSupervisedHeatmapTrackerMultiviewTransformer(5, 3, torch.nn.Identity(), torch.nn.Identity(), 32, **kw)


def test_class_and_constructor_keywords():
    cls = SemiSupervisedHeatmapTrackerMultiviewTransformer
    assert issubclass(cls, HeatmapTrackerMultiviewTransformer)
    params = inspect.signature(cls.__init__).parameters
    parent = inspect.signature(HeatmapTrackerMultiviewTransformer.__init__).parameters
    assert [n for n in parent if n not in params] == []  # the parent's arguments, plus the unsupervised factory
    assert [n for n in params if n not in parent] == ["loss_factory_unsupervised"]
    kept = [n for n in REFERENCE_KEYWORDS if n in params]
    assert kept == ["num_keypoints", "num_views", "loss_factory", "loss_factory_unsupervised", "downsample_factor", "torch_seed"]
    assert params["kwargs"].kind is inspect.Parameter.VAR_KEYWORD
    for name in ("get_loss_inputs_unlabeled", "evaluate_unlabeled", "training_step"):
        assert list(inspect.signature(getattr(cls, name)).parameters)[1] == "batch_dict"
    assert list(inspect.signature(cls.evaluate_unlabeled).parameters)[2:] == ["stage", "anneal_weight"]

    m = _model(loss_factory_unsupervised=None, backbone="vits_dino", pretrained=True, head="heatmap_cnn", image_size=256,
               optimizer="Adam", lr_scheduler="multisteplr")
    assert m.loss_factory_unsup is None
    w = m.total_unsupervised_importance
    assert w.shape == () and w.dtype == torch.float32 and float(w) == 1.0
    assert "total_unsupervised_importance" in dict(m.named_buffers())  # moves with .to(device)
    assert "total_unsupervised_importance" not in m.state_dict()  # as the reference's plain attribute
    w.fill_(0.25)
    assert float(m.total_unsupervised_importance) == 0.25


@pytest.mark.parametrize("shape", [(3, 1, 2, 3), (1, 3, 2, 3), (3, 2, 3)])
def test_view_transforms_accepts_the_reference_shapes(shape):
    tf = torch.arange(18, dtype=torch.float32).reshape(shape)
    out = view_transforms(tf, 3)
    assert out.shape == (3, 2, 3) and torch.equal(out.reshape(-1), tf.reshape(-1))


def test_view_transforms_unaugmented_and_malformed():
    assert view_transforms(torch.full((3, 1), -1.0), 3) is None  # frames_to_unlabeled_batch without augmentation
    assert view_transforms(torch.tensor([-1.0]), 3) is None
    assert view_transforms(torch.zeros(1, 1, 2, 3), 1).shape == (1, 2, 3)
    for bad in ((2, 2, 3), (3, 2, 2, 3), (2, 1, 2, 3), (2, 3), (6, 3)):
        with pytest.raises(ValueError, match="transforms"):
            view_transforms(torch.zeros(bad), 3)


def test_unlabeled_frames_must_hold_every_view():
    m = _model()
    for frames in (torch.zeros(4, 3, 32, 32), torch.zeros(4, 2, 3, 32, 32)):
        with pytest.raises(ValueError, match="expected frames"):
            m.get_loss_inputs_unlabeled({"frames": frames, "transforms": torch.full((3, 1), -1.0), "bbox": torch.zeros(4, 12)})


def test_package_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "lightning_pose_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            path = os.path.join(dirpath, f)
            with open(path) as fh:
                tree = ast.parse(fh.read(), path)
            for node in ast.walk(tree):
                names = [a.name for a in node.names] if isinstance(node, ast.Import) else []
                if isinstance(node, ast.ImportFrom) and node.level == 0:
                    names = [node.module or ""]
                if any(n == "oracle" or n.startswith("oracle.") for n in names):
                    offenders.append(os.path.relpath(path, ROOT))
    assert offenders == []
