"""Backbone metadata needed by the head (``lightning_pose/models/backbones/factory.py:98-124``).

Only the stride table is on the hot path: ``HeatmapHead`` derives its number of deconv layers
from it (``n_layers = log2(stride) - downsample_factor - 1``).  Convnets and SAM2 Hiera reach
stride 32, standard 16x16-patch ViTs stride 16.
"""

import torch

_STRIDE32 = (
    "resnet18 resnet34 resnet50 resnet101 resnet152 resnet50_animal_apose resnet50_animal_ap10k "
    "resnet50_human_jhmdb resnet50_human_res_rle resnet50_human_top_res resnet50_human_hand "
    "efficientnet_b0 efficientnet_b1 efficientnet_b2 vitb_sam2 vits_sam2 vitt_sam2"
).split()
_STRIDE16 = "vits_dino vits_dinov2 vits_dinov3 vitb_dino vitb_dinov2 vitb_dinov3 vitb_imagenet vitb_sam".split()

BACKBONE_STRIDES: dict[str, int] = {**{n: 32 for n in _STRIDE32}, **{n: 16 for n in _STRIDE16}}


def tokens_to_feature_map(tokens: torch.Tensor, grid: tuple[int, int]) -> torch.Tensor:
    """A transformer encoder's patch tokens ``(N, h * w, D)`` as the feature map ``(N, D, h, w)`` the heads take, without
    moving them: a channels-last view (``torch.channels_last`` strides) of contiguous tokens.

    The reference permutes the tokens into an NCHW copy; the heads here read channels-last features in place and
    return the gradient in the same layout, so neither pass copies the features.  ``.contiguous()`` on the result gives
    the NCHW tensor."""
    h, w = grid
    n, p, d = tokens.shape
    if p != h * w:
        raise ValueError(f"{p} tokens do not fill a {h} x {w} grid")
    return tokens.contiguous().reshape(n, h, w, d).permute(0, 3, 1, 2)
