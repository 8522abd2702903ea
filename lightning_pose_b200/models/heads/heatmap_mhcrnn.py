"""Multi-head convolutional-RNN head on H100: drop-in for ``lightning_pose.models.heads.heatmap_mhcrnn``.

Same public surface as the reference module (``lightning_pose/models/heads/heatmap_mhcrnn.py``):
``HeatmapMHCRNNHead`` (:18-137) and ``UpsamplingCRNN`` (:139-316) with identical constructor arguments, attributes and
state-dict keys (``head_sf.upsampling_layers.<i>.*``, ``head_mf.{W_pre,W_f,H_f.0,H_f.1,W_b,H_b.0,H_b.1}.*`` and the
``head_mf.layers.<i>`` aliases), so reference checkpoints load unchanged.

What differs is what runs.  The modules are parameter containers; the arithmetic is
  * ``W_pre`` / ``W_f`` / ``W_b``: the head's own transposed-convolution kernels (tensor-core for bf16 features), applied to
    every frame ONCE - a frame that sits in five overlapping windows of a video sequence is never tiled five times
    (the reference does, ``models/base.py:380-390``);
  * the bidirectional recurrence: ``H_f`` / ``H_b`` (grouped Conv2d k2 s2 -> grouped ConvTranspose2d k2 s2, no
    nonlinearity) are 4x4 affine maps per keypoint on 2x2 blocks, so the five steps per direction are evaluated per
    block by one kernel from the per-frame maps and a window index table (``csrc/crnn.cu``), with a native backward;
  * the final spatial softmax and the soft-argmax decode are the package's kernels.
``forward`` keeps the reference call form (already-gathered ``(batch, C, h, w, 5)`` features);
``forward_sequence`` is the fused video form (``(T, C, h, w)`` features in, the ``T - 4`` valid frames out).
"""
from __future__ import annotations

from typing import Literal

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.models.heads.heatmap import HeatmapHead, _HeadFunction, _needs_grad, run_subpixelmaxima

__all__: list[str] = []


def get_context_from_sequence(img_seq: torch.Tensor, context_length: int) -> torch.Tensor:
    """(seq_len, ...) -> (seq_len, context_length, ...) windows centred on each frame, edges replicated
    (reference ``models/base.py:159-196``; result is float32 there, and here for float32 input)."""
    return ops.context_gather(img_seq, int(context_length))


def _deconv(in_channels: int, out_channels: int) -> nn.ConvTranspose2d:
    return nn.ConvTranspose2d(in_channels, out_channels, kernel_size=(3, 3), stride=(2, 2), padding=(1, 1), output_padding=(1, 1))


def _hidden(num_keypoints: int, nfilters_channel: int, hkernel: int, hstride: int, hpad: int) -> nn.Sequential:
    return nn.Sequential(
        nn.Conv2d(num_keypoints, num_keypoints * nfilters_channel, kernel_size=(hkernel, hkernel), stride=(hstride, hstride),
                  padding=(hpad, hpad), groups=num_keypoints),
        nn.ConvTranspose2d(num_keypoints * nfilters_channel, num_keypoints, kernel_size=(hkernel, hkernel), stride=(hstride, hstride),
                           padding=(hpad, hpad), output_padding=(hpad, hpad), groups=num_keypoints),
    )


class UpsamplingCRNN(nn.Module):
    """Bidirectional convolutional RNN over the heatmaps of the context frames (reference :139-316)."""

    def __init__(
        self,
        num_filters_for_upsampling: int,
        num_keypoints: int,
        upsampling_factor: Literal[1, 2] = 2,
        hkernel: int = 2,
        hstride: int = 2,
        hpad: int = 0,
        nfilters_channel: int = 16,
    ) -> None:
        super().__init__()
        if (hkernel, hstride, hpad) != (2, 2, 0):
            raise NotImplementedError("the block-affine recurrence kernel covers the reference's hidden layers (kernel 2, stride 2, pad 0)")
        self.upsampling_factor = upsampling_factor
        self.pixel_shuffle = nn.PixelShuffle(2)
        if self.upsampling_factor == 2:
            self.W_pre = _deconv(num_filters_for_upsampling // 4, num_keypoints)
            in_channels_rnn = num_keypoints
        else:
            in_channels_rnn = num_filters_for_upsampling // 4
        self.W_f = _deconv(in_channels_rnn, num_keypoints)
        self.H_f = _hidden(num_keypoints, nfilters_channel, hkernel, hstride, hpad)
        self.W_b = _deconv(in_channels_rnn, num_keypoints)
        self.H_b = _hidden(num_keypoints, nfilters_channel, hkernel, hstride, hpad)
        self._initialize_layers()
        if self.upsampling_factor == 2:
            self.layers = nn.ModuleList([self.W_pre, self.W_f, self.H_f, self.W_b, self.H_b])
        else:
            self.layers = nn.ModuleList([self.W_f, self.H_f, self.W_b, self.H_b])

    def _initialize_layers(self) -> None:
        """xavier-uniform (gain 1) weights, zero biases (reference :250-266)."""
        mods = ([self.W_pre] if self.upsampling_factor == 2 else []) + [self.W_f, *self.H_f, self.W_b, *self.H_b]
        for m in mods:
            nn.init.xavier_uniform_(m.weight, gain=1.0)
            nn.init.zeros_(m.bias)

    def _maps(self, feats: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """W_f / W_b (after W_pre when upsampling_factor = 2) of every frame: (N, K, H, W) logits, once per frame."""
        outs = []
        for last in (self.W_f, self.W_b):
            layers = ([self.W_pre] if self.upsampling_factor == 2 else []) + [last]
            params = [m.weight for m in layers] + [m.bias for m in layers]
            outs.append(_HeadFunction.apply(feats, False, None, _needs_grad(feats, params), *params))
        return outs[0], outs[1]

    def forward_windows(self, feats: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
        """Fused form: features of N distinct frames (N, C, h, w) + window table idx (M, 5) -> heatmaps (M, K, H, W)."""
        wf, wb = self._maps(feats)
        hf = (self.H_f[0].weight, self.H_f[0].bias, self.H_f[1].weight, self.H_f[1].bias)
        hb = (self.H_b[0].weight, self.H_b[0].bias, self.H_b[1].weight, self.H_b[1].bias)
        return ops.plane_softmax(ops.crnn_combine(wf, wb, idx, hf, hb))

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        """Reference call form: (frames, batch, C, h, w) -> (batch, K, H, W)."""
        frames, batch = features.shape[:2]
        if frames != 5:
            raise NotImplementedError("the recurrence kernel is written for 5 context frames")
        flat = features.reshape(frames * batch, *features.shape[2:])
        idx = torch.arange(frames, device=features.device)[None, :] * batch + torch.arange(batch, device=features.device)[:, None]
        return self.forward_windows(flat, idx.to(torch.int32))


class HeatmapMHCRNNHead(nn.Module):
    """Single-frame head + multi-frame (context) head (reference :18-137)."""

    def __init__(
        self,
        backbone_arch: str,
        in_channels: int,
        out_channels: int,
        deconv_out_channels: int | None = None,
        downsample_factor: int = 2,
        upsampling_factor: Literal[1, 2] = 2,
    ) -> None:
        super().__init__()
        self.backbone_arch = backbone_arch
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.deconv_out_channels = deconv_out_channels
        self.downsample_factor = downsample_factor
        self.upsampling_factor = upsampling_factor
        self.temperature = torch.tensor(1000.0)
        self.head_sf = HeatmapHead(
            backbone_arch=backbone_arch, in_channels=in_channels, out_channels=out_channels,
            deconv_out_channels=deconv_out_channels, downsample_factor=downsample_factor,
        )
        self.head_mf = UpsamplingCRNN(
            num_filters_for_upsampling=self.head_sf.in_channels, num_keypoints=self.head_sf.out_channels, upsampling_factor=upsampling_factor,
        )

    def forward(self, features: torch.Tensor, batch_shape: torch.Size | tuple, is_multiview: bool) -> tuple[torch.Tensor, torch.Tensor]:
        """(batch, C, h, w, frames) features -> (heatmaps_sf, heatmaps_mf), view dimension folded back (reference :79-121)."""
        num_frames = int(batch_shape[0])
        if len(batch_shape) == 5 and is_multiview:
            shape_r = features.shape
            num_frames -= 4  # the first / last two frames of an unlabeled batch are lost to the context
            features = features.reshape(num_frames * int(batch_shape[1]), -1, shape_r[-3], shape_r[-2], shape_r[-1])
        features = torch.permute(features, (4, 0, 1, 2, 3)).contiguous()
        heatmaps_sf = self.head_sf(features[2])  # index 2 == middle frame
        heatmaps_mf = self.head_mf(features)
        if len(batch_shape) == 6 or len(batch_shape) == 5:
            heatmaps_sf = heatmaps_sf.reshape(num_frames, -1, heatmaps_sf.shape[-2], heatmaps_sf.shape[-1])
            heatmaps_mf = heatmaps_mf.reshape(num_frames, -1, heatmaps_mf.shape[-2], heatmaps_mf.shape[-1])
        return heatmaps_sf, heatmaps_mf

    def forward_sequence(self, features_seq: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """Video form: per-frame features (T, C, h, w) -> heatmaps of the T - 4 valid frames (those with two frames on
        either side, reference ``models/base.py:372-390``), without ever materialising the (T, 5, ...) window tensor."""
        t = features_seq.shape[0]
        if t < 5:
            raise RuntimeError("Not enough valid frames to make a context representation.")
        idx = torch.arange(t - 4, device=features_seq.device)[:, None] + torch.arange(5, device=features_seq.device)[None, :]
        heatmaps_sf = self.head_sf(features_seq[2 : t - 2])
        heatmaps_mf = self.head_mf.forward_windows(features_seq, idx.to(torch.int32))
        return heatmaps_sf, heatmaps_mf

    def run_subpixelmaxima(self, heatmaps: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        return run_subpixelmaxima(heatmaps, self.downsample_factor, self.temperature)
