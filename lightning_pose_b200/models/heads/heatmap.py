"""Heatmap head on H100: drop-in for ``lightning_pose.models.heads.heatmap``.

Same public surface as the reference module (``lightning_pose/models/heads/heatmap.py``):
``make_upsampling_layers`` (:20-71), ``initialize_upsampling_layers`` (:74-83), ``upsample``
(:86-100), ``run_subpixelmaxima`` (:103-144) and ``HeatmapHead`` (:147-227) with identical
constructor arguments, attributes and state-dict keys (``upsampling_layers.<i>.weight`` in
ConvTranspose2d ``(C_in, C_out, 3, 3)`` layout), so reference checkpoints load unchanged.

What differs is what runs: the ``nn.Sequential`` is only a parameter container.  ``forward``
hands its weights to the fused CUDA head (PixelShuffle folded into the first transposed
convolution's staging, gather-form deconvs, in-place plane softmax) and ``run_subpixelmaxima``
calls the fused soft-argmax decode, which never materialises the 4x-upsampled field.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from lightning_pose_b200 import ops
from lightning_pose_b200.models.backbones import BACKBONE_STRIDES

__all__: list[str] = []


def make_upsampling_layers(in_channels: int, out_channels: int, int_channels: int, n_layers: int) -> nn.Sequential:
    """``PixelShuffle(2)`` followed by ``n_layers`` stride-2 3x3 transposed convolutions.

    Channel plan (reference :44-71): the shuffle divides channels by 4; intermediate layers use
    ``int_channels``; the last layer emits ``out_channels``.
    """
    widths = [in_channels // 4] + [int_channels] * (n_layers - 1) + [out_channels]
    layers: list[nn.Module] = [nn.PixelShuffle(2)]
    for c_in, c_out in zip(widths[:-1], widths[1:]):
        layers.append(
            nn.ConvTranspose2d(c_in, c_out, kernel_size=(3, 3), stride=(2, 2), padding=(1, 1), output_padding=(1, 1))
        )
    return nn.Sequential(*layers)


def initialize_upsampling_layers(layers: nn.Sequential) -> None:
    """xavier-uniform (gain 0.01) weights and zero bias for the deconvs (reference :74-83)."""
    for layer in list(layers)[1:]:
        if isinstance(layer, nn.ConvTranspose2d):
            nn.init.xavier_uniform_(layer.weight, gain=0.01)
            nn.init.zeros_(layer.bias)
        elif isinstance(layer, nn.BatchNorm2d):
            nn.init.ones_(layer.weight)
            nn.init.zeros_(layer.bias)


def upsample(inputs: torch.Tensor) -> torch.Tensor:
    """One 2x stage: bicubic (align_corners=False) + zero-padded 5x5 binomial blur (reference :86-100)."""
    return ops.upsample2x(inputs)


def run_subpixelmaxima(
    heatmaps: torch.Tensor, downsample_factor: int, temperature: torch.Tensor | float
) -> tuple[torch.Tensor, torch.Tensor]:
    """Soft-argmax decode: (batch, 2*num_keypoints) keypoints and (batch, num_keypoints) confidences."""
    return ops.decode_softargmax(heatmaps, int(downsample_factor), float(temperature))


def _needs_grad(features: torch.Tensor, params) -> bool:
    """Whether a backward can follow (decided outside the autograd node: grad mode is off inside ``forward``).
    Inference skips everything the backward would need (saved operand copies, inter-layer activations)."""
    return torch.is_grad_enabled() and (features.requires_grad or any(p.requires_grad for p in params))


class _HeadFunction(torch.autograd.Function):
    """Fused head, optionally with the soft-argmax decode riding along (``decode = (ds, temperature)``).

    Forward: tensor-core head for bf16 features (one- or two-deconv heads inside the tensor-core tiling), the fp32
    CUDA-core kernels otherwise (+ decode kernel).  Backward: native in both cases.  On the tensor-core path the gradient
    w.r.t. the heatmaps is never materialised for the decode branch: the sparse decode windows, a dense heatmap-loss
    gradient if there is one, and the softmax backward are all folded into the kernel that writes the
    deconv-gradient operand.  Outputs: heatmaps [, keypoints (B, 2K), confidences (B, K)].
    """

    @staticmethod
    def forward(ctx, features, final_softmax, decode, train, *params):
        n = len(params) // 2
        weights, biases = list(params[:n]), list(params[n:])
        saved = acts = None
        if features.dtype == torch.bfloat16 and features.is_cuda and ops.head_bf16_supported(
                tuple(features.shape), [w.shape[1] for w in weights], train=train):
            res = ops._head_forward_bf16(features.contiguous(), weights, biases, final_softmax, train=train)
            out, saved = res if train else (res, None)
        elif train:
            out, acts = ops.head_forward_f32(features, weights, biases, final_softmax, keep_activations=True)
        else:
            out = ops.head_forward_f32(features, weights, biases, final_softmax)
        ctx.set_materialize_grads(False)
        ctx.final_softmax, ctx.n, ctx.saved, ctx.decode = final_softmax, n, saved, decode
        ctx.n_acts = len(acts) if acts is not None else 0
        extra = list(acts) if acts is not None else []
        if decode is None:
            ctx.save_for_backward(features, out, *params, *extra)
            return out
        ds, temperature = decode
        xy, conf, stats = ops.decode_forward(out, int(ds), float(temperature))
        ctx.save_for_backward(features, out, *params, *extra, stats)
        ctx.mark_non_differentiable(conf)
        return out, xy.reshape(-1, out.shape[1] * 2), conf

    @staticmethod
    def backward(ctx, g, g_xy=None, g_conf=None):
        tensors = list(ctx.saved_tensors)
        stats = tensors.pop() if ctx.decode is not None else None
        acts = [tensors.pop() for _ in range(ctx.n_acts)][::-1]
        features, out, *params = tensors
        n = ctx.n
        weights, biases = params[:n], params[n:]
        need_dfeat = ctx.needs_input_grad[0]
        if g is None and g_xy is None:
            return (None,) * (4 + 2 * n)
        if g is not None:
            g = g.contiguous().float()
        if ctx.saved is not None:
            windows = None
            if g_xy is not None:
                windows = ops.decode_backward_windows(out, stats, g_xy.contiguous().float(), int(ctx.decode[0]), float(ctx.decode[1]))
            dfeat, dw1, db1, dw2, db2 = ops.head_backward_bf16(
                g, ctx.saved, tuple(features.shape), weights[0], weights[1] if n == 2 else None, need_dfeat=need_dfeat,
                probs=out if ctx.final_softmax else None, windows=windows,
            )
            dws, dbs = ([dw1, dw2], [db1, db2]) if n == 2 else ([dw1], [db1])
            return (dfeat, None, None, None, *[d.to(w.dtype) for d, w in zip(dws, weights)], *[d.to(b.dtype) for d, b in zip(dbs, biases)])
        # fp32 path: dense decode gradient, softmax backward, then the deconvs' own backward kernels, last layer first
        if g_xy is not None:
            gd = ops._decode_bwd(out, stats, g_xy.contiguous().float(), int(ctx.decode[0]), float(ctx.decode[1]))
            g = gd if g is None else g + gd
        if ctx.final_softmax:  # d softmax: p * (g - sum(g * p)) per plane
            g = ops.plane_softmax_backward(out, g)
        dws, dbs = [None] * n, [None] * n
        for i in range(n - 1, -1, -1):
            g, dws[i], dbs[i] = ops.convt_backward_f32(acts[i], g, weights[i], shuffle=(i == 0), need_dx=(i > 0 or need_dfeat))
        gf = g.to(features.dtype) if need_dfeat else None
        return (gf, None, None, None, *[d.to(w.dtype) for d, w in zip(dws, weights)], *[d.to(b.dtype) for d, b in zip(dbs, biases)])


class HeatmapHead(nn.Module):
    """Deconvolution head: backbone features -> per-keypoint spatial-softmax heatmaps.

    Constructor / attributes follow the reference (:155-201): ``n_layers = log2(stride) -
    downsample_factor - 1`` deconvs after the PixelShuffle, soft-argmax temperature 1000.
    """

    def __init__(
        self,
        backbone_arch: str,
        in_channels: int,
        out_channels: int,
        deconv_out_channels: int | None = None,
        downsample_factor: int = 2,
        final_softmax: bool = True,
    ) -> None:
        super().__init__()
        self.backbone_arch = backbone_arch
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.deconv_out_channels = deconv_out_channels
        self.downsample_factor = downsample_factor
        self.final_softmax = final_softmax
        self.temperature = torch.tensor(1000.0)
        stride = BACKBONE_STRIDES.get(backbone_arch, 32)
        n_layers = int(math.log2(stride)) - downsample_factor - 1
        self.upsampling_layers = make_upsampling_layers(
            in_channels=in_channels,
            out_channels=out_channels,
            int_channels=deconv_out_channels or out_channels,
            n_layers=n_layers,
        )
        initialize_upsampling_layers(self.upsampling_layers)

    def _deconvs(self) -> list[nn.ConvTranspose2d]:
        return [m for m in self.upsampling_layers if isinstance(m, nn.ConvTranspose2d)]

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        deconvs = self._deconvs()
        params = [d.weight for d in deconvs] + [d.bias for d in deconvs]
        return _HeadFunction.apply(features, bool(self.final_softmax), None, _needs_grad(features, params), *params)

    def forward_with_keypoints(self, features: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``forward`` + ``run_subpixelmaxima`` as one autograd node: (heatmaps, keypoints, confidences).

        Same values as calling the two methods in sequence (reference flow, heatmap_tracker.py:163-179); the
        difference is the backward, which never materialises the dense gradient of the soft-argmax.
        """
        deconvs = self._deconvs()
        params = [d.weight for d in deconvs] + [d.bias for d in deconvs]
        decode = (int(self.downsample_factor), float(self.temperature))
        return _HeadFunction.apply(features, bool(self.final_softmax), decode, _needs_grad(features, params), *params)

    def run_subpixelmaxima(self, heatmaps: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        return run_subpixelmaxima(heatmaps, self.downsample_factor, self.temperature)
