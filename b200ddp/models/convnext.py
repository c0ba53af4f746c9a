"""ConvNeXt (Liu et al., 2022) for image classification: ConvNeXt-T, -S and -B at 224 x 224, with torchvision's module and
parameter names, shapes, registration order and initialisation (``torchvision.models.convnext_tiny`` and the others), so
``load_state_dict`` takes a torchvision state dict strictly and DDP buckets match.  A 4x4 / stride-4 stem with a
LayerNorm2d, four stages of blocks x + layer_scale * (Linear(4C, C)(GELU(Linear(C, 4C)(LayerNorm(dwconv7x7(x)))))), a
LayerNorm2d and 2x2 / stride-2 convolution between stages, global average pooling, a LayerNorm and the head.  LayerNorm
eps 1e-6, erf GELU.  There is no stochastic depth: every block always runs, torchvision's ``stochastic_depth_prob=0.0``,
as the project trains without dropout.

bf16 CUDA input runs on the native kernels with the whole network on NHWC rows [B H W, C] and no NCHW permutes: the stem
and downsampling convolutions are a (ky, kx, c) patch gather (``ops.patchify_nhwc``) times the permuted weight on the
wgmma ``linear``, each block is ``ops.depthwise_conv2d``, ``layer_norm``, the GELU and plain ``linear`` and a
``torch.addcmul`` residual, and the pool is a mean over each image's rows.  That path needs H and W multiples of 32.  At a
batch that is not a multiple of 8, the last stage's B x 49 rows are no multiple of 8 and its linears run on ``linear``'s
cuBLAS fallback.  Anything else (CPU, fp32 on CUDA) runs torchvision's arithmetic in NCHW."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, depthwise_conv2d, layer_norm, linear, patchify_nhwc


@dataclass(frozen=True)
class ConvNeXtConfig:
    widths: tuple[int, ...]
    depths: tuple[int, ...]
    num_classes: int = 1000
    layer_scale: float = 1e-6
    eps: float = 1e-6


CONVNEXT_TINY = ConvNeXtConfig(widths=(96, 192, 384, 768), depths=(3, 3, 9, 3))
CONVNEXT_SMALL = ConvNeXtConfig(widths=(96, 192, 384, 768), depths=(3, 3, 27, 3))
CONVNEXT_BASE = ConvNeXtConfig(widths=(128, 256, 512, 1024), depths=(3, 3, 27, 3))

# the native path downsamples by 4 x 2 x 2 x 2
INPUT_MULTIPLE = 32


class LayerNorm2d(LayerNorm):
    """torchvision's ``LayerNorm2d``: a LayerNorm over the channels of an NCHW tensor."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), self.weight, self.bias, self.eps).permute(0, 3, 1, 2)


class _Keyed(nn.Module):
    """A container whose children keep torchvision's ``nn.Sequential`` indices, with the parameter-free ones left out."""

    def __init__(self, children: dict[int, nn.Module]):
        super().__init__()
        for i, m in children.items():
            self.add_module(str(i), m)

    def __getitem__(self, i: int) -> nn.Module:
        return self._modules[str(i)]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        for m in self._modules.values():
            x = m(x)
        return x


class CNBlock(nn.Module):
    """torchvision's ``CNBlock`` keys: ``block.0`` the depthwise 7x7 convolution, ``block.2`` the LayerNorm, ``block.3``
    Linear(C, 4C) with the erf GELU (torchvision's ``block.4``) in its epilogue, ``block.5`` Linear(4C, C), and
    ``layer_scale`` [C, 1, 1]."""

    def __init__(self, dim: int, layer_scale: float, eps: float):
        super().__init__()
        self.block = _Keyed({0: nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim),
                             2: LayerNorm(dim, eps=eps),
                             3: Linear(dim, 4 * dim, activation="gelu"),
                             5: Linear(4 * dim, dim)})
        self.layer_scale = nn.Parameter(torch.ones(dim, 1, 1) * layer_scale)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x NCHW, torchvision's arithmetic."""
        y = self.block[0](x).permute(0, 2, 3, 1)
        y = self.block[5](self.block[3](self.block[2](y))).permute(0, 3, 1, 2)
        result = self.layer_scale * y
        result += x
        return result

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        """x [B H W, C] NHWC rows, the native kernels."""
        C = x.shape[1]
        conv = self.block[0]
        y = depthwise_conv2d(x.view(B, H, W, C), conv.weight, conv.bias).view(-1, C)
        y = self.block[5](self.block[3](self.block[2](y)))
        return torch.addcmul(x, y, self.layer_scale.view(C))


def _conv_rows(x: torch.Tensor, conv: nn.Conv2d) -> torch.Tensor:
    """A kernel = stride convolution of x [B, H, W, C] (any strides) as its (ky, kx, c) patch rows times the weight."""
    D, p = conv.weight.shape[0], conv.weight.shape[-1]
    return linear(patchify_nhwc(x, p), conv.weight.permute(0, 2, 3, 1).reshape(D, -1), conv.bias)


class ConvNeXt(nn.Module):
    """forward(images [B, 3, H, W]) -> logits [B, num_classes]; ``config`` is the preset."""

    def __init__(self, config: ConvNeXtConfig):
        super().__init__()
        c = self.config = config
        if len(c.widths) != len(c.depths):
            raise ValueError(f"ConvNeXtConfig: {len(c.widths)} widths for {len(c.depths)} stages")
        layers = [_Keyed({0: nn.Conv2d(3, c.widths[0], kernel_size=4, stride=4), 1: LayerNorm2d(c.widths[0], eps=c.eps)})]
        for s, (width, depth) in enumerate(zip(c.widths, c.depths)):
            layers.append(nn.Sequential(*[CNBlock(width, c.layer_scale, c.eps) for _ in range(depth)]))
            if s + 1 < len(c.widths):
                layers.append(_Keyed({0: LayerNorm2d(width, eps=c.eps), 1: nn.Conv2d(width, c.widths[s + 1], kernel_size=2, stride=2)}))
        self.features = nn.Sequential(*layers)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.classifier = _Keyed({0: LayerNorm2d(c.widths[-1], eps=c.eps), 2: Linear(c.widths[-1], c.num_classes)})
        # torchvision's scheme: every convolution and linear weight normal with std 0.02 cut at +-2 (absolute), zero biases
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f"ConvNeXt: expected images [B, 3, H, W], got {tuple(images.shape)}")
        stem = self.features[0][0]
        if images.is_cuda and images.dtype == torch.bfloat16 and stem.weight.dtype == torch.bfloat16:
            return self._forward_rows(images)
        x = self.features(images)
        return self.classifier[2](self.classifier[0](self.avgpool(x)).flatten(1))

    def _forward_rows(self, images: torch.Tensor) -> torch.Tensor:
        B, _, H, W = images.shape
        if H % INPUT_MULTIPLE or W % INPUT_MULTIPLE:
            raise ValueError(f"ConvNeXt on the native path needs H and W multiples of {INPUT_MULTIPLE}, got {H}x{W}")
        stem, norm = self.features[0][0], self.features[0][1]
        x = layer_norm(_conv_rows(images.permute(0, 2, 3, 1), stem), norm.weight, norm.bias, norm.eps)
        H, W = H // 4, W // 4
        for s in range(len(self.config.widths)):
            if s:
                down = self.features[2 * s]
                C = x.shape[1]
                x = _conv_rows(layer_norm(x, down[0].weight, down[0].bias, down[0].eps).view(B, H, W, C), down[1])
                H, W = H // 2, W // 2
            for block in self.features[2 * s + 1]:
                x = block.forward_rows(x, B, H, W)
        norm = self.classifier[0]
        pooled = layer_norm(x.view(B, H * W, -1).mean(1), norm.weight, norm.bias, norm.eps)
        return self.classifier[2](pooled)


def convnext_tiny(num_classes: int = 1000) -> ConvNeXt:
    """ConvNeXt-T: widths 96 / 192 / 384 / 768, depths 3 / 3 / 9 / 3 (28,589,128 parameters)."""
    return ConvNeXt(replace(CONVNEXT_TINY, num_classes=num_classes))


def convnext_small(num_classes: int = 1000) -> ConvNeXt:
    """ConvNeXt-S: ConvNeXt-T's widths, depths 3 / 3 / 27 / 3 (50,223,688 parameters)."""
    return ConvNeXt(replace(CONVNEXT_SMALL, num_classes=num_classes))


def convnext_base(num_classes: int = 1000) -> ConvNeXt:
    """ConvNeXt-B: widths 128 / 256 / 512 / 1024, depths 3 / 3 / 27 / 3 (88,591,464 parameters)."""
    return ConvNeXt(replace(CONVNEXT_BASE, num_classes=num_classes))
