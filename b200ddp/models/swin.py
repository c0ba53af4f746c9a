"""Swin Transformer (Liu et al., 2021) for image classification: Swin-T, -S and -B at 224 x 224, with torchvision's module
and parameter names, shapes, registration order and initialisation (``torchvision.models.swin_t`` and the others), so
``load_state_dict`` takes a torchvision state dict strictly and DDP buckets match.  A 4x4 / stride-4 stem with a
LayerNorm, four stages of blocks x + proj(W-MSA(qkv(norm1(x)))), x + mlp(norm2(x)) whose odd blocks shift the windows
by 3, patch merging between stages, a LayerNorm, global average pooling and the head.  Window 7, head dim 32, LayerNorm
eps 1e-5, erf GELU.  There is no stochastic depth or dropout (torchvision's ``stochastic_depth_prob=0.0``), as the
project trains without dropout.

bf16 CUDA input runs on the native kernels with the whole network on NHWC rows [B H W, C] in raster order and no roll,
window partition or permute: the stem is a (ky, kx, c) patch gather times the permuted weight on the wgmma ``linear``,
each block is ``layer_norm``, the qkv ``linear``, ``ops.window_attention`` (which reads each token's qkv row and writes
its output row in place of the roll and partition), the proj ``linear`` and the GELU MLP, and patch merging is a strided
gather in torchvision's (kx, ky, c) order, ``layer_norm`` and the bias-free ``linear``.  That path needs H and W
multiples of 224, so that every stage is a whole number of windows.  Anything else (CPU, fp32 on CUDA) runs torchvision's
arithmetic, padding included."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, layer_norm, linear, swin_relative_position_index, window_attention
from ..ops.functional import SWIN_MASK, SWIN_WINDOW
from .convnext import _conv_rows, _Keyed


@dataclass(frozen=True)
class SwinConfig:
    embed_dim: int
    depths: tuple[int, ...]
    heads: tuple[int, ...]
    num_classes: int = 1000
    window: int = SWIN_WINDOW
    patch: int = 4
    mlp_ratio: int = 4
    eps: float = 1e-5


SWIN_T = SwinConfig(embed_dim=96, depths=(2, 2, 6, 2), heads=(3, 6, 12, 24))
SWIN_S = SwinConfig(embed_dim=96, depths=(2, 2, 18, 2), heads=(3, 6, 12, 24))
SWIN_B = SwinConfig(embed_dim=128, depths=(2, 2, 18, 2), heads=(4, 8, 16, 32))

# the native path downsamples by 4 x 2 x 2 x 2 and needs every stage to be whole 7 x 7 windows
INPUT_MULTIPLE = 224


def _shifts(window: int, shift: int, height: int, width: int) -> tuple[int, int]:
    """torchvision's rule: no shift along a dimension the window covers whole."""
    return (0 if window >= height else shift, 0 if window >= width else shift)


class ShiftedWindowAttention(nn.Module):
    """torchvision's ``ShiftedWindowAttention`` keys: ``qkv`` Linear(C, 3C), ``proj`` Linear(C, C), the
    ``relative_position_bias_table`` [169, heads] and the persistent int64 ``relative_position_index`` [2401]."""

    def __init__(self, dim: int, heads: int, window: int, shift: int):
        super().__init__()
        self.heads, self.window, self.shift = heads, window, shift
        self.qkv = Linear(dim, 3 * dim)
        self.proj = Linear(dim, dim)
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window - 1) ** 2, heads))
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)
        self.register_buffer("relative_position_index", swin_relative_position_index())

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, H, W, C], torchvision's ``shifted_window_attention`` arithmetic (padding to whole windows included)."""
        B, H, W, C = x.shape
        w = self.window
        x = F.pad(x, (0, 0, 0, (w - W % w) % w, 0, (w - H % w) % w))
        _, pH, pW, _ = x.shape
        sy, sx = _shifts(w, self.shift, pH, pW)
        if sy + sx > 0:
            x = torch.roll(x, shifts=(-sy, -sx), dims=(1, 2))
        n = (pH // w) * (pW // w)
        x = x.view(B, pH // w, w, pW // w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B * n, w * w, C)
        qkv = F.linear(x, self.qkv.weight, self.qkv.bias)
        qkv = qkv.reshape(x.size(0), x.size(1), 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        q = q * (C // self.heads) ** -0.5
        attn = q.matmul(k.transpose(-2, -1))
        bias = self.relative_position_bias_table[self.relative_position_index].view(w * w, w * w, -1)
        attn = attn + bias.permute(2, 0, 1).contiguous().unsqueeze(0)
        if sy + sx > 0:
            mask = x.new_zeros((pH, pW))
            count = 0
            for hs in ((0, -w), (-w, -sy), (-sy, None)):
                for ws in ((0, -w), (-w, -sx), (-sx, None)):
                    mask[hs[0]:hs[1], ws[0]:ws[1]] = count
                    count += 1
            mask = mask.view(pH // w, w, pW // w, w).permute(0, 2, 1, 3).reshape(n, w * w)
            mask = mask.unsqueeze(1) - mask.unsqueeze(2)
            mask = mask.masked_fill(mask != 0, SWIN_MASK).masked_fill(mask == 0, 0.0)
            attn = attn.view(x.size(0) // n, n, self.heads, x.size(1), x.size(1)) + mask.unsqueeze(1).unsqueeze(0)
            attn = attn.view(-1, self.heads, x.size(1), x.size(1))
        attn = F.softmax(attn, dim=-1)
        x = attn.matmul(v).transpose(1, 2).reshape(x.size(0), x.size(1), C)
        x = F.linear(x, self.proj.weight, self.proj.bias)
        x = x.view(B, pH // w, pW // w, w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B, pH, pW, C)
        if sy + sx > 0:
            x = torch.roll(x, shifts=(sy, sx), dims=(1, 2))
        return x[:, :H, :W, :].contiguous()

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        """x [B H W, C] raster rows, the native kernels."""
        qkv = linear(x, self.qkv.weight, self.qkv.bias)
        o = window_attention(qkv, self.relative_position_bias_table, B, H, W, self.heads, _shifts(self.window, self.shift, H, W))
        return linear(o, self.proj.weight, self.proj.bias)


class SwinTransformerBlock(nn.Module):
    """torchvision's ``SwinTransformerBlock`` keys: ``norm1``, ``attn``, ``norm2`` and ``mlp.0`` Linear(C, 4C) with the erf
    GELU (torchvision's ``mlp.1``) in its epilogue, ``mlp.3`` Linear(4C, C)."""

    def __init__(self, dim: int, heads: int, window: int, shift: int, mlp_ratio: int, eps: float):
        super().__init__()
        self.norm1 = LayerNorm(dim, eps=eps)
        self.attn = ShiftedWindowAttention(dim, heads, window, shift)
        self.norm2 = LayerNorm(dim, eps=eps)
        self.mlp = _Keyed({0: Linear(dim, mlp_ratio * dim, activation="gelu"), 3: Linear(mlp_ratio * dim, dim)})
        for m in self.mlp.modules():                                # torchvision's, overwritten by the model's pass below
            if isinstance(m, Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.normal_(m.bias, std=1e-6)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        x = x + self.attn.forward_rows(self.norm1(x), B, H, W)
        return x + self.mlp(self.norm2(x))


def merge_patches(x: torch.Tensor) -> torch.Tensor:
    """torchvision's patch-merging gather of x [..., H, W, C] (H and W even): [..., H/2, W/2, 4C] holding the pixels
    (0, 0), (1, 0), (0, 1), (1, 1) of each 2 x 2 patch as (row offset, column offset), i.e. in (kx, ky, c) order."""
    return torch.cat([x[..., 0::2, 0::2, :], x[..., 1::2, 0::2, :], x[..., 0::2, 1::2, :], x[..., 1::2, 1::2, :]], -1)


class PatchMerging(nn.Module):
    """torchvision's ``PatchMerging`` keys: the bias-free ``reduction`` Linear(4C, 2C), then ``norm`` LayerNorm(4C)."""

    def __init__(self, dim: int, eps: float):
        super().__init__()
        self.reduction = Linear(4 * dim, 2 * dim, bias=False)
        self.norm = LayerNorm(4 * dim, eps=eps)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, H, W, C], torchvision's arithmetic (an odd H or W is padded by one)."""
        H, W = x.shape[-3], x.shape[-2]
        return self.reduction(self.norm(merge_patches(F.pad(x, (0, 0, 0, W % 2, 0, H % 2)))))

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        return self.reduction(self.norm(merge_patches(x.view(B, H, W, -1)).reshape(B * (H // 2) * (W // 2), -1)))


class SwinTransformer(nn.Module):
    """forward(images [B, 3, H, W]) -> logits [B, num_classes]; ``config`` is the preset."""

    def __init__(self, config: SwinConfig):
        super().__init__()
        c = self.config = config
        if len(c.depths) != len(c.heads):
            raise ValueError(f"SwinConfig: {len(c.depths)} depths for {len(c.heads)} head counts")
        layers = [_Keyed({0: nn.Conv2d(3, c.embed_dim, kernel_size=c.patch, stride=c.patch), 2: LayerNorm(c.embed_dim, eps=c.eps)})]
        for s, (depth, heads) in enumerate(zip(c.depths, c.heads)):
            dim = c.embed_dim * 2 ** s
            layers.append(nn.Sequential(*[SwinTransformerBlock(dim, heads, c.window, 0 if i % 2 == 0 else c.window // 2, c.mlp_ratio, c.eps)
                                          for i in range(depth)]))
            if s + 1 < len(c.depths):
                layers.append(PatchMerging(dim, c.eps))
        self.features = nn.Sequential(*layers)
        width = c.embed_dim * 2 ** (len(c.depths) - 1)
        self.norm = LayerNorm(width, eps=c.eps)
        self.head = Linear(width, c.num_classes)
        # torchvision's scheme: every linear weight normal with std 0.02 cut at +-2 (absolute), zero biases
        for m in self.modules():
            if isinstance(m, Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f"SwinTransformer: expected images [B, 3, H, W], got {tuple(images.shape)}")
        stem = self.features[0][0]
        if images.is_cuda and images.dtype == torch.bfloat16 and stem.weight.dtype == torch.bfloat16:
            return self._forward_rows(images)
        x = self.features[0][2](stem(images).permute(0, 2, 3, 1))
        for layer in list(self.features)[1:]:
            x = layer(x)
        x = F.adaptive_avg_pool2d(self.norm(x).permute(0, 3, 1, 2), 1).flatten(1)
        return self.head(x)

    def _forward_rows(self, images: torch.Tensor) -> torch.Tensor:
        B, _, H, W = images.shape
        if H % INPUT_MULTIPLE or W % INPUT_MULTIPLE:
            raise ValueError(f"SwinTransformer on the native path needs H and W multiples of {INPUT_MULTIPLE}, got {H}x{W}")
        stem, norm = self.features[0][0], self.features[0][2]
        x = layer_norm(_conv_rows(images.permute(0, 2, 3, 1), stem), norm.weight, norm.bias, norm.eps)
        H, W = H // self.config.patch, W // self.config.patch
        for s in range(len(self.config.depths)):
            if s:
                x = self.features[2 * s].forward_rows(x, B, H, W)
                H, W = H // 2, W // 2
            for block in self.features[2 * s + 1]:
                x = block.forward_rows(x, B, H, W)
        x = layer_norm(x, self.norm.weight, self.norm.bias, self.norm.eps)
        return self.head(x.view(B, H * W, -1).mean(1))


def swin_t(num_classes: int = 1000) -> SwinTransformer:
    """Swin-T: embedding 96, depths 2 / 2 / 6 / 2, heads 3 / 6 / 12 / 24 (28,288,354 parameters)."""
    return SwinTransformer(replace(SWIN_T, num_classes=num_classes))


def swin_s(num_classes: int = 1000) -> SwinTransformer:
    """Swin-S: Swin-T's widths and heads, depths 2 / 2 / 18 / 2 (49,606,258 parameters)."""
    return SwinTransformer(replace(SWIN_S, num_classes=num_classes))


def swin_b(num_classes: int = 1000) -> SwinTransformer:
    """Swin-B: embedding 128, depths 2 / 2 / 18 / 2, heads 4 / 8 / 16 / 32 (87,768,224 parameters)."""
    return SwinTransformer(replace(SWIN_B, num_classes=num_classes))
