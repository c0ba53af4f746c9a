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
arithmetic, padding included.

Swin Transformer V2 (Liu et al., 2022): Swin-V2-T, -S and -B at 256 x 256, torchvision's ``swin_v2_t`` and the others
with the same keys, shapes, registration order and initialisation.  Window 8; each block is x + norm1(attn(x)),
x + norm2(mlp(x)) (res-post-norm); the attention scores are exp(min(logit_scale, log 100)) cos(q, k) plus
16 sigmoid(cpb_mlp(relative_coords_table)), a 2 -> 512 -> heads MLP over log-spaced relative coordinates; the k third
of the qkv bias is held at zero; patch merging reduces 4C -> 2C before its LayerNorm.  Natively the attention is
``ops.window_attention_v2``; the logit-scale clamp and exponential and the MLP table are small torch ops (fp32
parameters, ``keep_fp32_params``) whose gradients come back from the kernel.  The native path needs H and W multiples
of 256."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import (LayerNorm, Linear, layer_norm, linear, swin_relative_position_index, swin_v2_relative_coords_table, window_attention,
                   window_attention_v2)
from ..ops.functional import SWIN_MASK, SWIN_V2_WINDOW, SWIN_WINDOW
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
    v2: bool = False                   # Swin V2's blocks, attention and patch merging


SWIN_T = SwinConfig(embed_dim=96, depths=(2, 2, 6, 2), heads=(3, 6, 12, 24))
SWIN_S = SwinConfig(embed_dim=96, depths=(2, 2, 18, 2), heads=(3, 6, 12, 24))
SWIN_B = SwinConfig(embed_dim=128, depths=(2, 2, 18, 2), heads=(4, 8, 16, 32))
SWIN_V2_T = SwinConfig(embed_dim=96, depths=(2, 2, 6, 2), heads=(3, 6, 12, 24), window=SWIN_V2_WINDOW, v2=True)
SWIN_V2_S = SwinConfig(embed_dim=96, depths=(2, 2, 18, 2), heads=(3, 6, 12, 24), window=SWIN_V2_WINDOW, v2=True)
SWIN_V2_B = SwinConfig(embed_dim=128, depths=(2, 2, 18, 2), heads=(4, 8, 16, 32), window=SWIN_V2_WINDOW, v2=True)

# the native path downsamples by 4 x 2 x 2 x 2 and needs every stage to be whole 7 x 7 windows (V2: 8 x 8, so 256)
INPUT_MULTIPLE = 224


def _shifts(window: int, shift: int, height: int, width: int) -> tuple[int, int]:
    """torchvision's rule: no shift along a dimension the window covers whole."""
    return (0 if window >= height else shift, 0 if window >= width else shift)


def _shifted_window_attention(x, qkv_weight, qkv_bias, proj_weight, proj_bias, bias, w, heads, shift, logit_scale=None):
    """x [B, H, W, C], torchvision's ``shifted_window_attention`` arithmetic (padding to whole windows included); bias
    [1, heads, w^2, w^2]; V2's cosine scores when ``logit_scale`` [heads, 1, 1] is given."""
    B, H, W, C = x.shape
    x = F.pad(x, (0, 0, 0, (w - W % w) % w, 0, (w - H % w) % w))
    _, pH, pW, _ = x.shape
    sy, sx = _shifts(w, shift, pH, pW)
    if sy + sx > 0:
        x = torch.roll(x, shifts=(-sy, -sx), dims=(1, 2))
    n = (pH // w) * (pW // w)
    x = x.view(B, pH // w, w, pW // w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B * n, w * w, C)
    if logit_scale is not None:
        qkv_bias = qkv_bias.clone()
        qkv_bias[C:2 * C].zero_()
    qkv = F.linear(x, qkv_weight, qkv_bias)
    qkv = qkv.reshape(x.size(0), x.size(1), 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if logit_scale is not None:
        attn = F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-2, -1)
        attn = attn * torch.clamp(logit_scale, max=math.log(100.0)).exp()
    else:
        q = q * (C // heads) ** -0.5
        attn = q.matmul(k.transpose(-2, -1))
    attn = attn + bias
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
        attn = attn.view(x.size(0) // n, n, heads, x.size(1), x.size(1)) + mask.unsqueeze(1).unsqueeze(0)
        attn = attn.view(-1, heads, x.size(1), x.size(1))
    attn = F.softmax(attn, dim=-1)
    x = attn.matmul(v).transpose(1, 2).reshape(x.size(0), x.size(1), C)
    x = F.linear(x, proj_weight, proj_bias)
    x = x.view(B, pH // w, pW // w, w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B, pH, pW, C)
    if sy + sx > 0:
        x = torch.roll(x, shifts=(sy, sx), dims=(1, 2))
    return x[:, :H, :W, :].contiguous()


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
        w = self.window
        bias = self.relative_position_bias_table[self.relative_position_index].view(w * w, w * w, -1)
        return _shifted_window_attention(x, self.qkv.weight, self.qkv.bias, self.proj.weight, self.proj.bias,
                                         bias.permute(2, 0, 1).contiguous().unsqueeze(0), w, self.heads, self.shift)

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        """x [B H W, C] raster rows, the native kernels."""
        qkv = linear(x, self.qkv.weight, self.qkv.bias)
        o = window_attention(qkv, self.relative_position_bias_table, B, H, W, self.heads, _shifts(self.window, self.shift, H, W))
        return linear(o, self.proj.weight, self.proj.bias)


class ShiftedWindowAttentionV2(nn.Module):
    """torchvision's ``ShiftedWindowAttentionV2`` keys: ``qkv`` Linear(C, 3C) whose k third of the bias is held at zero,
    ``proj`` Linear(C, C), the persistent ``relative_coords_table`` [1, 15, 15, 2] and int64 ``relative_position_index``
    [4096] buffers, ``logit_scale`` [heads, 1, 1] = log 10, and ``cpb_mlp.0`` Linear(2, 512), ReLU, ``cpb_mlp.2``
    Linear(512, heads, bias=False).  ``logit_scale`` and the MLP stay fp32 under bf16 training: the kernel reads
    exp(logit_scale) and the sigmoid table in fp32, which bf16 weights would round."""
    keep_fp32_params = ("logit_scale", "cpb_mlp.0.weight", "cpb_mlp.0.bias", "cpb_mlp.2.weight")

    def __init__(self, dim: int, heads: int, window: int, shift: int):
        super().__init__()
        self.heads, self.window, self.shift = heads, window, shift
        self.qkv = Linear(dim, 3 * dim)
        self.proj = Linear(dim, dim)
        self.register_buffer("relative_coords_table", swin_v2_relative_coords_table(window))
        self.register_buffer("relative_position_index", swin_relative_position_index(window=window))
        self.logit_scale = nn.Parameter(torch.log(10 * torch.ones((heads, 1, 1))))
        self.cpb_mlp = nn.Sequential(nn.Linear(2, 512, bias=True), nn.ReLU(inplace=True), nn.Linear(512, heads, bias=False))
        with torch.no_grad():
            self.qkv.bias[dim:2 * dim].zero_()

    def bias_table(self) -> torch.Tensor:
        """[(2w - 1)^2, heads]: 16 sigmoid(cpb_mlp(relative_coords_table)) in the MLP's dtype."""
        coords = self.relative_coords_table
        if coords.dtype != self.cpb_mlp[0].weight.dtype:      # a bf16 model rounds the buffer; the MLP reads it exactly
            coords = swin_v2_relative_coords_table(self.window, coords.device).to(self.cpb_mlp[0].weight.dtype)
        return 16 * torch.sigmoid(self.cpb_mlp(coords).view(-1, self.heads))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, H, W, C], torchvision's arithmetic (padding to whole windows included)."""
        w = self.window
        table = self.cpb_mlp(self.relative_coords_table).view(-1, self.heads)
        bias = 16 * torch.sigmoid(table[self.relative_position_index].view(w * w, w * w, -1).permute(2, 0, 1).contiguous().unsqueeze(0))
        return _shifted_window_attention(x, self.qkv.weight, self.qkv.bias, self.proj.weight, self.proj.bias, bias, w, self.heads,
                                         self.shift, self.logit_scale)

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        """x [B H W, C] raster rows, the native kernels; the k bias enters as an exact zero, so its gradient is zero."""
        C = x.shape[1]
        b = self.qkv.bias
        qkv = linear(x, self.qkv.weight, torch.cat([b[:C], torch.zeros_like(b[C:2 * C]), b[2 * C:]]))
        scale = torch.clamp(self.logit_scale, max=math.log(100.0)).exp().view(-1)
        o = window_attention_v2(qkv, self.bias_table(), scale, B, H, W, self.heads, _shifts(self.window, self.shift, H, W))
        return linear(o, self.proj.weight, self.proj.bias)


class SwinTransformerBlock(nn.Module):
    """torchvision's ``SwinTransformerBlock`` keys: ``norm1``, ``attn``, ``norm2`` and ``mlp.0`` Linear(C, 4C) with the erf
    GELU (torchvision's ``mlp.1``) in its epilogue, ``mlp.3`` Linear(4C, C)."""
    attention = ShiftedWindowAttention

    def __init__(self, dim: int, heads: int, window: int, shift: int, mlp_ratio: int, eps: float):
        super().__init__()
        self.norm1 = LayerNorm(dim, eps=eps)
        self.attn = self.attention(dim, heads, window, shift)
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


class SwinTransformerBlockV2(SwinTransformerBlock):
    """torchvision's ``SwinTransformerBlockV2``: V1's keys with ``ShiftedWindowAttentionV2``, and res-post-norm,
    x + norm1(attn(x)), x + norm2(mlp(x))."""
    attention = ShiftedWindowAttentionV2

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x + self.norm1(self.attn(x))
        return x + self.norm2(self.mlp(x))

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        x = x + self.norm1(self.attn.forward_rows(x, B, H, W))
        return x + self.norm2(self.mlp(x))


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


class PatchMergingV2(nn.Module):
    """torchvision's ``PatchMergingV2`` keys: the bias-free ``reduction`` Linear(4C, 2C), then ``norm`` LayerNorm(2C)."""

    def __init__(self, dim: int, eps: float):
        super().__init__()
        self.reduction = Linear(4 * dim, 2 * dim, bias=False)
        self.norm = LayerNorm(2 * dim, eps=eps)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, H, W, C], torchvision's arithmetic (an odd H or W is padded by one)."""
        H, W = x.shape[-3], x.shape[-2]
        return self.norm(self.reduction(merge_patches(F.pad(x, (0, 0, 0, W % 2, 0, H % 2)))))

    def forward_rows(self, x: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
        return self.norm(self.reduction(merge_patches(x.view(B, H, W, -1)).reshape(B * (H // 2) * (W // 2), -1)))


class SwinTransformer(nn.Module):
    """forward(images [B, 3, H, W]) -> logits [B, num_classes]; ``config`` is the preset."""

    def __init__(self, config: SwinConfig):
        super().__init__()
        c = self.config = config
        if len(c.depths) != len(c.heads):
            raise ValueError(f"SwinConfig: {len(c.depths)} depths for {len(c.heads)} head counts")
        block, merging = (SwinTransformerBlockV2, PatchMergingV2) if c.v2 else (SwinTransformerBlock, PatchMerging)
        layers = [_Keyed({0: nn.Conv2d(3, c.embed_dim, kernel_size=c.patch, stride=c.patch), 2: LayerNorm(c.embed_dim, eps=c.eps)})]
        for s, (depth, heads) in enumerate(zip(c.depths, c.heads)):
            dim = c.embed_dim * 2 ** s
            layers.append(nn.Sequential(*[block(dim, heads, c.window, 0 if i % 2 == 0 else c.window // 2, c.mlp_ratio, c.eps)
                                          for i in range(depth)]))
            if s + 1 < len(c.depths):
                layers.append(merging(dim, c.eps))
        self.features = nn.Sequential(*layers)
        width = c.embed_dim * 2 ** (len(c.depths) - 1)
        self.norm = LayerNorm(width, eps=c.eps)
        self.head = Linear(width, c.num_classes)
        # torchvision's scheme: every linear weight normal with std 0.02 cut at +-2 (absolute), zero biases (V2's cpb MLP too)
        for m in self.modules():
            if isinstance(m, (Linear, nn.Linear)):
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
        multiple = INPUT_MULTIPLE if self.config.window == SWIN_WINDOW else 32 * self.config.window
        if H % multiple or W % multiple:
            raise ValueError(f"SwinTransformer on the native path needs H and W multiples of {multiple}, got {H}x{W}")
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


def swin_v2_t(num_classes: int = 1000) -> SwinTransformer:
    """Swin-V2-T: embedding 96, depths 2 / 2 / 6 / 2, heads 3 / 6 / 12 / 24, window 8 (28,351,570 parameters)."""
    return SwinTransformer(replace(SWIN_V2_T, num_classes=num_classes))


def swin_v2_s(num_classes: int = 1000) -> SwinTransformer:
    """Swin-V2-S: Swin-V2-T's widths and heads, depths 2 / 2 / 18 / 2 (49,737,442 parameters)."""
    return SwinTransformer(replace(SWIN_V2_S, num_classes=num_classes))


def swin_v2_b(num_classes: int = 1000) -> SwinTransformer:
    """Swin-V2-B: embedding 128, depths 2 / 2 / 18 / 2, heads 4 / 8 / 16 / 32, window 8 (87,930,848 parameters)."""
    return SwinTransformer(replace(SWIN_V2_B, num_classes=num_classes))
