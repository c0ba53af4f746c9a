"""Vision Transformer (Dosovitskiy et al., 2020) for image classification: ViT-B/16, ViT-B/32 and ViT-L/16 at 224 x 224,
with torchvision's module and parameter names, shapes, registration order and initialisation (``torchvision.models.vit_b_16``
and the others), so ``load_state_dict`` takes a torchvision state dict strictly and DDP buckets match.  Pre-norm blocks:
x + out_proj(attention(ln_1(x))), then x + mlp(ln_2(x)); LayerNorm eps 1e-6, erf GELU, no dropout; the class token's
row goes through ``encoder.ln`` and ``heads.head``.

bf16 CUDA input runs on the native kernels with the whole batch as one token stream (``ops.patch_embed``): each image's
N + 1 tokens are one document of ``ops.image_token_bounds``, the stream is padded to a multiple of 128 rows, every linear
runs on all rows and attention is ``ops.packed_attention`` on the document bounds.  Anything else (CPU, fp32 on CUDA)
runs torchvision's arithmetic: the patch convolution and per-image attention on [B, heads, N + 1, head dim]."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, causal_attention, image_token_bounds, linear, packed_attention, patch_embed


@dataclass(frozen=True)
class ViTConfig:
    patch_size: int
    layers: int
    heads: int
    hidden: int
    mlp_dim: int
    image_size: int = 224
    num_classes: int = 1000
    eps: float = 1e-6

    @property
    def tokens(self) -> int:
        """Tokens per image: the patches and the class token."""
        return (self.image_size // self.patch_size) ** 2 + 1


VIT_B_16 = ViTConfig(patch_size=16, layers=12, heads=12, hidden=768, mlp_dim=3072)
VIT_B_32 = ViTConfig(patch_size=32, layers=12, heads=12, hidden=768, mlp_dim=3072)
VIT_L_16 = ViTConfig(patch_size=16, layers=24, heads=16, hidden=1024, mlp_dim=4096)


class SelfAttention(nn.Module):
    """``nn.MultiheadAttention``'s parameters: the fused q | k | v projection ``in_proj_weight`` [3D, D] (the column layout
    the attention kernels read) with ``in_proj_bias``, and ``out_proj``.  ``causal=True`` (CLIP's text tower) attends
    causally: ``causal_attention`` on the token stream, SDPA's causal mask per sequence."""

    def __init__(self, hidden: int, heads: int, causal: bool = False):
        super().__init__()
        self.heads = heads
        self.causal = causal
        self.in_proj_weight = nn.Parameter(torch.empty(3 * hidden, hidden))
        self.in_proj_bias = nn.Parameter(torch.empty(3 * hidden))
        self.out_proj = Linear(hidden, hidden)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.in_proj_bias)
        nn.init.zeros_(self.out_proj.bias)

    def forward(self, x: torch.Tensor, bounds: torch.Tensor | None = None) -> torch.Tensor:
        qkv = linear(x, self.in_proj_weight, self.in_proj_bias)
        if bounds is not None:                       # the token stream [T, D]: each image one document
            T = qkv.shape[0]
            attend = causal_attention if self.causal else packed_attention
            return self.out_proj(attend(qkv.view(1, T, -1), bounds, self.heads).view(T, -1))
        B, S, W = qkv.shape                          # [B, N + 1, 3D]: per image (or caption), no mask or the causal one
        q, k, v = (t.view(B, S, self.heads, -1).transpose(1, 2) for t in qkv.split(W // 3, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=self.causal)
        return self.out_proj(o.transpose(1, 2).reshape(B, S, W // 3))


class MLPBlock(nn.Module):
    """torchvision's ``MLPBlock`` keys: ``0`` (with the erf GELU, torchvision's ``1``, in its epilogue, or another
    ``activation`` of ``ops.linear``) and ``3``; its dropouts (``2``, ``4``) are identities at torchvision's default rate 0."""

    def __init__(self, hidden: int, mlp_dim: int, activation: str = "gelu"):
        super().__init__()
        self.add_module("0", Linear(hidden, mlp_dim, activation=activation))
        self.add_module("3", Linear(mlp_dim, hidden))
        for m in (self[0], self[3]):
            nn.init.xavier_uniform_(m.weight)
            nn.init.normal_(m.bias, std=1e-6)

    def __getitem__(self, i: int) -> Linear:
        return self._modules[str(i)]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self[3](self[0](x))


class EncoderBlock(nn.Module):
    """A pre-norm block on any config with ``hidden``, ``heads``, ``mlp_dim`` and ``eps``; ``activation`` is the MLP's and
    ``causal`` the attention's (CLIP's towers use QuickGELU, its text tower causal attention)."""

    def __init__(self, c: ViTConfig, activation: str = "gelu", causal: bool = False):
        super().__init__()
        self.ln_1 = LayerNorm(c.hidden, eps=c.eps)
        self.self_attention = SelfAttention(c.hidden, c.heads, causal)
        self.ln_2 = LayerNorm(c.hidden, eps=c.eps)
        self.mlp = MLPBlock(c.hidden, c.mlp_dim, activation)

    def forward(self, x: torch.Tensor, bounds: torch.Tensor | None = None) -> torch.Tensor:
        x = x + self.self_attention(self.ln_1(x), bounds)
        return x + self.mlp(self.ln_2(x))


class Encoder(nn.Module):
    def __init__(self, c: ViTConfig):
        super().__init__()
        self.pos_embedding = nn.Parameter(torch.empty(1, c.tokens, c.hidden).normal_(std=0.02))
        self.layers = nn.Sequential()
        for i in range(c.layers):
            self.layers.add_module(f"encoder_layer_{i}", EncoderBlock(c))
        self.ln = LayerNorm(c.hidden, eps=c.eps)


class VisionTransformer(nn.Module):
    """forward(images [B, 3, S, S]) -> logits [B, num_classes]; ``config`` is the preset."""

    def __init__(self, config: ViTConfig):
        super().__init__()
        c = self.config = config
        if c.image_size % c.patch_size or c.hidden % c.heads:
            raise ValueError(f"ViTConfig: patch size {c.patch_size} must divide image size {c.image_size} and heads {c.heads} "
                             f"hidden {c.hidden}")
        self.conv_proj = nn.Conv2d(3, c.hidden, kernel_size=c.patch_size, stride=c.patch_size)
        self.class_token = nn.Parameter(torch.zeros(1, 1, c.hidden))
        self.encoder = Encoder(c)
        self.heads = nn.Sequential()
        self.heads.add_module("head", Linear(c.hidden, c.num_classes))
        # torchvision's scheme (besides the blocks' own): patch weight normal cut at +-2 (absolute) with std 1 / sqrt(fan in),
        # zero patch bias, zero class token, zero head
        fan_in = 3 * c.patch_size * c.patch_size
        nn.init.trunc_normal_(self.conv_proj.weight, std=math.sqrt(1 / fan_in))
        nn.init.zeros_(self.conv_proj.bias)
        nn.init.zeros_(self.heads.head.weight)
        nn.init.zeros_(self.heads.head.bias)

    def _check(self, images: torch.Tensor) -> None:
        s = self.config.image_size
        if images.dim() != 4 or tuple(images.shape[1:]) != (3, s, s):
            raise ValueError(f"VisionTransformer: expected images [B, 3, {s}, {s}], got {tuple(images.shape)}")

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        self._check(images)
        c, B = self.config, images.shape[0]
        w = self.conv_proj.weight
        if images.is_cuda and images.dtype == torch.bfloat16 and w.dtype == torch.bfloat16:
            x = patch_embed(images, w, self.conv_proj.bias, self.class_token, self.encoder.pos_embedding)
            bounds = image_token_bounds(B, c.tokens, images.device)
            for layer in self.encoder.layers:
                x = layer(x, bounds)
            cls = x[:B * c.tokens:c.tokens]                  # the B class-token rows (a strided view)
        else:
            x = self.conv_proj(images).flatten(2).transpose(1, 2)
            x = torch.cat([self.class_token.expand(B, -1, -1), x], 1) + self.encoder.pos_embedding
            for layer in self.encoder.layers:
                x = layer(x)
            cls = x[:, 0]
        # LayerNorm is per row: normalising the class rows alone equals torchvision's ln(x)[:, 0]
        return self.heads.head(self.encoder.ln(cls))


def vit_b_16(num_classes: int = 1000) -> VisionTransformer:
    """ViT-B/16: 12 layers, hidden 768, 12 heads, MLP 3072, 197 tokens per image (86,567,656 parameters)."""
    return VisionTransformer(replace(VIT_B_16, num_classes=num_classes))


def vit_b_32(num_classes: int = 1000) -> VisionTransformer:
    """ViT-B/32: as ViT-B/16 with 32 x 32 patches, 50 tokens per image (88,224,232 parameters)."""
    return VisionTransformer(replace(VIT_B_32, num_classes=num_classes))


def vit_l_16(num_classes: int = 1000) -> VisionTransformer:
    """ViT-L/16: 24 layers, hidden 1024, 16 heads, MLP 4096, 197 tokens per image (304,326,632 parameters)."""
    return VisionTransformer(replace(VIT_L_16, num_classes=num_classes))
