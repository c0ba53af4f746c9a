"""Masked-autoencoder pretraining of a Vision Transformer (He et al., 2021): ViT-MAE base and large at 224 x 224 with 16 x 16
patches, as ``transformers``' ``ViTMAEForPreTraining`` defines them with ``ViTMAEConfig`` defaults.  Each image keeps
int(196 (1 - 0.75)) = 49 of its patches, chosen per image by ranking random noise; the encoder (pre-LN blocks, LayerNorm eps
1e-12, erf GELU, q / k / v biases, no dropout) sees the class token and those patches, a 512-wide decoder of 8 blocks with
16 heads sees all 196 again (mask tokens at the hidden ones), and the loss is the mean squared pixel error on the hidden
patches (per-patch normalised targets with ``norm_pix_loss``, the paper's setting; transformers' default is off).

The encoder's ``position_embeddings`` and the decoder's ``decoder_pos_embed`` are fixed 2-D sin-cos tables, kept as
``requires_grad=False`` parameters under transformers' keys: optimizers, DDP buckets and gradients skip them.  q / k / v are
one fused ``qkv`` projection per layer; ``load_hf_state_dict`` reads a transformers state dict strictly.

bf16 CUDA input runs the native path on token streams (``csrc/mae.cu``): ``ops.mae_shuffle`` ranks the noise on the device,
``ops.mae_patch_embed`` embeds the kept patches into one stream of 50 rows per image that attends on ``ops.packed_attention``,
``ops.mae_unshuffle`` builds the decoder's stream of 197 rows per image that attends on ``ops.image_attention`` (head dim 32),
and ``ops.mae_loss`` scores ``decoder_pred``'s rows against the image.  Nothing is read back to the host, so a training step
captures into one CUDA graph.  Everything else (CPU, fp32) runs transformers' arithmetic: ``argsort`` / ``gather``, the patch
convolution, per-image SDPA, ``patchify`` in (ky, kx, c) order and ``forward_loss``."""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Callable

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import (LayerNorm, Linear, image_attention, image_token_bounds, mae_loss, mae_loss_reference, mae_patch_embed,
                   mae_shuffle, mae_shuffle_reference, mae_unshuffle, packed_attention)


@dataclass(frozen=True)
class ViTMAEConfig:
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    intermediate: int = 3072
    decoder_hidden: int = 512
    decoder_layers: int = 8
    decoder_heads: int = 16
    decoder_intermediate: int = 2048
    image_size: int = 224
    patch_size: int = 16
    channels: int = 3
    mask_ratio: float = 0.75
    eps: float = 1e-12
    initializer_range: float = 0.02
    norm_pix_loss: bool = False

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2

    @property
    def keep(self) -> int:
        """Patches each image keeps, transformers' ``int(N (1 - mask_ratio))``: 49 of 196."""
        return int(self.num_patches * (1 - self.mask_ratio))


VIT_MAE_BASE = ViTMAEConfig()
VIT_MAE_LARGE = ViTMAEConfig(hidden=1024, layers=24, heads=16, intermediate=4096)


@dataclass
class ViTMAEOutput:
    """transformers' ``ViTMAEForPreTrainingOutput`` fields: loss [], logits [B, N, p p C], mask [B, N] (1 = hidden) and
    ids_restore [B, N] (int64)."""
    loss: torch.Tensor
    logits: torch.Tensor
    mask: torch.Tensor
    ids_restore: torch.Tensor


def sincos_pos_embed(dim: int, grid: int) -> torch.Tensor:
    """transformers' ``get_2d_sincos_pos_embed(dim, grid, add_cls_token=True)`` in fp64: [1 + grid², dim], a zero class row,
    then per raster position (row r, column c) sin | cos of c omega and sin | cos of r omega, omega_k = 10000^(-4k / dim)."""
    omega = 1.0 / 10000 ** (torch.arange(dim // 4, dtype=torch.float64) / (dim / 4))
    pos = torch.arange(grid * grid, dtype=torch.float64)

    def one(coord):
        out = coord[:, None] * omega[None, :]
        return torch.cat([out.sin(), out.cos()], 1)

    emb = torch.cat([one(pos % grid), one(torch.div(pos, grid, rounding_mode="floor"))], 1)
    return torch.cat([torch.zeros(1, dim, dtype=torch.float64), emb], 0)


def _sdpa(qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """Per-image attention on [B, S, 3D] (transformers' SDPA path, no mask)."""
    B, S, W = qkv.shape
    q, k, v = (t.view(B, S, heads, -1).transpose(1, 2) for t in qkv.split(W // 3, dim=-1))
    return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, S, W // 3)


class Dense(nn.Module):
    """One ``dense`` linear: transformers' ``attention.output``, ``intermediate`` and ``output`` key level."""

    def __init__(self, fan_in: int, fan_out: int, activation: str | None = None):
        super().__init__()
        self.dense = Linear(fan_in, fan_out, activation=activation)


class FusedSelfAttention(nn.Module):
    """transformers' ``ViTMAESelfAttention`` with ``query``, ``key`` and ``value`` fused into one ``qkv`` projection [3D, D]."""

    def __init__(self, hidden: int):
        super().__init__()
        self.qkv = Linear(hidden, 3 * hidden)


class Attention(nn.Module):
    def __init__(self, hidden: int):
        super().__init__()
        self.attention = FusedSelfAttention(hidden)
        self.output = Dense(hidden, hidden)


class ViTMAELayer(nn.Module):
    """A pre-LN block: x + output(attend(qkv(layernorm_before(x)))), then x + mlp(layernorm_after(x)).  ``attend(qkv, heads)``
    maps the fused projection to the attention output in the caller's layout."""

    def __init__(self, hidden: int, heads: int, intermediate: int, eps: float):
        super().__init__()
        self.heads = heads
        self.attention = Attention(hidden)
        self.intermediate = Dense(hidden, intermediate, activation="gelu")
        self.output = Dense(intermediate, hidden)
        self.layernorm_before = LayerNorm(hidden, eps=eps)
        self.layernorm_after = LayerNorm(hidden, eps=eps)

    def forward(self, x: torch.Tensor, attend: Callable[[torch.Tensor, int], torch.Tensor]) -> torch.Tensor:
        a = self.attention
        x = x + a.output.dense(attend(a.attention.qkv(self.layernorm_before(x)), self.heads))
        return x + self.output.dense(self.intermediate.dense(self.layernorm_after(x)))


class PatchEmbeddings(nn.Module):
    def __init__(self, c: ViTMAEConfig):
        super().__init__()
        self.projection = nn.Conv2d(c.channels, c.hidden, kernel_size=c.patch_size, stride=c.patch_size)


class Embeddings(nn.Module):
    def __init__(self, c: ViTMAEConfig):
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, c.hidden))
        self.position_embeddings = nn.Parameter(torch.zeros(1, c.num_patches + 1, c.hidden), requires_grad=False)
        self.patch_embeddings = PatchEmbeddings(c)


class Encoder(nn.Module):
    def __init__(self, c: ViTMAEConfig):
        super().__init__()
        self.layer = nn.ModuleList([ViTMAELayer(c.hidden, c.heads, c.intermediate, c.eps) for _ in range(c.layers)])


class ViTMAEModel(nn.Module):
    def __init__(self, c: ViTMAEConfig):
        super().__init__()
        self.embeddings = Embeddings(c)
        self.encoder = Encoder(c)
        self.layernorm = LayerNorm(c.hidden, eps=c.eps)


class ViTMAEDecoder(nn.Module):
    def __init__(self, c: ViTMAEConfig):
        super().__init__()
        self.decoder_embed = Linear(c.hidden, c.decoder_hidden)
        self.mask_token = nn.Parameter(torch.zeros(1, 1, c.decoder_hidden))
        self.decoder_pos_embed = nn.Parameter(torch.zeros(1, c.num_patches + 1, c.decoder_hidden), requires_grad=False)
        self.decoder_layers = nn.ModuleList([ViTMAELayer(c.decoder_hidden, c.decoder_heads, c.decoder_intermediate, c.eps)
                                             for _ in range(c.decoder_layers)])
        self.decoder_norm = LayerNorm(c.decoder_hidden, eps=c.eps)
        self.decoder_pred = Linear(c.decoder_hidden, c.patch_size ** 2 * c.channels)


class ViTMAEForPreTraining(nn.Module):
    """``forward(images [B, 3, 224, 224], noise=None)`` returns the scalar loss; ``pretraining_output`` also returns the
    prediction, the mask and ``ids_restore``.  ``noise`` [B, N] fp32 ranks each image's patches (kept iff the rank is below
    ``config.keep``); without it, ``torch.rand`` on the images' device."""

    def __init__(self, config: ViTMAEConfig):
        super().__init__()
        c = self.config = config
        if c.image_size % c.patch_size or c.hidden % c.heads or c.decoder_hidden % c.decoder_heads:
            raise ValueError(f"ViTMAEConfig: patch size {c.patch_size} must divide image size {c.image_size}, and heads the widths")
        self.vit = ViTMAEModel(c)
        self.decoder = ViTMAEDecoder(c)
        self._init_weights()

    @torch.no_grad()
    def _init_weights(self) -> None:
        """The MAE scheme of transformers' ``initialize_weights`` code: linears normal(0, 0.02) with zero biases, LayerNorms
        ones / zeros, the patch projection Xavier-uniform over its flattened [D, C p p] view with a zero bias, class and mask
        tokens normal(0, 0.02), and the fixed sin-cos position tables.  (A ``ViTMAEForPreTraining`` freshly constructed by
        transformers 5.5 comes out otherwise: its generic ``_init_weights`` runs last and leaves zero tables and tokens and a
        normal(0, 0.02) projection.)"""
        c = self.config
        for m in self.modules():
            if isinstance(m, Linear):
                nn.init.normal_(m.weight, std=c.initializer_range)
                nn.init.zeros_(m.bias)
        w = self.vit.embeddings.patch_embeddings.projection.weight
        nn.init.xavier_uniform_(w.view(w.shape[0], -1))
        nn.init.zeros_(self.vit.embeddings.patch_embeddings.projection.bias)
        nn.init.normal_(self.vit.embeddings.cls_token, std=c.initializer_range)
        nn.init.normal_(self.decoder.mask_token, std=c.initializer_range)
        grid = c.image_size // c.patch_size
        self.vit.embeddings.position_embeddings.copy_(sincos_pos_embed(c.hidden, grid).unsqueeze(0))
        self.decoder.decoder_pos_embed.copy_(sincos_pos_embed(c.decoder_hidden, grid).unsqueeze(0))

    def _check(self, images: torch.Tensor, noise: torch.Tensor | None) -> torch.Tensor:
        c = self.config
        s = c.image_size
        if images.dim() != 4 or tuple(images.shape[1:]) != (c.channels, s, s):
            raise ValueError(f"ViTMAEForPreTraining: expected images [B, {c.channels}, {s}, {s}], got {tuple(images.shape)}")
        if noise is None:
            return torch.rand(images.shape[0], c.num_patches, device=images.device)
        if tuple(noise.shape) != (images.shape[0], c.num_patches):
            raise ValueError(f"ViTMAEForPreTraining: expected noise [{images.shape[0]}, {c.num_patches}], got {tuple(noise.shape)}")
        return noise

    def forward(self, images: torch.Tensor, noise: torch.Tensor | None = None) -> torch.Tensor:
        return self._run(images, noise)[0]

    def pretraining_output(self, images: torch.Tensor, noise: torch.Tensor | None = None) -> ViTMAEOutput:
        loss, logits, ids_restore = self._run(images, noise)
        return ViTMAEOutput(loss, logits, (ids_restore >= self.config.keep).float(), ids_restore.long())

    def _run(self, images: torch.Tensor, noise: torch.Tensor | None):
        """(loss, logits [B, N, p p C], ids_restore [B, N]) on the native path or transformers' arithmetic."""
        noise = self._check(images, noise)
        w = self.vit.embeddings.patch_embeddings.projection.weight
        if images.is_cuda and images.dtype == torch.bfloat16 and w.dtype == torch.bfloat16:
            return self._native(images, noise)
        return self._reference(images, noise)

    def _native(self, images: torch.Tensor, noise: torch.Tensor):
        c, B = self.config, images.shape[0]
        N, keep = c.num_patches, c.keep
        e, d = self.vit.embeddings, self.decoder
        ids_keep, ids_restore = mae_shuffle(noise, keep)
        x = mae_patch_embed(images, e.patch_embeddings.projection.weight, e.patch_embeddings.projection.bias, e.cls_token,
                            e.position_embeddings, ids_keep)
        T = x.shape[0]
        bounds = image_token_bounds(B, keep + 1, images.device)
        for layer in self.vit.encoder.layer:
            x = layer(x, lambda qkv, heads: packed_attention(qkv.view(1, T, -1), bounds, heads).view(T, -1))
        z = mae_unshuffle(d.decoder_embed(self.vit.layernorm(x)), d.mask_token, d.decoder_pos_embed, ids_keep, ids_restore)
        for layer in d.decoder_layers:
            z = layer(z, lambda qkv, heads: image_attention(qkv, B, N + 1, heads))
        pred = d.decoder_pred(d.decoder_norm(z))
        loss = mae_loss(pred, images, ids_restore, keep, c.norm_pix_loss)
        return loss, pred[:B * (N + 1)].view(B, N + 1, -1)[:, 1:], ids_restore

    def _reference(self, images: torch.Tensor, noise: torch.Tensor):
        c, B = self.config, images.shape[0]
        N, keep = c.num_patches, c.keep
        e, d = self.vit.embeddings, self.decoder
        pos = e.position_embeddings
        x = e.patch_embeddings.projection(images).flatten(2).transpose(1, 2) + pos[:, 1:]
        ids_keep, ids_restore = mae_shuffle_reference(noise, keep)
        x = torch.gather(x, 1, ids_keep.unsqueeze(-1).expand(-1, -1, c.hidden))
        x = torch.cat([(e.cls_token + pos[:, :1]).expand(B, -1, -1), x], 1)
        for layer in self.vit.encoder.layer:
            x = layer(x, _sdpa)
        y = d.decoder_embed(self.vit.layernorm(x))
        x_ = torch.cat([y[:, 1:], d.mask_token.expand(B, N - keep, -1)], 1)
        x_ = torch.gather(x_, 1, ids_restore.unsqueeze(-1).expand(-1, -1, c.decoder_hidden))
        z = torch.cat([y[:, :1], x_], 1) + d.decoder_pos_embed
        for layer in d.decoder_layers:
            z = layer(z, _sdpa)
        pred = d.decoder_pred(d.decoder_norm(z))
        loss = mae_loss_reference(pred.reshape(B * (N + 1), -1), images, ids_restore, keep, c.norm_pix_loss)
        return loss, pred[:, 1:], ids_restore

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.ViTMAEForPreTraining`` state dict strictly (a missing or unexpected key raises): each layer's
        query / key / value fused into ``qkv``, every other key as it is."""
        own = self.state_dict()
        out, used = {}, set()
        for key in own:
            if ".attention.attention.qkv." in key:
                stem, wb = key.rsplit(".qkv.", 1)
                parts = [f"{stem}.{x}.{wb}" for x in ("query", "key", "value")]
                out[key] = torch.cat([hf[k] for k in parts]).to(own[key].dtype)
                used.update(parts)
            else:
                out[key] = hf[key].to(own[key].dtype)
                used.add(key)
        unknown = set(hf) - used
        if unknown:
            raise KeyError(f"load_hf_state_dict: unexpected keys {sorted(unknown)[:8]}")
        self.load_state_dict(out, strict=True)


def vit_mae_base(norm_pix_loss: bool = False) -> ViTMAEForPreTraining:
    """ViT-MAE base: encoder 12 layers, hidden 768, 12 heads, MLP 3072; decoder 8 layers, 512 wide, 16 heads, MLP 2048
    (111,907,840 parameters, 111,655,680 trainable)."""
    return ViTMAEForPreTraining(replace(VIT_MAE_BASE, norm_pix_loss=norm_pix_loss))


def vit_mae_large(norm_pix_loss: bool = False) -> ViTMAEForPreTraining:
    """ViT-MAE large: encoder 24 layers, hidden 1024, 16 heads, MLP 4096; the base's decoder (329,541,888 parameters,
    329,239,296 trainable)."""
    return ViTMAEForPreTraining(replace(VIT_MAE_LARGE, norm_pix_loss=norm_pix_loss))
