"""CLIP (Radford et al., 2021) image-text training: CLIP-ViT-B/32 and CLIP-ViT-B/16 with transformers' ``CLIPConfig``
defaults (projection dim 512, LayerNorm eps 1e-5, QuickGELU in both towers, ``logit_scale`` initialised to 2.6592).
The vision tower is ``models/vit.py``'s encoder block with QuickGELU and eps 1e-5 (width 768, 12 layers, 12 heads, MLP
3072); the text tower is the same block with causal attention (vocab 49408, 77 positions, width 512, 12 layers, 8 heads,
MLP 2048).  ``forward(images, input_ids)`` returns ``(image_embeds, text_embeds, logit_scale)``, the embeds unnormalised
as ``CLIPModel.get_image_features`` / ``get_text_features`` return them; ``ops.clip_loss`` is the training loss.

bf16 CUDA input runs on the native kernels, each batch as token streams:
- images: ``ops.patch_embed`` (no patch bias), each image one document of ``ops.image_token_bounds``, ``pre_layrnorm``
  on the stream, ``post_layernorm`` on the B class rows;
- captions: all B captions one stream of round_up(77 B, 128) rows, token plus position embedding, padding rows zero.
  Caption b is the causal document [77 b, 77 b + e_b + 1) with e_b its first EOT (``ops.caption_token_bounds``), rows
  after the EOT attend to nothing, and ``final_layer_norm`` runs on the B pooled (EOT) rows.
Every linear runs on all rows of its stream.  Anything else (CPU, fp32 on CUDA) runs transformers' arithmetic: the patch
convolution, and per-sequence attention with SDPA (the causal mask for captions).

``load_hf_state_dict`` reads a ``transformers.CLIPModel`` state dict strictly: every key is consumed, every parameter
written, and q | k | v are fused into the one [3D, D] projection the attention kernels read."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, caption_token_bounds, image_token_bounds, patch_embed
from .vit import EncoderBlock


@dataclass(frozen=True)
class CLIPTowerConfig:
    hidden: int
    layers: int
    heads: int
    mlp_dim: int
    eps: float = 1e-5


@dataclass(frozen=True)
class CLIPConfig:
    patch_size: int
    image_size: int = 224
    vision: CLIPTowerConfig = CLIPTowerConfig(hidden=768, layers=12, heads=12, mlp_dim=3072)
    text: CLIPTowerConfig = CLIPTowerConfig(hidden=512, layers=12, heads=8, mlp_dim=2048)
    vocab_size: int = 49408
    max_position: int = 77
    projection_dim: int = 512
    logit_scale_init: float = 2.6592
    bos_token_id: int = 49406              # <|startoftext|>
    eos_token_id: int = 49407              # <|endoftext|>
    activation: str = "quick_gelu"

    @property
    def tokens(self) -> int:
        """Tokens per image: the patches and the class token."""
        return (self.image_size // self.patch_size) ** 2 + 1


CLIP_VIT_B_32 = CLIPConfig(patch_size=32)
CLIP_VIT_B_16 = CLIPConfig(patch_size=16)


def _encoder(c: CLIPTowerConfig, activation: str, causal: bool) -> nn.ModuleList:
    layers = nn.ModuleList(EncoderBlock(c, activation, causal) for _ in range(c.layers))
    # CLIPPreTrainedModel._init_weights: q / k / v and fc2 normal with std D^-0.5 (2 layers)^-0.5, out_proj D^-0.5,
    # fc1 (2 D)^-0.5, every linear bias and LayerNorm bias zero, LayerNorm weight one
    in_std = c.hidden ** -0.5 * (2 * c.layers) ** -0.5
    for blk in layers:
        att, mlp = blk.self_attention, blk.mlp
        nn.init.normal_(att.in_proj_weight, std=in_std)
        nn.init.normal_(att.out_proj.weight, std=c.hidden ** -0.5)
        nn.init.normal_(mlp[0].weight, std=(2 * c.hidden) ** -0.5)
        nn.init.normal_(mlp[3].weight, std=in_std)
        for b in (att.in_proj_bias, att.out_proj.bias, mlp[0].bias, mlp[3].bias):
            nn.init.zeros_(b)
    return layers


class CLIPVisionTower(nn.Module):
    def __init__(self, c: CLIPConfig):
        super().__init__()
        v = c.vision
        self.config = c
        self.class_embedding = nn.Parameter(torch.empty(v.hidden).normal_(std=v.hidden ** -0.5))
        self.patch_embedding = nn.Conv2d(3, v.hidden, kernel_size=c.patch_size, stride=c.patch_size, bias=False)
        self.position_embedding = nn.Embedding(c.tokens, v.hidden)
        nn.init.normal_(self.patch_embedding.weight, std=0.02)
        nn.init.normal_(self.position_embedding.weight, std=0.02)
        self.pre_layrnorm = LayerNorm(v.hidden, eps=v.eps)
        self.layers = _encoder(v, c.activation, causal=False)
        self.post_layernorm = LayerNorm(v.hidden, eps=v.eps)

    def forward(self, images: torch.Tensor) -> torch.Tensor:
        """Pooled (class-token) features [B, width] after ``post_layernorm``."""
        c, B = self.config, images.shape[0]
        w = self.patch_embedding.weight
        if images.is_cuda and images.dtype == torch.bfloat16 and w.dtype == torch.bfloat16:
            x = patch_embed(images, w, None, self.class_embedding, self.position_embedding.weight)
            x = self.pre_layrnorm(x)
            bounds = image_token_bounds(B, c.tokens, images.device)
            for layer in self.layers:
                x = layer(x, bounds)
            cls = x[:B * c.tokens:c.tokens]                  # the B class-token rows (a strided view)
        else:
            x = self.patch_embedding(images.to(w.dtype)).flatten(2).transpose(1, 2)
            x = torch.cat([self.class_embedding.expand(B, 1, -1), x], 1) + self.position_embedding.weight
            x = self.pre_layrnorm(x)
            for layer in self.layers:
                x = layer(x)
            cls = x[:, 0]
        return self.post_layernorm(cls)


class CLIPTextTower(nn.Module):
    def __init__(self, c: CLIPConfig):
        super().__init__()
        t = c.text
        self.config = c
        self.token_embedding = nn.Embedding(c.vocab_size, t.hidden)
        self.position_embedding = nn.Embedding(c.max_position, t.hidden)
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.position_embedding.weight, std=0.02)
        self.layers = _encoder(t, c.activation, causal=True)
        self.final_layer_norm = LayerNorm(t.hidden, eps=t.eps)

    def forward(self, input_ids: torch.Tensor) -> torch.Tensor:
        """Pooled (first-EOT) features [B, width] after ``final_layer_norm``."""
        c = self.config
        B, L = input_ids.shape
        x = self.token_embedding(input_ids) + self.position_embedding(torch.arange(L, device=input_ids.device))
        if input_ids.is_cuda and x.dtype == torch.bfloat16:
            bounds, pooled = caption_token_bounds(input_ids, c.eos_token_id)
            x = F.pad(x.reshape(B * L, -1), (0, 0, 0, bounds.shape[1] - B * L))       # zero padding rows
            for layer in self.layers:
                x = layer(x, bounds)
            return self.final_layer_norm(x[pooled])
        for layer in self.layers:
            x = layer(x)
        eot = (input_ids == c.eos_token_id).int().argmax(-1)
        return self.final_layer_norm(x[torch.arange(B, device=x.device), eot])


class CLIPModel(nn.Module):
    """forward(images [B, 3, S, S], input_ids [B, 77]) -> (image_embeds [B, 512], text_embeds [B, 512], logit_scale).

    ``logit_scale`` is named in ``keep_fp32_params``: under ``--fp16`` it stays an fp32 parameter, as exp(logit_scale) in
    bf16 would be 0.3 % off at its initial value."""

    keep_fp32_params = ("logit_scale",)

    def __init__(self, config: CLIPConfig):
        super().__init__()
        c = self.config = config
        for t in (c.vision, c.text):
            if t.hidden % t.heads:
                raise ValueError(f"CLIPConfig: heads {t.heads} must divide width {t.hidden}")
        if c.image_size % c.patch_size:
            raise ValueError(f"CLIPConfig: patch size {c.patch_size} must divide image size {c.image_size}")
        self.vision_model = CLIPVisionTower(c)
        self.text_model = CLIPTextTower(c)
        self.visual_projection = Linear(c.vision.hidden, c.projection_dim, bias=False)
        self.text_projection = Linear(c.text.hidden, c.projection_dim, bias=False)
        nn.init.normal_(self.visual_projection.weight, std=c.vision.hidden ** -0.5)
        nn.init.normal_(self.text_projection.weight, std=c.text.hidden ** -0.5)
        self.logit_scale = nn.Parameter(torch.tensor(c.logit_scale_init))

    def _check(self, images: torch.Tensor, input_ids: torch.Tensor) -> None:
        s, L = self.config.image_size, self.config.max_position
        if images.dim() != 4 or tuple(images.shape[1:]) != (3, s, s):
            raise ValueError(f"CLIPModel: expected images [B, 3, {s}, {s}], got {tuple(images.shape)}")
        if input_ids.dim() != 2 or input_ids.shape[0] != images.shape[0] or not 1 <= input_ids.shape[1] <= L \
                or input_ids.is_floating_point():
            raise ValueError(f"CLIPModel: expected integer input_ids [{images.shape[0]}, <= {L}], got {input_ids.dtype} "
                             f"{tuple(input_ids.shape)}")

    def get_image_features(self, images: torch.Tensor) -> torch.Tensor:
        return self.visual_projection(self.vision_model(images))

    def get_text_features(self, input_ids: torch.Tensor) -> torch.Tensor:
        return self.text_projection(self.text_model(input_ids))

    def forward(self, images: torch.Tensor, input_ids: torch.Tensor):
        self._check(images, input_ids)
        return self.get_image_features(images), self.get_text_features(input_ids), self.logit_scale

    # ------------------------------------------------------------------------------------------
    _BLOCK_MAP = (("layer_norm1", "ln_1"), ("layer_norm2", "ln_2"), ("self_attn.out_proj", "self_attention.out_proj"),
                  ("mlp.fc1", "mlp.0"), ("mlp.fc2", "mlp.3"))

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.CLIPModel`` state dict.  Strict both ways: a key of ``hf`` this model does not read, or a
        parameter it leaves unwritten, raises ``RuntimeError``; q_proj | k_proj | v_proj become the rows of the fused
        ``in_proj_weight`` / ``in_proj_bias``."""
        own = self.state_dict()
        out, used = {}, set()

        def take(src):
            if src not in hf:
                raise RuntimeError(f"load_hf_state_dict: missing key {src!r}")
            used.add(src)
            return hf[src]

        def put(dst, src):
            out[dst] = take(src).to(own[dst].dtype).reshape(own[dst].shape)

        put("logit_scale", "logit_scale")
        put("visual_projection.weight", "visual_projection.weight")
        put("text_projection.weight", "text_projection.weight")
        for tower, ours, theirs, n in (("vision", "vision_model", "vision_model", self.config.vision.layers),
                                       ("text", "text_model", "text_model", self.config.text.layers)):
            if tower == "vision":
                put(f"{ours}.class_embedding", f"{theirs}.embeddings.class_embedding")
                put(f"{ours}.patch_embedding.weight", f"{theirs}.embeddings.patch_embedding.weight")
                put(f"{ours}.position_embedding.weight", f"{theirs}.embeddings.position_embedding.weight")
                norms = (("pre_layrnorm", "pre_layrnorm"), ("post_layernorm", "post_layernorm"))
            else:
                put(f"{ours}.token_embedding.weight", f"{theirs}.embeddings.token_embedding.weight")
                put(f"{ours}.position_embedding.weight", f"{theirs}.embeddings.position_embedding.weight")
                norms = (("final_layer_norm", "final_layer_norm"),)
            for wb in ("weight", "bias"):
                for dst, src in norms:
                    put(f"{ours}.{dst}.{wb}", f"{theirs}.{src}.{wb}")
                for i in range(n):
                    pre, hpre = f"{ours}.layers.{i}", f"{theirs}.encoder.layers.{i}"
                    for src, dst in self._BLOCK_MAP:
                        put(f"{pre}.{dst}.{wb}", f"{hpre}.{src}.{wb}")
                    fused = f"{pre}.self_attention.in_proj_{wb}"
                    out[fused] = torch.cat([take(f"{hpre}.self_attn.{p}_proj.{wb}") for p in "qkv"], 0).to(own[fused].dtype)
        unused = sorted(set(hf) - used)
        if unused:
            raise RuntimeError(f"load_hf_state_dict: unexpected keys {unused[:8]}{' ...' if len(unused) > 8 else ''}")
        self.load_state_dict(out, strict=True)


def clip_vit_b_32() -> CLIPModel:
    """CLIP-ViT-B/32: 32 x 32 patches, 50 tokens per image (151,277,313 parameters, as transformers' CLIPModel)."""
    return CLIPModel(CLIP_VIT_B_32)


def clip_vit_b_16() -> CLIPModel:
    """CLIP-ViT-B/16: 16 x 16 patches, 197 tokens per image (149,620,737 parameters, as transformers' CLIPModel)."""
    return CLIPModel(CLIP_VIT_B_16)
