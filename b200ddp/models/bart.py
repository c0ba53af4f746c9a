"""BART encoder-decoder (bart-base, bart-large) for sequence-to-sequence training, as ``transformers``'
``BartForConditionalGeneration`` defines it: post-LN blocks, ``layernorm_embedding`` on both sides, learned absolute
positions offset by 2, erf GELU, no embedding scale, token embeddings and LM head tied to ``shared``, and a
``final_logits_bias`` buffer.  No dropout.

Every linear is a ``b200ddp.ops.Linear`` and every LayerNorm the hand-written kernel.  Self-attention's q / k / v are one
fused ``qkv`` projection; cross-attention's query is its own ``q_proj`` and its key / value one fused ``cross_kv``
projection of the encoder output.  The encoder attends on ``ops.packed_attention``, the decoder on ``ops.causal_attention``
and across on ``ops.cross_attention``, all on ``document_bounds``: fixed-length, right-padded and packed rows take the same
path (the native kernels on CUDA in bf16, the dense-mask references on the CPU and in fp32).  In packed rows the k-th
target document attends to the k-th source document of its row (``ops.cross_bounds``) and positions restart in each.

``forward(input_ids, labels)`` derives the decoder input on the device: each target document shifted right by one, with
``decoder_start_token_id`` at its start and -100 replaced by the pad id (transformers' ``shift_tokens_right`` for one
document per row).  The vocabulary is padded to a multiple of 64 (50265 -> 50304); the padded rows get a -1e4 logit bias
through the GEMM epilogue together with ``final_logits_bias``.  ``load_hf_state_dict`` reads a
``transformers.BartForConditionalGeneration`` state dict."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import (LayerNorm, Linear, LinearCrossEntropyLoss, causal_attention, cross_attention, cross_bounds, document_bounds, linear,
                   packed_attention)

POSITION_OFFSET = 2                # transformers' BartLearnedPositionalEmbedding: position p reads row p + 2


def shift_documents_right(labels, start_id: int, pad_token_id, bos_token_id, default_fill: int):
    """(decoder input ids, decoder document bounds, decoder position ids) of an encoder-decoder from labels [B, Sq]
    (-100 = ignored): each target document shifted right by one with ``start_id`` at its start, -100 as the pad id
    (``default_fill`` when rows hold no padding).  Torch ops on the device, no host synchronisation."""
    fill = pad_token_id if pad_token_id is not None else default_fill
    target = labels.masked_fill(labels == -100, fill)
    bounds, position_ids = document_bounds(target, bos_token_id, pad_token_id)
    S = labels.shape[1]
    pos = torch.arange(S, device=labels.device)
    start = ((bounds[..., 0] == pos) & (bounds[..., 1] > pos)) | (pos == 0)
    shifted = torch.cat([torch.full_like(target[:, :1], fill), target[:, :-1]], 1)
    ids = torch.where(start, torch.full_like(target, start_id), shifted)
    return ids, bounds, (position_ids if bos_token_id is not None else pos.expand_as(labels))


@dataclass
class BartConfig:
    vocab_size: int = 50265
    max_position: int = 1024
    hidden: int = 768
    encoder_layers: int = 6
    decoder_layers: int = 6
    heads: int = 12
    intermediate: int = 3072
    eps: float = 1e-5
    pad_vocab_to: int = 64         # LM head rows padded so logits rows keep the 16-byte pitch TMA needs (50265 -> 50304)
    decoder_start_token_id: int = 2
    pad_token_id: int | None = None  # right-padded rows: length = non-pad count (sources) or non -100 count (labels)
    bos_token_id: int | None = None  # packed rows: a document starts at each such id (and at 0) on both sides
    fused_lm_loss: bool = False    # forward returns the decoder's final hidden states; ``lm_head_loss`` applies the head

    @property
    def padded_vocab(self) -> int:
        m = max(1, self.pad_vocab_to)
        return (self.vocab_size + m - 1) // m * m


class BartEncoderLayer(nn.Module):
    def __init__(self, c: BartConfig):
        super().__init__()
        self.heads = c.heads
        self.qkv = Linear(c.hidden, 3 * c.hidden)            # rows: q_proj | k_proj | v_proj
        self.out_proj = Linear(c.hidden, c.hidden)
        self.self_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.fc1 = Linear(c.hidden, c.intermediate, activation="gelu")
        self.fc2 = Linear(c.intermediate, c.hidden)
        self.final_layer_norm = LayerNorm(c.hidden, eps=c.eps)

    def forward(self, x, bounds):
        x = self.self_attn_layer_norm(x + self.out_proj(packed_attention(self.qkv(x), bounds, self.heads)))
        return self.final_layer_norm(x + self.fc2(self.fc1(x)))


class BartDecoderLayer(nn.Module):
    def __init__(self, c: BartConfig):
        super().__init__()
        self.heads = c.heads
        self.qkv = Linear(c.hidden, 3 * c.hidden)
        self.out_proj = Linear(c.hidden, c.hidden)
        self.self_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.q_proj = Linear(c.hidden, c.hidden)              # encoder_attn.q_proj
        self.cross_kv = Linear(c.hidden, 2 * c.hidden)        # rows: encoder_attn.k_proj | v_proj
        self.cross_out_proj = Linear(c.hidden, c.hidden)
        self.encoder_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.fc1 = Linear(c.hidden, c.intermediate, activation="gelu")
        self.fc2 = Linear(c.intermediate, c.hidden)
        self.final_layer_norm = LayerNorm(c.hidden, eps=c.eps)

    def forward(self, x, enc, bounds, q_bounds, kv_bounds):
        x = self.self_attn_layer_norm(x + self.out_proj(causal_attention(self.qkv(x), bounds, self.heads)))
        a = cross_attention(self.q_proj(x), self.cross_kv(enc), q_bounds, kv_bounds, self.heads)
        x = self.encoder_attn_layer_norm(x + self.cross_out_proj(a))
        return self.final_layer_norm(x + self.fc2(self.fc1(x)))


class BartStack(nn.Module):
    """One side's positions, ``layernorm_embedding`` and layers (the token embedding is the model's ``shared``)."""

    def __init__(self, c: BartConfig, layer, n: int):
        super().__init__()
        self.embed_positions = nn.Embedding(c.max_position + POSITION_OFFSET, c.hidden)
        self.layernorm_embedding = LayerNorm(c.hidden, eps=c.eps)
        self.layers = nn.ModuleList([layer(c) for _ in range(n)])

    def embed(self, tokens, position_ids):
        return self.layernorm_embedding(tokens + self.embed_positions(position_ids + POSITION_OFFSET))


class BartModel(nn.Module):
    def __init__(self, config: BartConfig | None = None):
        super().__init__()
        c = self.config = config or BartConfig()
        self.shared = nn.Embedding(c.padded_vocab, c.hidden)
        self.encoder = BartStack(c, BartEncoderLayer, c.encoder_layers)
        self.decoder = BartStack(c, BartDecoderLayer, c.decoder_layers)
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if getattr(m, "bias", None) is not None:
                nn.init.zeros_(m.bias)

    def decoder_inputs(self, labels):
        """(decoder input ids, decoder document bounds, decoder position ids) from labels [B, Sq]: ``shift_documents_right``
        with BART's ids (its own <pad>, 1, as the fill when rows hold no padding)."""
        c = self.config
        return shift_documents_right(labels, c.decoder_start_token_id, c.pad_token_id, c.bos_token_id, 1)

    def forward(self, input_ids, labels):
        c = self.config
        Sk, Sq = input_ids.shape[1], labels.shape[1]
        if max(Sk, Sq) > c.max_position:
            raise ValueError(f"BartModel: sequence length {max(Sk, Sq)} exceeds max_position {c.max_position}")
        enc_bounds, enc_pos = document_bounds(input_ids, c.bos_token_id, c.pad_token_id)
        if c.bos_token_id is None:
            enc_pos = torch.arange(Sk, device=input_ids.device).expand_as(input_ids)
        dec_ids, dec_bounds, dec_pos = self.decoder_inputs(labels)
        q_bounds, kv_bounds = cross_bounds(enc_bounds, dec_bounds)
        x = self.encoder.embed(self.shared(input_ids), enc_pos)
        for layer in self.encoder.layers:
            x = layer(x, enc_bounds)
        y = self.decoder.embed(self.shared(dec_ids), dec_pos)
        for layer in self.decoder.layers:
            y = layer(y, x, dec_bounds, q_bounds, kv_bounds)
        return y


class BartForConditionalGeneration(nn.Module):
    """Encoder-decoder + LM head tied to ``shared``; ``forward(input_ids, labels)`` returns logits [B, Sq, padded vocab]
    (or, with ``BartConfig.fused_lm_loss``, the decoder's final hidden states for ``lm_head_loss()``)."""

    def __init__(self, config: BartConfig | None = None):
        super().__init__()
        self.model = BartModel(config)
        c = self.model.config
        self.register_buffer("final_logits_bias", torch.zeros(1, c.padded_vocab))
        pad = torch.zeros(c.padded_vocab)
        pad[c.vocab_size:] = -1e4
        self.register_buffer("vocab_bias", pad, persistent=False)

    @property
    def config(self) -> BartConfig:
        return self.model.config

    def logits_bias(self) -> torch.Tensor:
        """final_logits_bias plus the padded-vocabulary rows' -1e4, in the head's dtype: the bias its GEMM epilogue adds."""
        return (self.final_logits_bias[0].float() + self.vocab_bias.float()).to(self.model.shared.weight.dtype)

    def forward(self, input_ids, labels):
        h = self.model(input_ids, labels)
        if self.config.fused_lm_loss:
            return h
        return linear(h, self.model.shared.weight, self.logits_bias().to(h.dtype))

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head and the combined bias, read from
        this model at every call."""
        return LinearCrossEntropyLoss(lambda: (self.model.shared.weight, self.logits_bias()), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.BartForConditionalGeneration`` state dict strictly: q / k / v fused into ``qkv``,
        cross-attention k / v into ``cross_kv``; vocabulary rows beyond the checkpoint's are zero."""
        c = self.config
        own = self.state_dict()
        out = {}
        used = {"model.encoder.embed_tokens.weight", "model.decoder.embed_tokens.weight", "lm_head.weight"}   # tied to shared

        def get(k):
            used.add(k)
            return hf[k]

        def put(dst, t):
            if own[dst].shape != t.shape:                         # padded vocabulary: the checkpoint's entries, then zeros
                full = torch.zeros_like(own[dst])
                full[tuple(slice(0, n) for n in t.shape)] = t
                t = full
            out[dst] = t.to(own[dst].dtype).contiguous()

        put("model.shared.weight", get("model.shared.weight"))
        put("final_logits_bias", get("final_logits_bias"))
        for side, n in (("encoder", c.encoder_layers), ("decoder", c.decoder_layers)):
            p = f"model.{side}"
            put(f"{p}.embed_positions.weight", get(f"{p}.embed_positions.weight"))
            for wb in ("weight", "bias"):
                put(f"{p}.layernorm_embedding.{wb}", get(f"{p}.layernorm_embedding.{wb}"))
            for i in range(n):
                s, d = f"{p}.layers.{i}", f"{p}.layers.{i}"
                for wb in ("weight", "bias"):
                    put(f"{d}.qkv.{wb}", torch.cat([get(f"{s}.self_attn.{x}_proj.{wb}") for x in "qkv"]))
                    put(f"{d}.out_proj.{wb}", get(f"{s}.self_attn.out_proj.{wb}"))
                    for name in ("self_attn_layer_norm", "fc1", "fc2", "final_layer_norm"):
                        put(f"{d}.{name}.{wb}", get(f"{s}.{name}.{wb}"))
                    if side == "decoder":
                        put(f"{d}.q_proj.{wb}", get(f"{s}.encoder_attn.q_proj.{wb}"))
                        put(f"{d}.cross_kv.{wb}", torch.cat([get(f"{s}.encoder_attn.{x}_proj.{wb}") for x in "kv"]))
                        put(f"{d}.cross_out_proj.{wb}", get(f"{s}.encoder_attn.out_proj.{wb}"))
                        put(f"{d}.encoder_attn_layer_norm.{wb}", get(f"{s}.encoder_attn_layer_norm.{wb}"))
        unknown = set(hf) - used
        if unknown:
            raise KeyError(f"load_hf_state_dict: unexpected keys {sorted(unknown)[:8]}")
        self.load_state_dict(out, strict=True)


BART_BASE = BartConfig()
BART_LARGE = BartConfig(hidden=1024, encoder_layers=12, decoder_layers=12, heads=16, intermediate=4096)


def _build(preset: BartConfig, pad_token_id, bos_token_id, fused_lm_loss) -> BartForConditionalGeneration:
    return BartForConditionalGeneration(replace(preset, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def bart_base(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """bart-base (6 + 6 layers, d 768, 12 heads).  ``pad_token_id`` takes right-padded rows (sources padded with it,
    labels with -100); ``bos_token_id`` packed rows whose documents start with that id on both sides.
    ``fused_lm_loss=True``: forward returns hidden states and ``lm_head_loss()`` computes the loss without the logits."""
    return _build(BART_BASE, pad_token_id, bos_token_id, fused_lm_loss)


def bart_large(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """bart-large (12 + 12 layers, d 1024, 16 heads); the arguments as ``bart_base``'s."""
    return _build(BART_LARGE, pad_token_id, bos_token_id, fused_lm_loss)
