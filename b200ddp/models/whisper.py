"""Whisper speech recognition (whisper-tiny, -base, -small) for training on waveform / transcript pairs, as ``transformers``'
``WhisperForConditionalGeneration`` defines it: a two-convolution stem (width 3, the second with stride 2, each followed by
erf GELU) over 80-bin log-mel features, the frozen sinusoid positions of the encoder, pre-LN blocks on both sides with a final
``layer_norm`` each, learned decoder positions, ``k_proj`` without a bias in every attention, and an LM head tied to
``embed_tokens``.  No dropout, no embedding scale.

``forward(input_features, labels)`` takes features [B, 80, F] (``ops.log_mel_spectrogram`` of 30-second clips: F = 3000)
and transcript labels [B, Sq] right-padded with -100.  On CUDA the stem gathers its im2col rows natively (``ops.mel_patches``,
``ops.frame_patches``) and multiplies them on the wgmma ``linear``; the encoder's F / 2 rows per clip are padded to a multiple
of 128 (``ops.encoder_rows``: 1536 for 3000 frames) and attend as one document on ``ops.packed_attention``, the padding rows
attending and attended by nothing.  The decoder runs on ``ops.causal_attention`` with its lengths taken from the labels' -100
padding, and across on ``ops.cross_attention`` / ``ops.cross_bounds``.  On the CPU and in fp32 the stem is ``F.conv1d`` and
attention the dense-mask references.

q / k / v of self-attention are one fused projection, and cross-attention's k / v another; their bias is ``q_bias | 0 |
v_bias`` built at every call, so the k part stays exactly zero and untrained.  The vocabulary is padded (51865 -> 51904); the
padded rows get a -1e4 logit bias through the GEMM epilogue.  ``load_hf_state_dict`` reads a
``transformers.WhisperForConditionalGeneration`` state dict."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import (LayerNorm, Linear, LinearCrossEntropyLoss, causal_attention, cross_attention, cross_bounds, document_bounds, encoder_rows,
                   frame_patches, linear, mel_patches, packed_attention)
from .bart import shift_documents_right


@dataclass
class WhisperConfig:
    vocab_size: int = 51865
    max_position: int = 448            # decoder (target) positions
    max_source_positions: int = 1500   # encoder rows per clip: the stem halves num_mel_bins' 2 x 1500 frames
    num_mel_bins: int = 80
    hidden: int = 384
    encoder_layers: int = 4
    decoder_layers: int = 4
    heads: int = 6
    intermediate: int = 1536
    eps: float = 1e-5
    pad_vocab_to: int = 64             # LM head rows padded so logits rows keep the 16-byte pitch TMA needs (51865 -> 51904)
    decoder_start_token_id: int = 50257   # <|startoftranscript|>
    fill_token_id: int = 50256         # transformers' pad_token_id: the decoder input where the labels hold -100
    pad_token_id: int | None = None    # recorded only: the labels' -100 padding gives the decoder lengths
    bos_token_id: int | None = None    # recorded only: a row holds one clip and its transcript
    fused_lm_loss: bool = False        # forward returns the decoder's final hidden states; ``lm_head_loss`` applies the head

    @property
    def padded_vocab(self) -> int:
        m = max(1, self.pad_vocab_to)
        return (self.vocab_size + m - 1) // m * m

    @property
    def frames(self) -> int:
        """Mel frames per clip the encoder takes (3000 for 30 seconds)."""
        return 2 * self.max_source_positions


def sinusoids(length: int, channels: int, max_timescale: float = 10000.0) -> torch.Tensor:
    """transformers' ``sinusoids``: [length, channels] = sin | cos of position x geometric timescales."""
    inc = math.log(max_timescale) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2))
    t = torch.arange(length).view(-1, 1) * inv.view(1, -1)
    return torch.cat([t.sin(), t.cos()], dim=1)


class KFreeProjection(nn.Module):
    """A fused projection whose rows are q | k | v (``parts="qkv"``) or k | v (``parts="kv"``), with no bias on k: the bias
    is ``q_bias | 0 | v_bias`` (or ``0 | v_bias``), built at every call."""

    def __init__(self, hidden: int, parts: str):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(len(parts) * hidden, hidden))
        self.q_bias = nn.Parameter(torch.zeros(hidden)) if "q" in parts else None
        self.v_bias = nn.Parameter(torch.zeros(hidden))

    def forward(self, x):
        zero = torch.zeros_like(self.v_bias)
        parts = [zero, self.v_bias] if self.q_bias is None else [self.q_bias, zero, self.v_bias]
        return linear(x, self.weight, torch.cat(parts))


class WhisperSelfAttention(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.heads = c.heads
        self.qkv = KFreeProjection(c.hidden, "qkv")
        self.out_proj = Linear(c.hidden, c.hidden)


class WhisperCrossAttention(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.heads = c.heads
        self.q_proj = Linear(c.hidden, c.hidden)
        self.kv = KFreeProjection(c.hidden, "kv")
        self.out_proj = Linear(c.hidden, c.hidden)


class WhisperEncoderLayer(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.self_attn = WhisperSelfAttention(c)
        self.self_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.fc1 = Linear(c.hidden, c.intermediate, activation="gelu")
        self.fc2 = Linear(c.intermediate, c.hidden)
        self.final_layer_norm = LayerNorm(c.hidden, eps=c.eps)

    def forward(self, x, bounds):
        a = self.self_attn
        x = x + a.out_proj(packed_attention(a.qkv(self.self_attn_layer_norm(x)), bounds, a.heads))
        return x + self.fc2(self.fc1(self.final_layer_norm(x)))


class WhisperDecoderLayer(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.self_attn = WhisperSelfAttention(c)
        self.self_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.encoder_attn = WhisperCrossAttention(c)
        self.encoder_attn_layer_norm = LayerNorm(c.hidden, eps=c.eps)
        self.fc1 = Linear(c.hidden, c.intermediate, activation="gelu")
        self.fc2 = Linear(c.intermediate, c.hidden)
        self.final_layer_norm = LayerNorm(c.hidden, eps=c.eps)

    def forward(self, x, enc, bounds, q_bounds, kv_bounds):
        a = self.self_attn
        x = x + a.out_proj(causal_attention(a.qkv(self.self_attn_layer_norm(x)), bounds, a.heads))
        e = self.encoder_attn
        q = e.q_proj(self.encoder_attn_layer_norm(x))
        x = x + e.out_proj(cross_attention(q, e.kv(enc), q_bounds, kv_bounds, e.heads))
        return x + self.fc2(self.fc1(self.final_layer_norm(x)))


class WhisperEncoder(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.conv1 = nn.Conv1d(c.num_mel_bins, c.hidden, kernel_size=3, padding=1)
        self.conv2 = nn.Conv1d(c.hidden, c.hidden, kernel_size=3, stride=2, padding=1)
        self.embed_positions = nn.Embedding(c.max_source_positions, c.hidden)
        self.embed_positions.weight.requires_grad_(False)        # frozen sinusoids: optimizers and DDP skip it
        self.layers = nn.ModuleList([WhisperEncoderLayer(c) for _ in range(c.encoder_layers)])
        self.layer_norm = LayerNorm(c.hidden, eps=c.eps)

    def stem(self, features):
        """The convolution stem plus positions: [B, encoder_rows(F), d], rows >= F / 2 padding (finite, never attended)."""
        B, _, T = features.shape
        S, L, d = encoder_rows(T), T // 2, self.conv1.out_channels
        if features.is_cuda:
            w1 = self.conv1.weight.permute(0, 2, 1).reshape(d, -1)
            w2 = self.conv2.weight.permute(0, 2, 1).reshape(d, -1)
            h1 = linear(mel_patches(features), w1, self.conv1.bias, activation="gelu")
            y = linear(frame_patches(h1, T, S), w2, self.conv2.bias, activation="gelu").view(B, S, d)
        else:
            h = F.gelu(self.conv1(features))
            y = F.pad(F.gelu(self.conv2(h)).transpose(1, 2), (0, 0, 0, S - L))
        return y + F.pad(self.embed_positions.weight[:L], (0, 0, 0, S - L))

    def forward(self, features):
        """(encoder output [B, S, d], bounds int32 [B, S, 2]: one document [0, F / 2) per clip, padding rows empty)."""
        B, T = features.shape[0], features.shape[2]
        x = self.stem(features)
        S, L = x.shape[1], T // 2
        row = torch.arange(S, device=x.device)
        end = torch.where(row < L, L, 0)
        bounds = torch.stack([torch.zeros_like(end), end], -1).to(torch.int32).expand(B, S, 2).contiguous()
        for layer in self.layers:
            x = layer(x, bounds)
        return self.layer_norm(x), bounds


class WhisperDecoder(nn.Module):
    def __init__(self, c: WhisperConfig):
        super().__init__()
        self.embed_tokens = nn.Embedding(c.padded_vocab, c.hidden)
        self.embed_positions = nn.Embedding(c.max_position, c.hidden)
        self.layers = nn.ModuleList([WhisperDecoderLayer(c) for _ in range(c.decoder_layers)])
        self.layer_norm = LayerNorm(c.hidden, eps=c.eps)


class WhisperModel(nn.Module):
    def __init__(self, config: WhisperConfig | None = None):
        super().__init__()
        c = self.config = config or WhisperConfig()
        self.encoder = WhisperEncoder(c)
        self.decoder = WhisperDecoder(c)
        self.apply(self._init)
        with torch.no_grad():
            self.encoder.embed_positions.weight.copy_(sinusoids(c.max_source_positions, c.hidden))
            self.decoder.embed_tokens.weight[c.fill_token_id].zero_()      # transformers' padding_idx row

    @staticmethod
    def _init(m):
        if isinstance(m, (Linear, nn.Conv1d, nn.Embedding, KFreeProjection)):
            nn.init.normal_(m.weight, std=0.02)
        for name in ("bias", "q_bias", "v_bias"):
            if isinstance(getattr(m, name, None), nn.Parameter) and not isinstance(m, LayerNorm):
                nn.init.zeros_(getattr(m, name))

    def forward(self, input_features, labels):
        c = self.config
        if input_features.dim() != 3 or input_features.shape[1] != c.num_mel_bins or input_features.shape[2] != c.frames:
            raise ValueError(f"WhisperModel: input_features must be [B, {c.num_mel_bins}, {c.frames}], got {tuple(input_features.shape)}")
        if labels.shape[1] > c.max_position:
            raise ValueError(f"WhisperModel: transcript length {labels.shape[1]} exceeds max_position {c.max_position}")
        enc, enc_bounds = self.encoder(input_features)
        dec_ids, _, dec_pos = shift_documents_right(labels, c.decoder_start_token_id, None, None, c.fill_token_id)
        dec_bounds, _ = document_bounds(labels, None, -100)                  # length = the labels' non -100 count
        q_bounds, kv_bounds = cross_bounds(enc_bounds, dec_bounds)
        d = self.decoder
        y = d.embed_tokens(dec_ids) + d.embed_positions(dec_pos)
        for layer in d.layers:
            y = layer(y, enc, dec_bounds, q_bounds, kv_bounds)
        return d.layer_norm(y)


class WhisperForConditionalGeneration(nn.Module):
    """Encoder-decoder + LM head tied to ``embed_tokens``; ``forward(input_features, labels)`` returns logits [B, Sq, padded
    vocab] (or, with ``WhisperConfig.fused_lm_loss``, the decoder's final hidden states for ``lm_head_loss()``)."""

    def __init__(self, config: WhisperConfig | None = None):
        super().__init__()
        self.model = WhisperModel(config)
        c = self.model.config
        pad = torch.zeros(c.padded_vocab)
        pad[c.vocab_size:] = -1e4
        self.register_buffer("vocab_bias", pad, persistent=False)

    @property
    def config(self) -> WhisperConfig:
        return self.model.config

    def logits_bias(self) -> torch.Tensor:
        """The padded-vocabulary rows' -1e4 in the head's dtype: the bias its GEMM epilogue adds."""
        return self.vocab_bias.to(self.model.decoder.embed_tokens.weight.dtype)

    def forward(self, input_features, labels):
        h = self.model(input_features, labels)
        if self.config.fused_lm_loss:
            return h
        return linear(h, self.model.decoder.embed_tokens.weight, self.logits_bias().to(h.dtype))

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s hidden states with ``fused_lm_loss``: the tied head and its bias, read from this model
        at every call."""
        return LinearCrossEntropyLoss(lambda: (self.model.decoder.embed_tokens.weight, self.logits_bias()), ignore_index)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.WhisperForConditionalGeneration`` state dict strictly: q / k / v fused into ``qkv``,
        cross-attention k / v into ``kv``, the k biases absent; vocabulary rows beyond the checkpoint's are zero."""
        c = self.config
        own = self.state_dict()
        out = {}
        used = {"proj_out.weight"}                                            # tied to embed_tokens

        def get(k):
            used.add(k)
            return hf[k]

        def put(dst, t):
            if own[dst].shape != t.shape:                         # padded vocabulary: the checkpoint's entries, then zeros
                full = torch.zeros_like(own[dst])
                full[tuple(slice(0, n) for n in t.shape)] = t
                t = full
            out[dst] = t.to(own[dst].dtype).contiguous()

        def same(key):
            put(key, get(key))

        def norm(key):
            for wb in ("weight", "bias"):
                same(f"{key}.{wb}")

        e, d = "model.encoder", "model.decoder"
        for k in ("conv1", "conv2"):
            norm(f"{e}.{k}")
        same(f"{e}.embed_positions.weight")
        same(f"{d}.embed_tokens.weight")
        same(f"{d}.embed_positions.weight")
        norm(f"{e}.layer_norm")
        norm(f"{d}.layer_norm")
        for side, n in ((e, c.encoder_layers), (d, c.decoder_layers)):
            for i in range(n):
                p = f"{side}.layers.{i}"
                s = f"{p}.self_attn"
                put(f"{s}.qkv.weight", torch.cat([get(f"{s}.{x}_proj.weight") for x in "qkv"]))
                put(f"{s}.qkv.q_bias", get(f"{s}.q_proj.bias"))
                put(f"{s}.qkv.v_bias", get(f"{s}.v_proj.bias"))
                norm(f"{s}.out_proj")
                for name in ("self_attn_layer_norm", "fc1", "fc2", "final_layer_norm"):
                    norm(f"{p}.{name}")
                if side == d:
                    x = f"{p}.encoder_attn"
                    norm(f"{x}.q_proj")
                    put(f"{x}.kv.weight", torch.cat([get(f"{x}.{t}_proj.weight") for t in "kv"]))
                    put(f"{x}.kv.v_bias", get(f"{x}.v_proj.bias"))
                    norm(f"{x}.out_proj")
                    norm(f"{p}.encoder_attn_layer_norm")
        unknown = set(hf) - used
        if unknown:
            raise KeyError(f"load_hf_state_dict: unexpected keys {sorted(unknown)[:8]}")
        self.load_state_dict(out, strict=True)


WHISPER_TINY = WhisperConfig()
WHISPER_BASE = WhisperConfig(hidden=512, encoder_layers=6, decoder_layers=6, heads=8, intermediate=2048)
WHISPER_SMALL = WhisperConfig(hidden=768, encoder_layers=12, decoder_layers=12, heads=12, intermediate=3072)


def _build(preset: WhisperConfig, pad_token_id, bos_token_id, fused_lm_loss) -> WhisperForConditionalGeneration:
    return WhisperForConditionalGeneration(replace(preset, pad_token_id=pad_token_id, bos_token_id=bos_token_id, fused_lm_loss=fused_lm_loss))


def whisper_tiny(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """whisper-tiny (4 + 4 layers, d 384, 6 heads).  ``pad_token_id`` and ``bos_token_id`` are recorded only: the decoder
    lengths come from the labels' -100 padding and a row holds one clip.  ``fused_lm_loss=True``: forward returns hidden
    states and ``lm_head_loss()`` computes the loss without the logits."""
    return _build(WHISPER_TINY, pad_token_id, bos_token_id, fused_lm_loss)


def whisper_base(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """whisper-base (6 + 6 layers, d 512, 8 heads); the arguments as ``whisper_tiny``'s."""
    return _build(WHISPER_BASE, pad_token_id, bos_token_id, fused_lm_loss)


def whisper_small(pad_token_id: int | None = None, bos_token_id: int | None = None, fused_lm_loss: bool = False) -> nn.Module:
    """whisper-small (12 + 12 layers, d 768, 12 heads); the arguments as ``whisper_tiny``'s."""
    return _build(WHISPER_SMALL, pad_token_id, bos_token_id, fused_lm_loss)
