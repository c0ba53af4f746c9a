"""ModernBERT masked-language-model encoder (Answer.AI / LightOn, 2024); the defaults are ModernBERT-base (hidden 768, 22
layers, 12 heads of dim 64, GeGLU intermediate 1152, vocabulary 50368, 8192 positions, 149,655,232 parameters).
Pre-norm encoder blocks: bias-free LayerNorm (none before layer 0's attention) -> fused Wqkv (q | k | v) -> rotary ->
bidirectional attention -> Wo -> LayerNorm -> Wi (input | gate) -> GeGLU -> Wo.  Every third layer, starting at layer 0,
is global (rope theta 160000); the others are local (rope theta 10000): each token sees the tokens within
``local_attention // 2`` positions of it.  Both run on the native document-bounds kernels (``ops.packed_attention``),
the local layers with ``ops.window_bounds``, so their kernels visit only the tiles near the diagonal.  Fixed-length,
right-padded (``pad_token_id``) and packed rows (documents starting with ``cls_token_id``, positions restarting in each)
take the same path.  No linear has a bias; the MLM head is dense -> GELU -> LayerNorm, and the decoder is tied to the
token embedding with a trained bias.  Module and parameter names are Hugging Face's (``transformers.ModernBertForMaskedLM``)."""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from ..ops import LayerNorm, Linear, LinearCrossEntropyLoss, document_bounds, geglu, linear, packed_attention, rotary, rotary_cos_sin, window_bounds


@dataclass
class ModernBertConfig:
    vocab_size: int = 50368
    hidden: int = 768
    layers: int = 22
    heads: int = 12
    intermediate: int = 1152
    max_position: int = 8192
    eps: float = 1e-5
    local_attention: int = 128       # a local layer's token sees the tokens within local_attention // 2 positions
    global_every: int = 3            # layer i is global iff i % global_every == 0
    global_rope_theta: float = 160000.0
    local_rope_theta: float = 10000.0
    fp8: bool = False                # block linears (Wqkv, attn.Wo, mlp.Wi, mlp.Wo) on FP8 tensor cores; same parameters
    pad_token_id: int | None = None  # right-padded input: length = non-pad count per row
    cls_token_id: int | None = None  # packed input: a document starts at each such id (and at 0), attention stays inside it
    sparse_prediction: bool = False  # forward returns the head's output; ``lm_head_loss`` decodes the labelled rows only

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads


class ModernBertEmbeddings(nn.Module):
    def __init__(self, c: ModernBertConfig):
        super().__init__()
        self.tok_embeddings = nn.Embedding(c.vocab_size, c.hidden)
        self.norm = LayerNorm(c.hidden, eps=c.eps, bias=False)

    def forward(self, input_ids):
        return self.norm(self.tok_embeddings(input_ids))


class ModernBertAttention(nn.Module):
    def __init__(self, c: ModernBertConfig):
        super().__init__()
        self.heads = c.heads
        self.Wqkv = Linear(c.hidden, 3 * c.hidden, bias=False, fp8=c.fp8)     # q | k | v, the layout attention reads
        self.Wo = Linear(c.hidden, c.hidden, bias=False, fp8=c.fp8)

    def forward(self, x, bounds, position_ids, cos_sin):
        qkv = rotary(self.Wqkv(x), position_ids, cos_sin, self.heads, self.heads)
        return self.Wo(packed_attention(qkv, bounds, self.heads))


class ModernBertMLP(nn.Module):
    def __init__(self, c: ModernBertConfig):
        super().__init__()
        self.Wi = Linear(c.hidden, 2 * c.intermediate, bias=False, fp8=c.fp8)   # input | gate
        self.Wo = Linear(c.intermediate, c.hidden, bias=False, fp8=c.fp8)

    def forward(self, x):
        return self.Wo(geglu(self.Wi(x)))


class ModernBertEncoderLayer(nn.Module):
    def __init__(self, c: ModernBertConfig, index: int):
        super().__init__()
        self.is_global = index % c.global_every == 0
        if index > 0:                                  # layer 0 reads the embedding norm's output directly
            self.attn_norm = LayerNorm(c.hidden, eps=c.eps, bias=False)
        self.attn = ModernBertAttention(c)
        self.mlp_norm = LayerNorm(c.hidden, eps=c.eps, bias=False)
        self.mlp = ModernBertMLP(c)

    def forward(self, x, bounds, position_ids, cos_sin):
        h = self.attn_norm(x) if hasattr(self, "attn_norm") else x
        x = x + self.attn(h, bounds, position_ids, cos_sin)
        return x + self.mlp(self.mlp_norm(x))


class ModernBertModel(nn.Module):
    def __init__(self, config: ModernBertConfig | None = None):
        super().__init__()
        c = self.config = config or ModernBertConfig()
        if c.hidden % c.heads or c.head_dim % 2:
            raise ValueError(f"ModernBertConfig: heads must divide hidden into an even head dim, got hidden={c.hidden}, heads={c.heads}")
        if c.local_attention < 0 or c.global_every < 1:
            raise ValueError(f"ModernBertConfig: needs local_attention >= 0 and global_every >= 1, got {c.local_attention}, "
                             f"{c.global_every}")
        self.embeddings = ModernBertEmbeddings(c)
        self.layers = nn.ModuleList([ModernBertEncoderLayer(c, i) for i in range(c.layers)])
        self.final_norm = LayerNorm(c.hidden, eps=c.eps, bias=False)
        self.register_buffer("global_cos_sin", rotary_cos_sin(c.max_position, c.head_dim, c.global_rope_theta), persistent=False)
        self.register_buffer("local_cos_sin", rotary_cos_sin(c.max_position, c.head_dim, c.local_rope_theta), persistent=False)

    def _apply(self, fn, recurse=True):
        # the rotary tables stay fp32 whatever dtype the parameters are cast to
        tables = self.global_cos_sin, self.local_cos_sin
        out = super()._apply(fn, recurse)
        self.global_cos_sin = tables[0].to(device=self.global_cos_sin.device, dtype=torch.float32)
        self.local_cos_sin = tables[1].to(device=self.local_cos_sin.device, dtype=torch.float32)
        return out

    def forward(self, input_ids):
        B, S = input_ids.shape
        c = self.config
        if S > c.max_position:
            raise ValueError(f"ModernBertModel: sequence length {S} exceeds max_position {c.max_position}")
        # documents, their local windows and per-document positions, once per call on the device (no host synchronisation)
        bounds, position_ids = document_bounds(input_ids, c.cls_token_id, c.pad_token_id)
        local = window_bounds(bounds, c.local_attention // 2)
        position_ids = position_ids.to(torch.int32)
        x = self.embeddings(input_ids)
        for layer in self.layers:
            if layer.is_global:
                x = layer(x, bounds, position_ids, self.global_cos_sin)
            else:
                x = layer(x, local, position_ids, self.local_cos_sin)
        return self.final_norm(x)


class ModernBertPredictionHead(nn.Module):
    def __init__(self, c: ModernBertConfig):
        super().__init__()
        self.dense = Linear(c.hidden, c.hidden, bias=False, activation="gelu")
        self.norm = LayerNorm(c.hidden, eps=c.eps, bias=False)

    def forward(self, x):
        return self.norm(self.dense(x))


class ModernBertForMaskedLM(nn.Module):
    """Encoder + MLM head; forward returns logits [B, S, vocab].  The decoder's weight is ``tok_embeddings.weight``, so
    ``state_dict()`` holds Hugging Face's keys without ``decoder.weight``.  With ``ModernBertConfig.sparse_prediction``
    (Hugging Face's name) forward returns the head's output [B, S, hidden] and ``lm_head_loss()`` is the criterion that
    decodes only the rows that carry a label (``ops.linear_cross_entropy(sparse=True)``)."""

    def __init__(self, config: ModernBertConfig | None = None):
        super().__init__()
        self.model = ModernBertModel(config)
        c = self.model.config
        self.head = ModernBertPredictionHead(c)
        self.decoder = nn.Module()                     # only the bias: the weight is tied to the token embedding
        self.decoder.bias = nn.Parameter(torch.zeros(c.vocab_size))
        self._init_weights()

    @property
    def config(self) -> ModernBertConfig:
        return self.model.config

    @torch.no_grad()
    def _init_weights(self) -> None:
        """Hugging Face's scheme: normal cut at +-2 sigma, sigma 0.02 for the embedding, Wqkv and Wi and
        0.02 / sqrt(2 layers) for attn.Wo, mlp.Wo and head.dense; LayerNorm weights 1, decoder bias 0."""
        def trunc(w, std):
            nn.init.trunc_normal_(w, std=std, a=-2 * std, b=2 * std)
        out = 0.02 / math.sqrt(2.0 * self.config.layers)
        trunc(self.model.embeddings.tok_embeddings.weight, 0.02)
        for layer in self.model.layers:
            trunc(layer.attn.Wqkv.weight, 0.02)
            trunc(layer.attn.Wo.weight, out)
            trunc(layer.mlp.Wi.weight, 0.02)
            trunc(layer.mlp.Wo.weight, out)
        trunc(self.head.dense.weight, out)

    def forward(self, input_ids):
        h = self.head(self.model(input_ids))
        if self.config.sparse_prediction:
            return h
        return linear(h, self.model.embeddings.tok_embeddings.weight, self.decoder.bias)

    def lm_head_loss(self, ignore_index: int = -100) -> LinearCrossEntropyLoss:
        """Criterion over ``forward``'s head output with ``sparse_prediction``: the tied decoder and its trained bias, read
        from this model at every call, on the labelled rows only."""
        return LinearCrossEntropyLoss(lambda: (self.model.embeddings.tok_embeddings.weight, self.decoder.bias), ignore_index, sparse=True)

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.ModernBertForMaskedLM`` state dict, strictly: the names are the same (``Wqkv`` is fused
        there too); a ``decoder.weight`` must equal ``tok_embeddings.weight`` (the tie) and is dropped."""
        hf = dict(hf)
        dec = hf.pop("decoder.weight", None)
        emb = hf.get("model.embeddings.tok_embeddings.weight")
        if dec is not None and (emb is None or not torch.equal(dec, emb)):
            raise ValueError("ModernBertForMaskedLM: decoder.weight differs from model.embeddings.tok_embeddings.weight; "
                             "this model ties them")
        own = self.state_dict()
        self.load_state_dict({k: v.to(own[k].dtype).contiguous() if k in own else v for k, v in hf.items()}, strict=True)


MODERNBERT_BASE = ModernBertConfig()
MODERNBERT_LARGE = ModernBertConfig(hidden=1024, layers=28, heads=16, intermediate=2624)


def modernbert_base(fp8: bool = False, pad_token_id: int | None = None, cls_token_id: int | None = None,
                    sparse_prediction: bool = False) -> nn.Module:
    """ModernBERT-base with its MLM head (8192 positions); ``fp8=True`` puts the 88 block linears on FP8 tensor cores
    (embedding, head and decoder stay bf16).  ``pad_token_id`` takes right-padded input; ``cls_token_id`` takes packed
    documents, each starting with that id (attention stays inside a document and position ids restart in each).
    ``sparse_prediction=True``: forward returns the head's output and ``lm_head_loss()`` decodes the labelled rows only;
    the state dict is the same."""
    return ModernBertForMaskedLM(replace(MODERNBERT_BASE, fp8=fp8, pad_token_id=pad_token_id, cls_token_id=cls_token_id,
                                         sparse_prediction=sparse_prediction))


def modernbert_large(fp8: bool = False, pad_token_id: int | None = None, cls_token_id: int | None = None,
                     sparse_prediction: bool = False) -> nn.Module:
    """ModernBERT-large (hidden 1024, 28 layers, 16 heads, GeGLU intermediate 2624; 395,881,664 parameters) with its MLM
    head; ``fp8=True`` puts the 112 block linears on FP8 tensor cores.  The other arguments as for ``modernbert_base``."""
    return ModernBertForMaskedLM(replace(MODERNBERT_LARGE, fp8=fp8, pad_token_id=pad_token_id, cls_token_id=cls_token_id,
                                         sparse_prediction=sparse_prediction))
