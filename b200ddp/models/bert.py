"""BERT-base encoder + MLM head for the "BERT-base DDP bf16, seq 512" config.
Every linear is a ``b200ddp.ops.Linear`` (wgmma GEMM with bias / bias+GELU epilogues), every
LayerNorm the hand-written kernel, the loss the fused cross-entropy; attention uses torch's SDPA
(library flash attention - not a named hot op).  109.5 M encoder parameters as in the stock model
(199 tensors in the stock naming; 151 here because Q / K / V are one stored parameter) when built with ``with_mlm_head=False``."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    intermediate: int = 3072
    max_position: int = 512
    type_vocab: int = 2
    eps: float = 1e-12
    dropout: float = 0.0
    pad_vocab_to: int = 1          # MLM head pads to 64 so logits rows keep the 16-byte pitch TMA needs

    @property
    def padded_vocab(self) -> int:
        m = max(1, self.pad_vocab_to)
        return (self.vocab_size + m - 1) // m * m


class BertEmbeddings(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.word_embeddings = nn.Embedding(c.padded_vocab, c.hidden)
        self.position_embeddings = nn.Embedding(c.max_position, c.hidden)
        self.token_type_embeddings = nn.Embedding(c.type_vocab, c.hidden)
        self.LayerNorm = LayerNorm(c.hidden, eps=c.eps)
        self.dropout = nn.Dropout(c.dropout)

    def forward(self, input_ids, token_type_ids=None):
        B, S = input_ids.shape
        pos = torch.arange(S, device=input_ids.device)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        x = self.word_embeddings(input_ids) + self.position_embeddings(pos)[None] + self.token_type_embeddings(token_type_ids)
        return self.dropout(self.LayerNorm(x))


class BertLayer(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.heads = c.heads
        # Q, K and V projections are ONE stored [3*hidden, hidden] parameter (rows: query, key, value): forward, dgrad and
        # wgrad are one wgmma launch each and nothing is concatenated per step.  ``load_hf_state_dict`` fuses the stock
        # model's three tensors; ``split_qkv_state_dict`` gives them back.
        self.qkv = Linear(c.hidden, 3 * c.hidden)
        self.attn_out = Linear(c.hidden, c.hidden)
        self.attn_norm = LayerNorm(c.hidden, eps=c.eps)
        self.ffn_in = Linear(c.hidden, c.intermediate, activation="gelu")
        self.ffn_out = Linear(c.intermediate, c.hidden)
        self.ffn_norm = LayerNorm(c.hidden, eps=c.eps)
        self.dropout = nn.Dropout(c.dropout)

    def forward(self, x, attn_mask=None):
        B, S, H = x.shape
        hd = H // self.heads

        def split(t):
            return t.view(B, S, self.heads, hd).transpose(1, 2)

        qkv = self.qkv(x)
        q, k, v = (split(t) for t in qkv.split(H, dim=-1))
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask)
        a = a.transpose(1, 2).reshape(B, S, H)
        x = self.attn_norm(x + self.dropout(self.attn_out(a)))
        return self.ffn_norm(x + self.dropout(self.ffn_out(self.ffn_in(x))))


class BertModel(nn.Module):
    def __init__(self, config: BertConfig | None = None, with_pooler: bool = True):
        super().__init__()
        c = self.config = config or BertConfig()
        self.embeddings = BertEmbeddings(c)
        self.encoder = nn.ModuleList([BertLayer(c) for _ in range(c.layers)])
        self.pooler = Linear(c.hidden, c.hidden) if with_pooler else None
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if getattr(m, "bias", None) is not None:
                nn.init.zeros_(m.bias)

    def forward(self, input_ids, token_type_ids=None, attn_mask=None):
        x = self.embeddings(input_ids, token_type_ids)
        for layer in self.encoder:
            x = layer(x, attn_mask)
        return x


class BertForMaskedLM(nn.Module):
    """Encoder + tied-embedding MLM head; forward returns logits [B, S, vocab]."""

    def __init__(self, config: BertConfig | None = None):
        super().__init__()
        config = config or BertConfig(pad_vocab_to=64)
        self.bert = BertModel(config, with_pooler=False)
        c = self.bert.config
        self.transform = Linear(c.hidden, c.hidden, activation="gelu")
        self.transform_norm = LayerNorm(c.hidden, eps=c.eps)
        self.decoder_bias = nn.Parameter(torch.zeros(c.padded_vocab))

    def forward(self, input_ids, token_type_ids=None, attn_mask=None):
        from ..ops import linear
        h = self.transform_norm(self.transform(self.bert(input_ids, token_type_ids, attn_mask)))
        return linear(h, self.bert.embeddings.word_embeddings.weight, self.decoder_bias)


    # ---- interchange with the stock (Hugging Face) parameter naming ---------------------------------------
    _LAYER_MAP = (("attention.output.dense", "attn_out"), ("attention.output.LayerNorm", "attn_norm"),
                  ("intermediate.dense", "ffn_in"), ("output.dense", "ffn_out"), ("output.LayerNorm", "ffn_norm"))

    def load_hf_state_dict(self, hf: dict) -> None:
        """Load a ``transformers.BertForMaskedLM`` state dict (the model the stock arm of ``bench.py`` trains), so a
        checkpoint of the stock model continues on this one.  Vocabulary rows beyond the checkpoint's (padding up
        to a multiple of ``pad_vocab_to``) are zero and their logits get a -inf-like bias so they never win."""
        c = self.bert.config
        own = self.state_dict()
        out = {}

        def put(dst, src):
            t = hf[src]
            if own[dst].shape != t.shape:                         # padded vocabulary
                full = torch.zeros_like(own[dst])
                if dst == "decoder_bias":
                    full.fill_(-1e4)
                full[:t.shape[0]] = t
                t = full
            out[dst] = t.to(own[dst].dtype)

        for n in ("word_embeddings", "position_embeddings", "token_type_embeddings"):
            put(f"bert.embeddings.{n}.weight", f"bert.embeddings.{n}.weight")
        for wb in ("weight", "bias"):
            put(f"bert.embeddings.LayerNorm.{wb}", f"bert.embeddings.LayerNorm.{wb}")
            for i in range(c.layers):
                for src, dst in self._LAYER_MAP:
                    put(f"bert.encoder.{i}.{dst}.{wb}", f"bert.encoder.layer.{i}.{src}.{wb}")
                # the stock model's separate query / key / value tensors become the rows of the fused projection
                out[f"bert.encoder.{i}.qkv.{wb}"] = torch.cat(
                    [hf[f"bert.encoder.layer.{i}.attention.self.{n}.{wb}"] for n in ("query", "key", "value")], dim=0).to(own[f"bert.encoder.{i}.qkv.{wb}"].dtype)
            put(f"transform.{wb}", f"cls.predictions.transform.dense.{wb}")
            put(f"transform_norm.{wb}", f"cls.predictions.transform.LayerNorm.{wb}")
        put("decoder_bias", "cls.predictions.bias")
        self.load_state_dict(out, strict=True)


def split_qkv_state_dict(state: dict) -> dict:
    """State dict with every fused ``qkv`` projection split back into ``query`` / ``key`` / ``value`` entries (the stock naming)."""
    out = {}
    for k, v in state.items():
        if ".qkv." in k:
            for n, part in zip(("query", "key", "value"), v.chunk(3, dim=0)):
                out[k.replace(".qkv.", f".{n}.")] = part.clone()
        else:
            out[k] = v
    return out


def bert_base(with_mlm_head: bool = True) -> nn.Module:
    return BertForMaskedLM() if with_mlm_head else BertModel()
