"""BERT-base encoder + MLM head for the "BERT-base DDP bf16, seq 512" config.
Every linear is a ``b200ddp.ops.Linear`` (wgmma GEMM with bias / bias+GELU epilogues), every
LayerNorm the hand-written kernel, the loss the fused cross-entropy.  Attention on fixed-length rows uses torch's SDPA
(library flash attention); with ``BertConfig.pad_token_id`` set, right-padded rows run on the native key-padding
attention kernel (``ops.attention``), which reads Q / K / V straight out of the fused projection; with
``BertConfig.cls_token_id`` set as well, rows hold packed documents (each starting with that id) and run on the
document-boundary kernel (``ops.packed_attention``), with position ids restarting per document.  109.5 M encoder parameters as in the stock model
(199 tensors in the stock naming; 151 here because Q / K / V are one stored parameter) when built with ``with_mlm_head=False``."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import LayerNorm, Linear, attention, document_bounds, packed_attention


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
    fp8: bool = False              # encoder linears (qkv, attn_out, ffn_in, ffn_out) on FP8 tensor cores; same parameters
    pad_token_id: int | None = None  # right-padded input: lengths = non-pad count per row, padded keys hidden (ops.attention)
    cls_token_id: int | None = None  # packed input: a document starts at each such id (and at 0), attention stays inside it

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

    def forward(self, input_ids, token_type_ids=None, position_ids=None):
        B, S = input_ids.shape
        pos = self.position_embeddings(torch.arange(S, device=input_ids.device))[None] if position_ids is None \
            else self.position_embeddings(position_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        x = self.word_embeddings(input_ids) + pos + self.token_type_embeddings(token_type_ids)
        return self.dropout(self.LayerNorm(x))


class BertLayer(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.heads = c.heads
        # Q, K and V projections are ONE stored [3*hidden, hidden] parameter (rows: query, key, value): forward, dgrad and
        # wgrad are one wgmma launch each and nothing is concatenated per step.  ``load_hf_state_dict`` fuses the stock
        # model's three tensors; ``split_qkv_state_dict`` gives them back.
        self.qkv = Linear(c.hidden, 3 * c.hidden, fp8=c.fp8)
        self.attn_out = Linear(c.hidden, c.hidden, fp8=c.fp8)
        self.attn_norm = LayerNorm(c.hidden, eps=c.eps)
        self.ffn_in = Linear(c.hidden, c.intermediate, activation="gelu", fp8=c.fp8)
        self.ffn_out = Linear(c.intermediate, c.hidden, fp8=c.fp8)
        self.ffn_norm = LayerNorm(c.hidden, eps=c.eps)
        self.dropout = nn.Dropout(c.dropout)

    def forward(self, x, attn_mask=None, seq_lens=None, bounds=None):
        B, S, H = x.shape
        hd = H // self.heads

        def split(t):
            return t.view(B, S, self.heads, hd).transpose(1, 2)

        qkv = self.qkv(x)
        if bounds is not None:
            a = packed_attention(qkv, bounds, self.heads)  # [B, S, H], the layout attn_out reads
        elif seq_lens is not None:
            a = attention(qkv, seq_lens, self.heads)
        else:
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
        seq_lens = bounds = position_ids = None
        pad, cls = self.config.pad_token_id, self.config.cls_token_id
        if attn_mask is not None and (pad is not None or cls is not None):
            raise ValueError("BertModel: pass either attn_mask or a config with pad_token_id / cls_token_id, not both "
                             "(with those ids the mask comes from input_ids)")
        if cls is not None:
            # packed documents: boundaries and per-document positions, computed on the device (no host synchronisation)
            bounds, position_ids = document_bounds(input_ids, cls, pad)
        elif pad is not None:
            # right padding: the length is the non-pad count; computed on the device, so no host synchronisation
            seq_lens = (input_ids != pad).sum(1, dtype=torch.int32)
        x = self.embeddings(input_ids, token_type_ids, position_ids)
        for layer in self.encoder:
            x = layer(x, attn_mask, seq_lens, bounds)
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


def bert_base(with_mlm_head: bool = True, fp8: bool = False, pad_token_id: int | None = None,
              cls_token_id: int | None = None) -> nn.Module:
    """BERT-base; ``fp8=True`` puts the 48 encoder linears on FP8 tensor cores (embeddings, MLM transform and the tied
    decoder stay bf16).  ``pad_token_id`` takes right-padded input (padded keys are hidden from attention);
    ``cls_token_id`` takes packed documents, each starting with that id (attention stays inside a document and position
    ids restart in each).  The state dict is the same either way."""
    if with_mlm_head:
        return BertForMaskedLM(BertConfig(pad_vocab_to=64, fp8=fp8, pad_token_id=pad_token_id, cls_token_id=cls_token_id))
    return BertModel(BertConfig(fp8=fp8, pad_token_id=pad_token_id, cls_token_id=cls_token_id))
