"""Model registry: the reference hard-codes ``FooModel()`` (``ddp.py:311``); ``--model`` selects here."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Callable

from .foo import FooModel, BranchyFooModel
from .resnet import ResNet, resnet50, resnet152
from .bert import BERT_BASE, BertConfig, BertModel, BertForMaskedLM, bert_base
from .gpt import GPT2, GPTConfig, GPTModel, GPTLMHeadModel, gpt2
from .llama import (GRANITE_3_0_1B_A400M, QWEN2_5_1_5B, QWEN3_0_6B, SMOLLM_135M, LlamaConfig, LlamaModel, LlamaForCausalLM,
                    smollm_135m, qwen2_5_1_5b, qwen3_0_6b, granite_3_0_1b_a400m)
from .modernbert import (MODERNBERT_BASE, MODERNBERT_LARGE, ModernBertConfig, ModernBertModel, ModernBertForMaskedLM, modernbert_base,
                         modernbert_large)
from .vit import VIT_B_16, VIT_B_32, VIT_L_16, ViTConfig, VisionTransformer, vit_b_16, vit_b_32, vit_l_16
from .convnext import CONVNEXT_BASE, CONVNEXT_SMALL, CONVNEXT_TINY, ConvNeXt, ConvNeXtConfig, convnext_base, convnext_small, convnext_tiny
from .swin import (SWIN_B, SWIN_S, SWIN_T, SWIN_V2_B, SWIN_V2_S, SWIN_V2_T, SwinConfig, SwinTransformer, swin_b, swin_s, swin_t, swin_v2_b,
                   swin_v2_s, swin_v2_t)
from .clip import CLIP_VIT_B_16, CLIP_VIT_B_32, CLIPConfig, CLIPModel, clip_vit_b_16, clip_vit_b_32
from .bart import BART_BASE, BART_LARGE, BartConfig, BartForConditionalGeneration, bart_base, bart_large
from .t5 import T5_BASE, T5_SMALL, T5Config, T5ForConditionalGeneration, t5_base, t5_small
from .mamba import MAMBA_130M, MAMBA_370M, MambaConfig, MambaForCausalLM, mamba_130m, mamba_370m
from .mamba2 import MAMBA2_130M, MAMBA2_370M, Mamba2Config, Mamba2ForCausalLM, mamba2_130m, mamba2_370m
from .vit_mae import VIT_MAE_BASE, VIT_MAE_LARGE, ViTMAEConfig, ViTMAEForPreTraining, vit_mae_base, vit_mae_large
from .whisper import (WHISPER_BASE, WHISPER_SMALL, WHISPER_TINY, WhisperConfig, WhisperForConditionalGeneration, whisper_base, whisper_small,
                      whisper_tiny)


@dataclass(frozen=True)
class ModelEntry:
    """A registered model: its builder and what training needs to know about it without building it."""
    build: Callable[..., Any]
    kind: str                          # "foo", "image", "encoder" (BERT, ModernBERT) or "causal" (the language models)
    config: Any = None                 # token models: the preset config, whose vocab_size and max_position training reads
    start_id: int | None = None        # token models: the id each packed document starts with
    fp8: bool = False                  # build takes fp8=True (block linears on FP8 tensor cores)
    moe: bool = False                  # mixture of experts: build takes router_aux_loss_coef
    max_seq_len: int | None = None     # a training cap on --seq_len below config.max_position
    contrastive: bool = False          # image models trained on image-caption pairs with their own contrastive loss
                                       # (CLIP): forward(images, input_ids), the criterion ops.ClipLoss
    seq2seq: bool = False              # encoder-decoder trained on source / target pairs (BART, T5): forward(source_ids, labels),
                                       # kind "causal" (the decoder is a causal LM over the target)
    speech: bool = False               # an encoder-decoder trained on waveform / transcript pairs (Whisper): forward(features,
                                       # labels) on the log-mel features of int16 clips
    own_loss: bool = False             # image models whose forward returns their own loss (MAE pretraining): forward(images),
                                       # the criterion passes it through and the labels are ignored
    image_size: int = 224              # image models: the side of the square synthetic images they train on

    @property
    def token_model(self) -> bool:
        return self.kind in ("encoder", "causal")


MODEL_REGISTRY = {
    "foo": ModelEntry(FooModel, "foo"),
    "resnet50": ModelEntry(resnet50, "image"),
    "resnet152": ModelEntry(resnet152, "image"),
    "vit-b-16": ModelEntry(vit_b_16, "image"),
    "vit-b-32": ModelEntry(vit_b_32, "image"),
    "vit-l-16": ModelEntry(vit_l_16, "image"),
    "convnext-tiny": ModelEntry(convnext_tiny, "image"),
    "convnext-small": ModelEntry(convnext_small, "image"),
    "convnext-base": ModelEntry(convnext_base, "image"),
    "swin-t": ModelEntry(swin_t, "image"),
    "swin-s": ModelEntry(swin_s, "image"),
    "swin-b": ModelEntry(swin_b, "image"),
    # Swin V2's 8 x 8 windows tile every stage of a 256 x 256 image (224 leaves stage 2 28 wide)
    "swin-v2-t": ModelEntry(swin_v2_t, "image", image_size=256),
    "swin-v2-s": ModelEntry(swin_v2_s, "image", image_size=256),
    "swin-v2-b": ModelEntry(swin_v2_b, "image", image_size=256),
    "vit-mae-base": ModelEntry(vit_mae_base, "image", own_loss=True),
    "vit-mae-large": ModelEntry(vit_mae_large, "image", own_loss=True),
    "clip-vit-b-32": ModelEntry(clip_vit_b_32, "image", contrastive=True),
    "clip-vit-b-16": ModelEntry(clip_vit_b_16, "image", contrastive=True),
    "bert-base": ModelEntry(bert_base, "encoder", BERT_BASE, start_id=101, fp8=True),                 # [CLS]
    "modernbert-base": ModelEntry(modernbert_base, "encoder", MODERNBERT_BASE, start_id=50281, fp8=True),   # [CLS]
    "modernbert-large": ModelEntry(modernbert_large, "encoder", MODERNBERT_LARGE, start_id=50281, fp8=True),
    "gpt2": ModelEntry(gpt2, "causal", GPT2, start_id=50256, fp8=True),                               # <|endoftext|>
    "smollm-135m": ModelEntry(smollm_135m, "causal", SMOLLM_135M, start_id=1, fp8=True),              # <s>
    "qwen2.5-1.5b": ModelEntry(qwen2_5_1_5b, "causal", QWEN2_5_1_5B, start_id=151643, fp8=True),      # <|endoftext|>
    # Qwen3's native context is 32768 tokens; the position table's 40960 rows leave room to generate past it
    "qwen3-0.6b": ModelEntry(qwen3_0_6b, "causal", QWEN3_0_6B, start_id=151643, fp8=True, max_seq_len=32768),
    # Granite's own start id, <|end_of_text|> = 0, is the padding id here, so packed documents start with id 1 instead
    "granite-3.0-1b-a400m": ModelEntry(granite_3_0_1b_a400m, "causal", GRANITE_3_0_1B_A400M, start_id=1, moe=True),
    # BART's own <s> = 0 is the padding id here and </s> = 2 starts every decoder input, so packed documents start with
    # id 3 (<unk>), which the synthetic text never holds otherwise
    "bart-base": ModelEntry(bart_base, "causal", BART_BASE, start_id=3, seq2seq=True),
    "bart-large": ModelEntry(bart_large, "causal", BART_LARGE, start_id=3, seq2seq=True),
    # T5's pad and decoder start id is 0 and </s> is 1, so packed documents start with id 2 (<unk>), which the synthetic
    # text never holds otherwise
    "t5-small": ModelEntry(t5_small, "causal", T5_SMALL, start_id=2, seq2seq=True),
    "t5-base": ModelEntry(t5_base, "causal", T5_BASE, start_id=2, seq2seq=True),
    # Mamba's own start id, <|endoftext|> = 0, is the padding id here, so packed documents start with id 1 instead
    "mamba-130m": ModelEntry(mamba_130m, "causal", MAMBA_130M, start_id=1),
    "mamba-370m": ModelEntry(mamba_370m, "causal", MAMBA_370M, start_id=1),
    "mamba2-130m": ModelEntry(mamba2_130m, "causal", MAMBA2_130M, start_id=1),
    "mamba2-370m": ModelEntry(mamba2_370m, "causal", MAMBA2_370M, start_id=1),
    # <|startoftranscript|>; a row holds one clip and its transcript, so the id only starts each decoder input
    "whisper-tiny": ModelEntry(whisper_tiny, "causal", WHISPER_TINY, start_id=50257, seq2seq=True, speech=True),
    "whisper-base": ModelEntry(whisper_base, "causal", WHISPER_BASE, start_id=50257, seq2seq=True, speech=True),
    "whisper-small": ModelEntry(whisper_small, "causal", WHISPER_SMALL, start_id=50257, seq2seq=True, speech=True),
}


def model_entry(name: str) -> ModelEntry:
    try:
        return MODEL_REGISTRY[name]
    except KeyError:
        raise ValueError(f"unknown model {name!r}; choose from {sorted(MODEL_REGISTRY)}") from None


def build_model(name: str, **kwargs):
    return model_entry(name).build(**kwargs)


__all__ = ["FooModel", "BranchyFooModel", "ResNet", "resnet50", "resnet152", "BertConfig", "BertModel",
           "BertForMaskedLM", "bert_base", "GPTConfig", "GPTModel", "GPTLMHeadModel", "gpt2", "LlamaConfig", "LlamaModel", "LlamaForCausalLM", "smollm_135m", "qwen2_5_1_5b", "qwen3_0_6b", "granite_3_0_1b_a400m", "ModernBertConfig", "ModernBertModel", "ModernBertForMaskedLM", "modernbert_base", "modernbert_large", "ViTConfig", "VisionTransformer", "vit_b_16", "vit_b_32", "vit_l_16", "ViTMAEConfig", "ViTMAEForPreTraining", "vit_mae_base", "vit_mae_large", "ConvNeXtConfig", "ConvNeXt", "convnext_tiny", "convnext_small", "convnext_base", "SwinConfig", "SwinTransformer", "swin_t", "swin_s", "swin_b", "swin_v2_t", "swin_v2_s", "swin_v2_b", "CLIPConfig", "CLIPModel", "clip_vit_b_32", "clip_vit_b_16", "BartConfig", "BartForConditionalGeneration", "bart_base", "bart_large", "T5Config", "T5ForConditionalGeneration", "t5_small", "t5_base", "MambaConfig", "MambaForCausalLM", "mamba_130m", "mamba_370m", "Mamba2Config", "Mamba2ForCausalLM", "mamba2_130m", "mamba2_370m", "WhisperConfig", "WhisperForConditionalGeneration", "whisper_tiny", "whisper_base", "whisper_small", "ModelEntry", "MODEL_REGISTRY", "model_entry", "build_model"]
