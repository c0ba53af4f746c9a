"""Model registry: the reference hard-codes ``FooModel()`` (``ddp.py:311``); ``--model`` selects here."""
from .foo import FooModel, BranchyFooModel
from .resnet import ResNet, resnet50, resnet152
from .bert import BertConfig, BertModel, BertForMaskedLM, bert_base
from .gpt import GPTConfig, GPTModel, GPTLMHeadModel, gpt2
from .llama import LlamaConfig, LlamaModel, LlamaForCausalLM, smollm_135m, qwen2_5_1_5b

MODEL_REGISTRY = {
    "foo": FooModel,
    "resnet50": resnet50,
    "resnet152": resnet152,
    "bert-base": bert_base,
    "gpt2": gpt2,
    "smollm-135m": smollm_135m,
    "qwen2.5-1.5b": qwen2_5_1_5b,
}


def build_model(name: str, **kwargs):
    try:
        return MODEL_REGISTRY[name](**kwargs)
    except KeyError:
        raise ValueError(f"unknown model {name!r}; choose from {sorted(MODEL_REGISTRY)}") from None


__all__ = ["FooModel", "BranchyFooModel", "ResNet", "resnet50", "resnet152", "BertConfig", "BertModel",
           "BertForMaskedLM", "bert_base", "GPTConfig", "GPTModel", "GPTLMHeadModel", "gpt2", "LlamaConfig", "LlamaModel", "LlamaForCausalLM", "smollm_135m", "qwen2_5_1_5b", "MODEL_REGISTRY", "build_model"]
