"""Every ``MODEL_REGISTRY`` entry agrees with the model its builder makes (built on the meta device), and ``--model``
offers exactly the registered models."""
import pytest
import torch

from b200ddp.data import SyntheticTokens
from b200ddp.models import MODEL_REGISTRY


def _config(model):
    return next(m.config for m in model.modules() if hasattr(m, "config"))


@pytest.mark.parametrize("name", sorted(MODEL_REGISTRY))
def test_entry_agrees_with_its_model(name):
    entry = MODEL_REGISTRY[name]
    assert entry.kind in ("foo", "image", "encoder", "causal")
    if not entry.token_model:
        with torch.device("meta"):
            entry.build()
        assert entry.config is None and entry.start_id is None and not entry.fp8 and not entry.moe
        return
    doc_attr = "cls_token_id" if entry.kind == "encoder" else "bos_token_id"
    vocab = entry.config.vocab_size
    assert entry.start_id != SyntheticTokens.PAD_ID and 0 < entry.start_id < vocab
    assert entry.max_seq_len is None or entry.max_seq_len <= entry.config.max_position
    with torch.device("meta"):
        plain = entry.build()
        packed = entry.build(pad_token_id=SyntheticTokens.PAD_ID, **{doc_attr: entry.start_id})
    c = _config(plain)
    assert hasattr(c, doc_attr) and getattr(c, doc_attr) is None
    assert (c.vocab_size, c.max_position) == (vocab, entry.config.max_position)
    assert getattr(_config(packed), doc_attr) == entry.start_id and _config(packed).pad_token_id == SyntheticTokens.PAD_ID
    assert not any(getattr(m, "fp8", False) is True for m in plain.modules())
    if entry.fp8:
        with torch.device("meta"):
            fp8 = entry.build(fp8=True)
        assert any(getattr(m, "fp8", False) is True for m in fp8.modules())
    else:
        with pytest.raises(TypeError):
            entry.build(fp8=True)
    assert (getattr(c, "num_experts", 0) > 0) == entry.moe


def test_model_choices_are_the_registry():
    from b200ddp.engine import cli
    action = next(a for a in cli.build_parser()._actions if a.dest == "model")
    assert sorted(action.choices) == sorted(MODEL_REGISTRY)


def test_bert_seq_len_beyond_its_positions_is_rejected_at_setup(tmp_path):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "bert-base",
                                          "--no_cuda", "--seq_len", "1024"])
    with pytest.raises(ValueError, match="512"):
        cli.setup(args)
