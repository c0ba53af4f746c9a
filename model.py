"""User-replaceable workload, as in the reference layout (reference ``model.py:8-16``: ``FooModel``).  ``FooModel`` is the reference's toy MLP built
from b200ddp's native linear layers; the registry adds the models the benchmark runs."""
from b200ddp.models import (FooModel, BranchyFooModel, resnet50, resnet152, bert_base, build_model,  # noqa: F401
                            MODEL_REGISTRY)
