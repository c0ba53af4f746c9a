from .adamw import FusedAdamW, weight_decay_groups
from .schedule import LinearWarmupDecay, get_linear_schedule_with_warmup, warmup_decay_factor
from .sgd import FusedSGD

__all__ = ["LinearWarmupDecay", "get_linear_schedule_with_warmup", "warmup_decay_factor", "FusedSGD", "FusedAdamW",
           "weight_decay_groups"]
