"""b200ddp - a Hopper-native (sm_90a) distributed-data-parallel training template.

Same capabilities and launch shape as howardlau1999/pytorch-ddp-template (``ddp.py`` + ``model.py`` +
``dataset.py``, torchrun-spawned) with the delegated native layers rebuilt for 8xH100: a DDP wrapper
whose C++ reducer launches fused allreduce kernels over NVSwitch peer memory, a peer-memory init
broadcast, wgmma/TMA GEMMs, fused LayerNorm / loss / clip+SGD kernels, CUDA-graph steps.
"""
__version__ = "0.1.0"

from . import utils  # noqa: F401
from .parallel import DistributedDataParallel, DataParallel, ShardedSampler  # noqa: F401
from .optim import FusedSGD, get_linear_schedule_with_warmup  # noqa: F401
from .models import FooModel, build_model  # noqa: F401
