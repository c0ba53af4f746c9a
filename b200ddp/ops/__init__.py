from .functional import attention, attention_reference, causal_attention, causal_attention_reference, document_bounds, packed_attention, packed_attention_reference, linear, stem_conv, stem_conv_supported, conv2d_tc, conv_tc_supported, conv_tc_wanted, mse_loss, cross_entropy, layer_norm, rms_norm, rotary, rotary_cos_sin, swiglu
from .modules import Linear, Conv2dTC, PointwiseConv2d, Conv3x3, StemConv7x7, LayerNorm, RMSNorm, MSELoss, CrossEntropyLoss
from .batchnorm import FusedBatchNormAct2d, MaxPool3x3s2

__all__ = ["attention", "attention_reference", "causal_attention", "causal_attention_reference", "document_bounds", "packed_attention", "packed_attention_reference", "linear", "conv2d_tc", "conv_tc_supported", "conv_tc_wanted", "Conv2dTC", "PointwiseConv2d", "Conv3x3", "StemConv7x7", "stem_conv", "stem_conv_supported", "mse_loss", "cross_entropy", "layer_norm", "rms_norm", "rotary", "rotary_cos_sin", "swiglu", "Linear",
           "LayerNorm", "RMSNorm", "MSELoss", "CrossEntropyLoss", "FusedBatchNormAct2d", "MaxPool3x3s2"]
