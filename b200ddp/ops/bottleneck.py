"""ResNet Bottleneck block as ONE autograd node whose backward is written out by hand, so that work the autograd engine would
schedule as separate kernels rides in the convolution epilogues instead (``csrc/conv_wgmma.cu``):

forward    conv (+ BatchNorm statistics from the epilogue) -> BatchNorm apply (+ReLU, +shortcut): the activations are read
           once for normalisation, never for statistics.
backward   the data gradient of conv2 / conv3 also emits the partial sums S1 = sum dy*m, S2 = sum dy*m*xhat of the BatchNorm
           backward that consumes it (bn1 / bn2: no reduction pass over dy and x), and the data gradient of conv1 adds the
           shortcut gradient in its epilogue (no separate add kernel).

Reference hot path replaced: ``outputs = model(x)`` / ``loss.backward()`` (``the reference ddp.py:221,231``) with a ResNet
handed to ``train()``.  Used by ``models.resnet.Bottleneck`` for blocks whose convolutions all run on the native kernels
(stride 1, channels_last bf16 CUDA tensors); other blocks compose the per-layer ops."""
from __future__ import annotations

import torch

from .. import _ext
from . import functional as Fn


def _bn_args(bn):
    momentum = bn.momentum if bn.momentum is not None else 0.1
    return bn.running_mean, bn.running_var, bn.num_batches_tracked, bn.eps, momentum


class _BottleneckFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, g1, b1, w2, g2, b2, w3, g3, b3, wd, gd, bd, block):
        C = _ext.get()
        cl = Fn._cl
        x = cl(x)
        w1c, w2c, w3c = cl(w1), cl(w2), cl(w3)
        y1, p1 = C.conv_fprop(x, w1c, 1, 0, -1, 0, 0, True)
        a1, s1, m1 = C.bn_forward_partials(y1, None, g1, b1, *_bn_args(block.bn1), True, p1)
        y2, p2 = C.conv_fprop(a1, w2c, 1, 1, -1, 0, 0, True)
        a2, s2, m2 = C.bn_forward_partials(y2, None, g2, b2, *_bn_args(block.bn2), True, p2)
        y3, p3 = C.conv_fprop(a2, w3c, 1, 0, -1, 0, 0, True)
        has_ds = wd is not None
        if has_ds:
            wdc = cl(wd)
            yd, pd = C.conv_fprop(x, wdc, 1, 0, -1, 0, 0, True)
            idn, sd, _ = C.bn_forward_partials(yd, None, gd, bd, *_bn_args(block.downsample[1]), False, pd)
        else:
            wdc = yd = sd = None
            idn = x
        out, s3, m3 = C.bn_forward_partials(y3, idn, g3, b3, *_bn_args(block.bn3), True, p3)
        ctx.save_for_backward(x, w1c, w2c, w3c, wdc, y1, a1, y2, a2, y3, yd, s1, s2, s3, sd, m1, m2, m3, g1, g2, g3, gd)
        ctx.block = block
        ctx.has_ds = has_ds
        ctx.strides = (w1.stride(), w3.stride(), wd.stride() if has_ds else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        C = _ext.get()
        (x, w1, w2, w3, wd, y1, a1, y2, a2, y3, yd, s1, s2, s3, sd, m1, m2, m3, g1, g2, g3, gd) = ctx.saved_tensors
        blk = ctx.block
        dout = Fn._cl(dout)

        def wgrad(dy, inp, w, k, strides=None):
            n, cin, h, wdt = inp.shape
            if Fn._wgrad_native(cin, w.shape[0], k, n * h * wdt):
                dw = C.conv_wgrad(dy, inp, k, 1, (k - 1) // 2, 0, 0, 0)
            else:
                pad = (k - 1) // 2
                dw = torch.ops.aten.convolution_backward(dy, inp, w, None, [1, 1], [pad, pad], [1, 1], False, [0, 0], 1, [False, True, False])[1]
            if strides is not None and tuple(dw.stride()) != tuple(strides):
                dw = dw.as_strided(dw.shape, strides)     # 1x1 filters: same memory order, match the parameter's strides
            return dw

        # bn3 (+shortcut, +ReLU): its output gradient arrives from outside the block -> regular reduction + apply
        ws = blk.bn3._workspace(y3)
        dy3, dres, dp3 = C.bn_backward(dout, y3, m3, g3, s3, True, True, ws[2], ws[3])
        dw3 = wgrad(dy3, a2, w3, 1, ctx.strides[1])
        da2, part2 = C.conv_dgrad(dy3, w3, 1, 0, -1, 0, 0, 0, None, y2, m2, s2)           # + S1/S2 of bn2's backward
        dy2, _, dp2 = C.bn_backward_partials(da2, y2, m2, g2, s2, True, False, part2)
        dw2 = wgrad(dy2, a1, w2, 3)
        da1, part1 = C.conv_dgrad(dy2, w2, 1, 1, -1, 0, 0, 0, None, y1, m1, s1)           # + S1/S2 of bn1's backward
        dy1, _, dp1 = C.bn_backward_partials(da1, y1, m1, g1, s1, True, False, part1)
        dw1 = wgrad(dy1, x, w1, 1, ctx.strides[0])
        dwd = dgd = dbd = None
        if ctx.has_ds:
            wsd = blk.downsample[1]._workspace(yd)
            dyd, _, dpd = C.bn_backward(dres, yd, None, gd, sd, False, False, wsd[2], wsd[3])
            dwd = wgrad(dyd, x, wd, 1, ctx.strides[2])
            shortcut = C.conv_dgrad(dyd, wd, 1, 0, -1, 0, 0, 0)[0]
            dgd, dbd = dpd[0], dpd[1]
        else:
            shortcut = dres
        dx = C.conv_dgrad(dy1, w1, 1, 0, -1, 0, 0, 0, shortcut)[0] if ctx.needs_input_grad[0] else None   # + shortcut gradient in the epilogue
        return (dx, dw1, dp1[0], dp1[1], dw2, dp2[0], dp2[1], dw3, dp3[0], dp3[1], dwd, dgd, dbd, None)


def bottleneck_native_ok(block, x: torch.Tensor) -> bool:
    """Every convolution of the block on the native kernels, training-mode BatchNorm on the fused kernels."""
    if not (x.is_cuda and block.training and torch.is_grad_enabled() and x.dim() == 4 and x.dtype == torch.bfloat16):
        return False
    convs = [block.conv1, block.conv2, block.conv3] + ([block.downsample[0]] if block.downsample is not None else [])
    bns = [block.bn1, block.bn2, block.bn3] + ([block.downsample[1]] if block.downsample is not None else [])
    xin = x
    for conv in convs:
        if not (conv.stride[0] == 1 and conv.weight.dtype == torch.bfloat16 and conv.in_channels % 64 == 0 and conv.out_channels % 64 == 0):
            return False
    if not Fn.conv_tc_supported(xin, block.conv1.weight, 1, 0):
        return False
    for bn in bns:
        if not (bn.track_running_stats and bn.weight is not None and bn.weight.dtype == torch.float32):
            return False
    return True


def bottleneck_forward(block, x: torch.Tensor) -> torch.Tensor:
    ds = block.downsample
    return _BottleneckFn.apply(x, block.conv1.weight, block.bn1.weight, block.bn1.bias, block.conv2.weight, block.bn2.weight, block.bn2.bias,
                               block.conv3.weight, block.bn3.weight, block.bn3.bias,
                               ds[0].weight if ds is not None else None, ds[1].weight if ds is not None else None,
                               ds[1].bias if ds is not None else None, block)
