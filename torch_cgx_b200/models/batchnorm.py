"""Training BatchNorm of the ResNet blocks, with the block ReLU fused, as native kernels both ways.

Eagerly ``relu_(bn(x))`` costs five passes over the activation in forward (ATen's statistics kernel
reads x, its transform reads x and writes y, ``relu_`` reads and writes y) and eight in backward
(``threshold_backward`` reads g and y and writes the masked gradient, the reduction reads it and x, the
element-wise kernel reads both and writes grad_input). The native kernels need three forward and five
backward: the backward recomputes the ReLU mask from x. Results are bit-identical to ATen's
channels_last kernels: output, saved mean and invstd, running stats, grad_input, grad_weight and
grad_bias (DESIGN §2.11).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import _C

_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _eager_runs_aten_cl(x: torch.Tensor) -> bool:
    """True when eager ``F.batch_norm`` would run ATen's channels_last kernels on ``x``: bf16 input
    never goes to cuDNN; fp32 and fp16 do whenever cuDNN is enabled. ATen also picks its contiguous
    kernels for an NCHW-contiguous x whose channel stride is not 1 (possible here only with C == 1)."""
    if x.is_contiguous() and x.stride(1) != 1:
        return False
    if x.dtype == torch.bfloat16:
        return True
    return not (torch.backends.cudnn.enabled and torch.backends.cudnn.is_available())


def native_ok(bn: nn.BatchNorm2d, x: torch.Tensor) -> bool:
    """The conditions under which the native forward computes what eager would. Eager training
    BatchNorm refuses a single value per channel, so that case stays eager too."""
    if not (bn.training and bn.affine and bn.track_running_stats and isinstance(bn.momentum, float)):
        return False
    if not (x.is_cuda and x.dim() == 4 and x.dtype in _DTYPES and 0 < x.numel() < 2**31
            and x.numel() // x.shape[1] >= 2
            and x.is_contiguous(memory_format=torch.channels_last) and _eager_runs_aten_cl(x)):
        return False
    return all(t.is_cuda and t.device == x.device and t.dtype == torch.float32 and t.is_contiguous()
               for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))


class BatchNormAct(torch.autograd.Function):
    """``y = relu_(bn(x))`` (or ``bn(x)``) in training mode; running stats of ``bn`` are updated."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn: nn.BatchNorm2d, relu: bool):
        y, mean, invstd = _C.batchnorm_cl_forward(x, weight, bias, bn.running_mean, bn.running_var,
                                                  bn.momentum, bn.eps, relu)
        ctx.relu, ctx.eps = relu, bn.eps
        # y is kept only for the eager fallback below; it is the next conv's saved input anyway
        ctx.save_for_backward(x, weight, bias, mean, invstd, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, bias, mean, invstd, y = ctx.saved_tensors
        if gy.dtype == x.dtype and gy.stride() == x.stride():
            gx, gw, gb = _C.batchnorm_cl_backward(gy, x, weight, bias, mean, invstd, ctx.relu)
        else:  # what autograd runs for the eager relu_(bn(x))
            if ctx.relu:
                gy = torch.ops.aten.threshold_backward(gy, y, 0)
            gx, gw, gb = torch.ops.aten.native_batch_norm_backward(
                gy, x, weight, None, None, mean, invstd, True, ctx.eps, [True, True, True])
        return gx, gw, gb, None, None


def batch_norm_act(bn: nn.BatchNorm2d, x: torch.Tensor, relu: bool) -> torch.Tensor:
    """``relu_(bn(x))`` when ``relu``, else ``bn(x)``. Runs the native kernels where eager would run
    ATen's channels_last kernels (see ``native_ok``), otherwise the eager modules (the only path on
    CPU). Both count ``bn.num_batches_tracked`` as ``nn.BatchNorm2d.forward`` does."""
    if not native_ok(bn, x):
        y = bn(x)
        return torch.relu_(y) if relu else y
    bn.num_batches_tracked.add_(1)
    return BatchNormAct.apply(x, bn.weight, bn.bias, bn, relu)
