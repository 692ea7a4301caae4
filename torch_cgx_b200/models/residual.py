"""The residual join of the ResNet blocks, ``relu(a + b)``, as one native kernel each way.

Eagerly the join costs five passes over the block output in forward (``add`` reads two tensors
and writes one, ``relu_`` reads and writes one) and, for a block output that feeds the next block
through two consumers (conv1 and the identity or downsample path), six in backward: the autograd
engine adds the two incoming gradients, then ``threshold_backward`` masks the sum. The native
kernels need three passes forward and four backward and give bit-identical results.

To keep the engine's accumulation out of the backward, ``ResidualReLU`` returns ``y`` twice: the
tensor and a view of it, sharing storage. The next block feeds the first to conv1 and the second
to its identity or downsample path, so each arrives with its own gradient and the backward adds
them inside the kernel.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _C

_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _dense(t: torch.Tensor) -> bool:
    return t.is_contiguous() or (t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last))


def fusable(*ts: Optional[torch.Tensor]) -> bool:
    """True when the native kernels accept these operands (``None`` entries are skipped): CUDA
    tensors on one device with one dtype among fp32 / fp16 / bf16, identical sizes and strides, and
    dense (contiguous or channels_last)."""
    ts = [t for t in ts if t is not None]
    r = ts[0]
    if not (r.is_cuda and r.dtype in _DTYPES and _dense(r)):
        return False
    return all(t.is_cuda and t.device == r.device and t.dtype == r.dtype and t.shape == r.shape
               and t.stride() == r.stride() for t in ts[1:])


class ResidualReLU(torch.autograd.Function):
    """``(y, y_alias) = relu(a + b)`` with ``y_alias`` a view of ``y``; backward returns the masked
    sum of both outputs' gradients for ``a`` and for ``b``."""

    @staticmethod
    def forward(ctx, a: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        y = _C.residual_relu_forward(a, b)
        ctx.save_for_backward(y)
        ctx.set_materialize_grads(False)  # an unused output's gradient stays None instead of zeros
        return y, y.view_as(y)

    @staticmethod
    def backward(ctx, ga: Optional[torch.Tensor], gb: Optional[torch.Tensor]):
        (y,) = ctx.saved_tensors
        if ga is None:
            ga, gb = gb, None
        if ga is None:
            return None, None
        if fusable(y, ga, gb):
            g = _C.residual_relu_backward(y, ga, gb)
        else:  # e.g. a gradient with other strides than y: what autograd does for the eager join
            g = torch.ops.aten.threshold_backward(ga if gb is None else ga + gb, y, 0)
        return g, g


def residual_relu(a: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``relu(a + b)`` returned as a pair for the next block's two consumers. Runs the native kernels
    when they accept ``a`` and ``b`` (see ``fusable``), otherwise the eager ``relu_(a + b)`` (the
    only path on CPU) and returns that tensor twice."""
    if fusable(a, b):
        return ResidualReLU.apply(a, b)
    y = torch.relu_(a + b)
    return y, y
