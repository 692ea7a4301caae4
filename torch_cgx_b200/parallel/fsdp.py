"""FSDP2 (``fully_shard``) gradient reduce-scatter through the compressed kernel.

FSDP2 takes a custom reduce-scatter per module (``FSDPModule.set_custom_reduce_scatter``), so no
FSDP code is patched::

    model = fully_shard(model)                       # after fully_shard on the sub-modules
    cgx.set_cgx_reduce_scatter(model, bits=8)        # every FSDPModule of the model
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.distributed as dist
from torch.distributed.fsdp._fully_shard._fsdp_api import ReduceScatter

from .functional import _reduce_scatter


class CGXReduceScatter(ReduceScatter):
    """FSDP2 reduce-scatter comm: SUM and AVG go through the compressed kernel (with at most
    ``CGX_OVERLAP_LANES`` CTAs, since FSDP overlaps it with backward); any other op, such as
    premul-sum, goes to ``dist.reduce_scatter_tensor`` unchanged."""

    def __init__(self, bits: int = 4, bucket_size: int = 512, stochastic: bool = False):
        self.bits = int(bits)
        self.bucket_size = int(bucket_size)
        self.stochastic = bool(stochastic)

    def allocate(self, size: Sequence[int], *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        return torch.empty(*size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group: dist.ProcessGroup,
                 op, async_op: bool = False):
        if op == dist.ReduceOp.SUM or op == dist.ReduceOp.AVG:
            return _reduce_scatter(output_tensor, input_tensor, bits=self.bits, bucket_size=self.bucket_size,
                                   average=op == dist.ReduceOp.AVG, group=group, async_op=async_op,
                                   stochastic=self.stochastic, seed=None, layers=None, skip_incomplete=False,
                                   overlapped=True)
        return dist.reduce_scatter_tensor(output_tensor, input_tensor, op=op, group=group, async_op=async_op)


def set_cgx_reduce_scatter(model: torch.nn.Module, bits: int = 4, bucket_size: int = 512,
                           stochastic: bool = False) -> CGXReduceScatter:
    """Install one :class:`CGXReduceScatter` on every ``FSDPModule`` of ``model``; returns it."""
    from torch.distributed.fsdp import FSDPModule

    comm = CGXReduceScatter(bits, bucket_size, stochastic)
    for m in model.modules():
        if isinstance(m, FSDPModule):
            m.set_custom_reduce_scatter(comm)
    return comm
