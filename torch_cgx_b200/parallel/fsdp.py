"""FSDP2 (``fully_shard``) gradient reduce-scatter and parameter all-gather through the compressed
kernels.

FSDP2 takes a custom reduce-scatter and all-gather per module (``FSDPModule.set_custom_reduce_scatter``
/ ``set_custom_all_gather``), so no FSDP code is patched::

    model = fully_shard(model)                       # after fully_shard on the sub-modules
    cgx.set_cgx_reduce_scatter(model, bits=8)        # every FSDPModule of the model
    cgx.set_cgx_all_gather(model, bits=8)            # one comm per FSDPModule, per-parameter table

``bits`` may also be an FP8 wire format: ``"e4m3"`` for the parameter all-gather and ``"e5m2"`` for
the gradient reduce-scatter are the usual choice, and ``"e4m3_pow2"`` / ``"e5m2_pow2"`` give the
same codes with power-of-two scales. The reduce-scatter also takes ``"e5m2_sr"`` / ``"e4m3_sr"``,
rounded stochastically; the all-gather does not.

Both work over any number of nodes: across nodes they run in two stages, the semantics of
``reduce_scatter_tensor`` and ``all_gather_into_tensor`` (functional.py).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
from torch.distributed.fsdp._fully_shard._fsdp_api import AllGather, ReduceScatter

from .functional import A2aBits, _all_gather, _reduce_scatter

RAW_BITS = 32


Layer = Tuple[int, int, int, int]


def _table(layers: Optional[Sequence[Layer]]) -> Optional[List[Layer]]:
    return None if layers is None else [tuple(int(v) for v in l) for l in layers]


def _bits(bits: A2aBits, adaptive) -> A2aBits:
    """a comm's ``bits``: an int, or an FP8 format name, which adaptive widths do not take"""
    if isinstance(bits, str):
        if adaptive is not None:
            raise ValueError(f"cgx: adaptive widths are max-min widths; bits={bits!r} cannot be adapted")
        return bits
    return int(bits)


def _check_gather_bits(bits: A2aBits) -> None:
    """ValueError for a stochastic FP8 format: the FSDP2 all-gather rounds to nearest, so that the
    backward re-gather sees the weights the forward saw"""
    if isinstance(bits, str) and bits.endswith("_sr"):
        raise ValueError(f"cgx: the FSDP2 all-gather rounds to nearest, so that the backward re-gather sees "
                         f"the forward's weights; bits={bits!r} rounds stochastically")


def _table_bits(bits: A2aBits) -> int:
    """the width of a table entry for ``bits``: an FP8 format travels in 8-bit records"""
    return 8 if isinstance(bits, str) else int(bits)


class CGXReduceScatter(ReduceScatter):
    """FSDP2 reduce-scatter comm: SUM and AVG go through the compressed kernel (with at most
    ``CGX_OVERLAP_LANES`` CTAs, since FSDP overlaps it with backward); any other op, such as
    premul-sum, goes to ``dist.reduce_scatter_tensor`` unchanged. ``layers`` optionally gives one
    shard's table as ``(elem_off, numel, bits, bucket_size)`` tuples (None = one layer of ``bits`` /
    ``bucket_size`` per shard). ``adaptive`` is an :class:`~torch_cgx_b200.AdaptiveFSDPState` that
    rewrites ``layers``; ``set_cgx_adaptive`` sets it. ``bits`` may be an FP8 format, ``"e5m2"`` or
    ``"e4m3"`` (``layers`` then of bits 8 or 32, no ``stochastic``, no ``adaptive``), or ``"e5m2_sr"``
    / ``"e4m3_sr"``, which round stochastically whatever ``stochastic`` says."""

    def __init__(self, bits: A2aBits = 4, bucket_size: int = 512, stochastic: bool = False,
                 layers: Optional[Sequence[Layer]] = None, name: str = "", adaptive=None):
        self.bits = _bits(bits, adaptive)
        self.bucket_size = int(bucket_size)
        self.stochastic = bool(stochastic)
        self.layers = _table(layers)
        self.name = name
        self.numel = None if self.layers is None else sum(l[1] for l in self.layers)
        self.adaptive = adaptive

    def allocate(self, size: Sequence[int], *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        return torch.empty(*size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group: dist.ProcessGroup,
                 op, async_op: bool = False):
        if op == dist.ReduceOp.SUM or op == dist.ReduceOp.AVG:
            if self.numel is not None and output_tensor.numel() != self.numel:
                raise RuntimeError(
                    f"cgx reduce-scatter of module '{self.name}': the shard has {output_tensor.numel()} elements "
                    f"but its table covers {self.numel} (parameters changed after the comm was installed?)")
            if self.adaptive is not None:
                self.adaptive.maybe_estimate(self, input_tensor, group, average=op == dist.ReduceOp.AVG)
            return _reduce_scatter(output_tensor, input_tensor, bits=self.bits, bucket_size=self.bucket_size,
                                   average=op == dist.ReduceOp.AVG, group=group, async_op=async_op,
                                   stochastic=self.stochastic, seed=None, layers=self.layers, skip_incomplete=False,
                                   overlapped=True)
        return dist.reduce_scatter_tensor(output_tensor, input_tensor, op=op, group=group, async_op=async_op)


def set_cgx_reduce_scatter(model: torch.nn.Module, bits: A2aBits = 4, bucket_size: int = 512,
                           stochastic: bool = False) -> CGXReduceScatter:
    """Install one :class:`CGXReduceScatter` on every ``FSDPModule`` of ``model``; returns it."""
    from torch.distributed.fsdp import FSDPModule

    comm = CGXReduceScatter(bits, bucket_size, stochastic)
    for m in model.modules():
        if isinstance(m, FSDPModule):
            m.set_custom_reduce_scatter(comm)
    return comm


def fsdp_shard_table(params: Sequence[Tuple[Sequence[int], int]], bits: A2aBits = 4,
                     bucket_size: int = 512) -> List[Layer]:
    """The all-gather shard table of one FSDP parameter group.

    ``params`` holds one ``(orig_size, padded_shard_numel)`` pair per parameter, in FSDP's
    all-gather order. Each parameter is one layer of ``padded_shard_numel`` elements, so no bucket
    spans two parameters; parameters of at most one dimension (biases, norm weights) travel
    uncompressed (bits 32): they are small, and their values sit far from those of the weights.
    With an FP8 ``bits`` the other parameters get 8, the width of its records."""
    table, off = [], 0
    for orig_size, n in params:
        n = int(n)
        if n == 0:
            continue
        table.append((off, n, RAW_BITS if len(orig_size) <= 1 else _table_bits(bits), int(bucket_size)))
        off += n
    return table


class CGXAllGather(AllGather):
    """FSDP2 all-gather comm: the parameters go through the compressed kernel, quantized to nearest
    with the shard table ``layers`` (one shard's ``(elem_off, numel, bits, bucket_size)`` tuples;
    None = one layer of ``bits`` / ``bucket_size``), with at most ``CGX_OVERLAP_LANES`` CTAs since
    FSDP prefetches during compute. There is no stochastic rounding: the backward re-gather must
    see the weights the forward saw. A ``uint8`` buffer (FSDP2's all-gather of mixed-dtype inputs)
    goes to ``dist.all_gather_into_tensor`` unchanged. ``adaptive`` is an
    :class:`~torch_cgx_b200.AdaptiveFSDPState` that rewrites ``layers``; ``set_cgx_adaptive`` sets it.
    ``bits`` may be an FP8 format, usually ``"e4m3"`` (``layers`` then of bits 8 or 32, no ``adaptive``),
    but not a stochastic one (``"e4m3_sr"`` / ``"e5m2_sr"``: ValueError), for the same reason."""

    def __init__(self, bits: A2aBits = 4, bucket_size: int = 512, layers: Optional[Sequence[Layer]] = None,
                 name: str = "", adaptive=None):
        _check_gather_bits(bits)
        self.bits = _bits(bits, adaptive)
        self.bucket_size = int(bucket_size)
        self.layers = _table(layers)
        self.name = name
        self.numel = None if self.layers is None else sum(l[1] for l in self.layers)
        self.adaptive = adaptive

    def allocate(self, size: Sequence[int], *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        return torch.empty(*size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group: dist.ProcessGroup,
                 async_op: bool = False):
        if input_tensor.dtype == torch.uint8:
            return dist.all_gather_into_tensor(output_tensor, input_tensor, group=group, async_op=async_op)
        if self.numel is not None and input_tensor.numel() != self.numel:
            raise RuntimeError(
                f"cgx all-gather of module '{self.name}': the all-gather input has {input_tensor.numel()} elements "
                f"but its shard table covers {self.numel} (parameters changed after set_cgx_all_gather?)")
        if self.adaptive is not None:
            self.adaptive.maybe_estimate(self, input_tensor, group, average=False)
        return _all_gather(output_tensor, input_tensor, bits=self.bits, bucket_size=self.bucket_size, group=group,
                           async_op=async_op, stochastic=False, seed=None, layers=self.layers, overlapped=True)


def set_cgx_all_gather(model: torch.nn.Module, bits: A2aBits = 4,
                       bucket_size: int = 512) -> List[CGXAllGather]:
    """Install a :class:`CGXAllGather` on every ``FSDPModule`` of ``model``, each with the
    per-parameter shard table (:func:`fsdp_shard_table`) of that module's parameter group; returns
    the comms. Call it after ``fully_shard`` and before the first forward."""
    from torch.distributed.fsdp import FSDPModule

    _check_gather_bits(bits)
    comms = []
    for name, m in model.named_modules():
        if not isinstance(m, FSDPModule):
            continue
        group = m._get_fsdp_state()._fsdp_param_group
        if group is None:  # a module without parameters of its own
            continue
        table = fsdp_shard_table([(p._orig_size, p.padded_sharded_param_size.numel()) for p in group.fsdp_params],
                                 bits, bucket_size)
        comm = CGXAllGather(bits, bucket_size, table, name or type(m).__name__)
        m.set_custom_all_gather(comm)
        comms.append(comm)
    return comms
