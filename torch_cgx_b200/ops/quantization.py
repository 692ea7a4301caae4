"""Standalone quantize / dequantize ops over a layer table.

``quantize`` turns a flat fp32/fp16/bf16 tensor into the packed wire bytes of
the compressed allreduce (per-bucket fp32 ``{unit, min}`` + ``bits``-bit
levels), ``dequantize`` inverts it.  CUDA tensors run the sm_90a kernels of
``csrc/kernels/quantize.cu``; CPU tensors run the bit-identical C++ path
(``csrc/common/block_ops.h``).  Role of ``gpu::quantize_maxmin`` /
``gpu::dequantize_maxmin`` in the reference (/root/reference/src/common/
compression/gpu_compression_operations.h:43-66).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from .. import _C

Layer = Tuple[int, int, int, int]  # (elem_off, numel, bits, bucket_size)


def _default_layers(t: torch.Tensor, bits: int, bucket_size: int) -> List[Layer]:
    return [(0, t.numel(), bits, bucket_size)]


def quantize(
    t: torch.Tensor,
    bits: int = 4,
    bucket_size: int = 512,
    layers: Optional[Sequence[Layer]] = None,
    *,
    stochastic: bool = False,
    seed: int = 0,
    seq: int = 0,
    skip_incomplete: bool = False,
    prescale: float = 1.0,
) -> torch.Tensor:
    """Packed wire bytes (uint8 tensor) of ``t``."""
    layers = list(layers) if layers is not None else _default_layers(t, bits, bucket_size)
    return _C.quantize(t.contiguous().view(-1), layers, 1, 1, skip_incomplete, prescale, stochastic, seed, seq, 0, 0, 2048)


def dequantize(
    wire: torch.Tensor,
    like: torch.Tensor,
    bits: int = 4,
    bucket_size: int = 512,
    layers: Optional[Sequence[Layer]] = None,
    *,
    skip_incomplete: bool = False,
) -> torch.Tensor:
    layers = list(layers) if layers is not None else _default_layers(like, bits, bucket_size)
    out = _C.dequantize(wire, like.contiguous().view(-1), layers, 1, 1, skip_incomplete, 2048)
    return out.view_as(like)


def fake_quantize(t: torch.Tensor, bits: int = 4, bucket_size: int = 512, **kw) -> torch.Tensor:
    """quantize -> dequantize round trip (what one compression step does to a gradient)."""
    return dequantize(quantize(t, bits, bucket_size, **kw), t, bits, bucket_size,
                      skip_incomplete=kw.get("skip_incomplete", False))


def wire_bytes(numel: int, bits: int, bucket_size: int, elsize: int = 4) -> int:
    """Packed size of one layer (meta is 2 x fp32 per bucket)."""
    if bits >= 32:
        return numel * elsize
    nb = (numel + bucket_size - 1) // bucket_size
    # every bucket starts a fresh pack group of 8 values (wire.h: block_num_groups)
    groups = (numel // bucket_size) * ((bucket_size + 7) // 8) + ((numel % bucket_size) + 7) // 8
    return nb * 8 + groups * bits


def compression_ratio(numel: int, bits: int, bucket_size: int, elsize: int = 4) -> float:
    return numel * elsize / wire_bytes(numel, bits, bucket_size, elsize)


def quantization_error(
    t: torch.Tensor,
    layers: Sequence[Layer],
    candidates: Sequence[int] = (2, 3, 4, 5, 6, 7, 8),
    *,
    stochastic: bool = False,
    prescale: float = 1.0,
    skip_incomplete: bool = False,
    chunks: int = 1,
    skip_chunk: int = -1,
) -> torch.Tensor:
    """Squared quantization error of every layer at every candidate width.

    ``t`` is flat fp32 / fp16 / bf16 on the CPU or a CUDA device; ``layers`` are
    ``(elem_off, numel, bits, bucket_size)`` tuples whose ``bits`` is ignored. Returns a float64
    ``[len(layers), len(candidates)]`` tensor on ``t.device``: entry ``[l, k]`` is
    sum_i (decode(encode(x_i)) - x_i)^2 of layer ``l`` at ``candidates[k]`` bits, with the levels of
    the real quantizer (or, ``stochastic=True``, the expected squared error of stochastic rounding).
    ``x_i`` is the fp32 value after ``prescale``. A bucket with NaN / Inf makes its layer's row NaN.
    CUDA tensors run ``csrc/kernels/quant_error.cu``, CPU tensors its C++ oracle
    (``csrc/common/quant_error.h``); both give the same bits.

    ``chunks > 1`` estimates what a reduce-scatter quantizes, in one launch: ``t`` holds ``chunks``
    shards of ``t.numel() // chunks`` elements, ``layers`` is one shard's table (offsets from the
    shard start, as in ``reduce_scatter_tensor``), and row ``l`` is layer ``l``'s error summed over
    every shard except ``skip_chunk`` (the receiving rank's own, which is not quantized; -1 keeps
    all). The sum runs chunk by chunk, then bucket by bucket, in the same order on the CPU and the
    GPU. ``chunks=1`` is the plain table above, bit for bit.
    """
    return _C.quantization_error(t.view(-1), [tuple(int(v) for v in l) for l in layers],
                                 [int(c) for c in candidates], stochastic, float(prescale), skip_incomplete,
                                 int(chunks), int(skip_chunk))
