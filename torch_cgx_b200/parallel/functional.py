"""Per-call control of the compression parameters.

The backend re-reads ``CGX_COMPRESSION_*`` on every allreduce (like the reference,
/root/reference/src/common/compressor.cc:39-45,258-263 -- its tests rely on it), so a context
manager that sets them is all that is needed to quantize *one* collective differently::

    with cgx.compression(bits=2, bucket_size=256, stochastic=True):
        dist.all_reduce(grad)              # 2-bit QSGD for this call only
    cgx.all_reduce(t, bits=8, average=True)  # same thing as a function

The compressed reduce-scatter is asked for explicitly (``dist.reduce_scatter_tensor`` on a
``cgx`` group keeps going to the uncompressed delegate)::

    cgx.reduce_scatter_tensor(shard, flat_grads, bits=4, average=True)

and so is the compressed all-gather (``dist.all_gather_into_tensor`` stays uncompressed)::

    cgx.all_gather_into_tensor(flat_params, shard, bits=8)
"""
from __future__ import annotations

import contextlib
import os
from typing import Iterator, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

_VARS = {
    "bits": "CGX_COMPRESSION_QUANTIZATION_BITS",
    "bucket_size": "CGX_COMPRESSION_BUCKET_SIZE",
    "skip_incomplete": "CGX_COMPRESSION_SKIP_INCOMPLETE_BUCKETS",
    "stochastic": "CGX_STOCHASTIC_ROUNDING",
    "seed": "CGX_SEED",
}


@contextlib.contextmanager
def compression(bits: Optional[int] = None, bucket_size: Optional[int] = None,
                skip_incomplete: Optional[bool] = None, stochastic: Optional[bool] = None,
                seed: Optional[int] = None) -> Iterator[None]:
    """Temporarily override the env-level compression config (None = leave as is; bits=32 disables)."""
    new = {"bits": bits, "bucket_size": bucket_size, "skip_incomplete": skip_incomplete,
           "stochastic": stochastic, "seed": seed}
    saved = {}
    try:
        for k, v in new.items():
            if v is None:
                continue
            var = _VARS[k]
            saved[var] = os.environ.get(var)
            os.environ[var] = str(int(v))
        yield
    finally:
        for var, old in saved.items():
            if old is None:
                os.environ.pop(var, None)
            else:
                os.environ[var] = old


def all_reduce(tensor: torch.Tensor, bits: Optional[int] = None, bucket_size: Optional[int] = None,
               average: bool = False, group=None, async_op: bool = False, **kw):
    """``dist.all_reduce`` (SUM or AVG) with the given quantization for this call.

    Note: with ``async_op=True`` the parameters are captured when the call is *issued*.
    """
    op = dist.ReduceOp.AVG if average else dist.ReduceOp.SUM
    with compression(bits=bits, bucket_size=bucket_size, **kw):
        return dist.all_reduce(tensor, op=op, group=group, async_op=async_op)


def _sharded(method: str, api: str, output: torch.Tensor, input: torch.Tensor, head: tuple, *, group,
             async_op: bool, stochastic: bool, seed: Optional[int],
             layers: Optional[Sequence[Tuple[int, int, int, int]]], overlapped: bool):
    """``native.<method>(output, input, *head, stochastic, seed, overlapped, layers)`` on the group's cgx backend."""
    from .hooks import _native_backend

    native = _native_backend(group if group is not None else dist.group.WORLD, input)
    if native is None:
        raise RuntimeError(f"cgx.{api} needs a process group with the cgx backend")
    work = getattr(native, method)(output, input, *head, bool(stochastic), -1 if seed is None else int(seed),
                                   bool(overlapped), [tuple(int(v) for v in l) for l in (layers or [])])
    if async_op:
        return work
    work.wait()  # the current stream waits for the kernel; the host does not
    return None


def _reduce_scatter(output: torch.Tensor, input: torch.Tensor, *, bits: int, bucket_size: int, average: bool,
                    group, async_op: bool, stochastic: bool, seed: Optional[int],
                    layers: Optional[Sequence[Tuple[int, int, int, int]]], skip_incomplete: bool,
                    overlapped: bool):
    return _sharded("reduce_scatter_compressed", "reduce_scatter_tensor", output, input,
                    (bool(average), int(bits), int(bucket_size), bool(skip_incomplete)), group=group,
                    async_op=async_op, stochastic=stochastic, seed=seed, layers=layers, overlapped=overlapped)


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, bits: int = 4, bucket_size: int = 512,
                          average: bool = False, group=None, async_op: bool = False, stochastic: bool = False,
                          seed: Optional[int] = None, layers: Optional[Sequence[Tuple[int, int, int, int]]] = None,
                          skip_incomplete: bool = False):
    """Compressed ``dist.reduce_scatter_tensor`` (SUM, or AVG with ``average=True``) on a ``cgx`` group.

    ``input`` holds ``world * output.numel()`` elements; rank r receives shard r. Every peer's
    contribution is quantized once (``bits``, buckets of ``bucket_size`` counted from each shard's
    start) and summed in fp32 with the receiving rank's own, unquantized values. ``layers``
    optionally gives one shard's quantization table as ``(elem_off, numel, bits, bucket_size)``
    tuples relative to the shard start (bits 32: uncompressed); the same table applies to every
    shard. ``seed=None`` uses ``CGX_SEED``. ``output`` may be the rank's own chunk of ``input``.
    Single node, CUDA float32 / float16 / bfloat16.
    """
    return _reduce_scatter(output, input, bits=bits, bucket_size=bucket_size, average=average, group=group,
                           async_op=async_op, stochastic=stochastic, seed=seed, layers=layers,
                           skip_incomplete=skip_incomplete, overlapped=False)


def _all_gather(output: torch.Tensor, input: torch.Tensor, *, bits: int, bucket_size: int, group, async_op: bool,
                stochastic: bool, seed: Optional[int], layers: Optional[Sequence[Tuple[int, int, int, int]]],
                overlapped: bool):
    return _sharded("all_gather_compressed", "all_gather_into_tensor", output, input, (int(bits), int(bucket_size)),
                    group=group, async_op=async_op, stochastic=stochastic, seed=seed, layers=layers,
                    overlapped=overlapped)


def all_gather_into_tensor(output: torch.Tensor, input: torch.Tensor, bits: int = 4, bucket_size: int = 512,
                           group=None, async_op: bool = False, stochastic: bool = False, seed: Optional[int] = None,
                           layers: Optional[Sequence[Tuple[int, int, int, int]]] = None):
    """Compressed ``dist.all_gather_into_tensor`` on a ``cgx`` group.

    ``output`` holds ``world * input.numel()`` elements; chunk q receives rank q's ``input``
    quantized once (``bits``, buckets of ``bucket_size`` counted from each shard's start) and
    decoded. The owner's own chunk is decoded from the same bytes, so every rank's ``output`` is
    identical (at world 1 it is the quantization round trip of ``input``). ``layers`` optionally
    gives one shard's quantization table as ``(elem_off, numel, bits, bucket_size)`` tuples
    (bits 32: copied unchanged). Round to nearest unless ``stochastic``; ``seed=None`` uses
    ``CGX_SEED``. ``input`` may be the rank's own chunk of ``output``. Single node, CUDA float32 /
    float16 / bfloat16.
    """
    return _all_gather(output, input, bits=bits, bucket_size=bucket_size, group=group, async_op=async_op,
                       stochastic=stochastic, seed=seed, layers=layers, overlapped=False)
