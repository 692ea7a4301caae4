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

Both also take an FP8 wire format, ``bits="e4m3"`` or ``"e5m2"`` (or ``"e4m3_pow2"`` / ``"e5m2_pow2"``,
with power-of-two scales, or ``"e4m3_sr"`` / ``"e5m2_sr"``, rounded stochastically), in place of
max-min 8-bit.

and the compressed all-to-all of expert-parallel MoE layers (``dist.all_to_all_single`` stays
uncompressed)::

    cgx.all_to_all_single(recv, tokens, recv_splits, send_splits, bits=8)
    y = cgx.differentiable_all_to_all_single(tokens, recv_splits, send_splits, bits="e4m3", grad_bits="e5m2")
    x = cgx.differentiable_all_to_all_dispatch(tokens, slot_order, recv_splits, send_splits, bits="e4m3")
"""
from __future__ import annotations

import contextlib
import os
from typing import Iterator, List, Optional, Sequence, Tuple, Union

import torch
import torch.distributed as dist

_VARS = {
    "bits": "CGX_COMPRESSION_QUANTIZATION_BITS",
    "bucket_size": "CGX_COMPRESSION_BUCKET_SIZE",
    "skip_incomplete": "CGX_COMPRESSION_SKIP_INCOMPLETE_BUCKETS",
    "stochastic": "CGX_STOCHASTIC_ROUNDING",
    "seed": "CGX_SEED",
}


_FORMAT_VAR = "CGX_COMPRESSION_FORMAT"


@contextlib.contextmanager
def compression(bits: Optional[A2aBits] = None, bucket_size: Optional[int] = None,
                skip_incomplete: Optional[bool] = None, stochastic: Optional[bool] = None,
                seed: Optional[int] = None) -> Iterator[None]:
    """Temporarily override the env-level compression config (None = leave as is; bits=32 disables).

    ``bits="e4m3"``, ``"e5m2"``, ``"e4m3_pow2"``, ``"e5m2_pow2"``, ``"e4m3_sr"`` or ``"e5m2_sr"``
    compresses at 8 bits and sends the allreduce's 8-bit layers as FP8 codes with one fp32 scale per
    bucket (``CGX_COMPRESSION_FORMAT``; the ``_pow2`` formats' scales are powers of two, the ``_sr``
    formats round stochastically, see ``all_to_all_single``); an integer ``bits`` selects max-min.
    The other FP8 formats round to nearest: an unknown name, or one of them with ``stochastic=True``
    or ``CGX_STOCHASTIC_ROUNDING=1``, raises ValueError before anything is changed.
    """
    fmt = None
    if bits is not None:
        if isinstance(bits, str):
            from .. import _C

            _C.a2a_bits(bits, bool(stochastic), "allreduce")  # CGX_STOCHASTIC_ROUNDING=1: the call raises
            fmt, bits = bits, 8
        else:
            fmt = "maxmin"
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
        if fmt is not None:
            saved[_FORMAT_VAR] = os.environ.get(_FORMAT_VAR)
            os.environ[_FORMAT_VAR] = fmt
        yield
    finally:
        for var, old in saved.items():
            if old is None:
                os.environ.pop(var, None)
            else:
                os.environ[var] = old


def all_reduce(tensor: torch.Tensor, bits: Optional[A2aBits] = None, bucket_size: Optional[int] = None,
               average: bool = False, group=None, async_op: bool = False, **kw):
    """``dist.all_reduce`` (SUM or AVG) with the given quantization for this call; ``bits`` may be an
    FP8 format, ``"e4m3"`` or ``"e5m2"`` (see :func:`compression`).

    Note: with ``async_op=True`` the parameters are captured when the call is *issued*.
    """
    op = dist.ReduceOp.AVG if average else dist.ReduceOp.SUM
    with compression(bits=bits, bucket_size=bucket_size, **kw):
        return dist.all_reduce(tensor, op=op, group=group, async_op=async_op)


def _sharded(method: str, api: str, output: torch.Tensor, input: torch.Tensor, head: tuple, *, group,
             async_op: bool, stochastic: bool, seed: Optional[int],
             layers: Optional[Sequence[Tuple[int, int, int, int]]], overlapped: bool, **native_kw):
    """``native.<method>(output, input, *head, stochastic, seed, overlapped, layers, **native_kw)`` on the
    group's cgx backend."""
    from .hooks import _native_backend

    native = _native_backend(group if group is not None else dist.group.WORLD, input)
    if native is None:
        raise RuntimeError(f"cgx.{api} needs a process group with the cgx backend")
    work = getattr(native, method)(output, input, *head, bool(stochastic), -1 if seed is None else int(seed),
                                   bool(overlapped), [tuple(int(v) for v in l) for l in (layers or [])],
                                   **native_kw)
    if async_op:
        return work
    work.wait()  # the current stream waits for the kernel; the host does not
    return None


A2aBits = Union[int, str]  # 1..8, 32, or an FP8 wire format: "e4m3" / "e5m2" / "e4m3_pow2" / "e5m2_pow2" /
# "e4m3_sr" / "e5m2_sr"


def _sharded_bits(bits: A2aBits, stochastic: bool, layers: Optional[Sequence[Tuple[int, int, int, int]]],
                  op: str) -> A2aBits:
    """``bits`` of the compressed reduce-scatter / all-gather as the native call takes it: an int, or
    an FP8 format name, whose ``layers`` table may hold bits 8 (FP8) and 32 (raw) only. ValueError
    otherwise, before anything is sent."""
    if not isinstance(bits, str):
        return int(bits)
    from .. import _C

    _C.a2a_bits(bits, bool(stochastic), op)
    for l in layers or []:
        if int(l[2]) != 8 and int(l[2]) < 32:
            raise ValueError(f"cgx {op}: bits={bits!r} needs a layer table of bits 8 or 32, got a layer of {l[2]}")
    return bits


def _reduce_scatter(output: torch.Tensor, input: torch.Tensor, *, bits: A2aBits, bucket_size: int, average: bool,
                    group, async_op: bool, stochastic: bool, seed: Optional[int],
                    layers: Optional[Sequence[Tuple[int, int, int, int]]], skip_incomplete: bool,
                    overlapped: bool):
    bits = _sharded_bits(bits, stochastic, layers, "reduce_scatter")
    return _sharded("reduce_scatter_compressed", "reduce_scatter_tensor", output, input,
                    (bool(average), bits, int(bucket_size), bool(skip_incomplete)), group=group,
                    async_op=async_op, stochastic=stochastic, seed=seed, layers=layers, overlapped=overlapped)


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, bits: A2aBits = 4, bucket_size: int = 512,
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
    CUDA float32 / float16 / bfloat16.

    ``bits="e4m3"`` or ``"e5m2"`` sends the bytes of ``bits=8`` as FP8 (see ``all_to_all_single``):
    per bucket one fp32 scale ``unit = max|y| / FMAX`` of the prescaled values ``y``, and one FP8 code
    of ``y / unit`` per element. The receiver adds each decoded value ``code * unit`` to its fp32 sum
    in rank order. ``e5m2``'s wider exponent range suits gradients. A ``layers`` table may then hold
    bits 8 (FP8) and 32 (raw) only. A NaN or an Inf in a peer's bucket makes that bucket of the sum
    NaN. FP8 rounds to nearest only: ``stochastic=True`` raises ``ValueError``, as does any other
    string. ``"e4m3_pow2"`` / ``"e5m2_pow2"`` use power-of-two scales, and ``"e4m3_sr"`` /
    ``"e5m2_sr"`` round stochastically whatever ``stochastic`` says (see ``all_to_all_single``).

    Over several nodes (``local_size`` consecutive ranks each) the reduction has two stages: inside
    each node, for every node's block of shards, the reduce-scatter above over the local ranks
    (prescaled by 1/world when averaging; uncompressed with ``CGX_INTRA_COMPRESS=0``) gives the
    node's partial sum of each shard; then across nodes, among the ranks of one local rank, the
    same reduce-scatter of those partials: a rank's own node partial stays unquantized and every
    other node's is quantized once. A local peer's values are thus quantized once and a remote
    one's at most twice. With one rank per node it is the single-stage reduce-scatter over all ranks.
    """
    return _reduce_scatter(output, input, bits=bits, bucket_size=bucket_size, average=average, group=group,
                           async_op=async_op, stochastic=stochastic, seed=seed, layers=layers,
                           skip_incomplete=skip_incomplete, overlapped=False)


def _all_gather(output: torch.Tensor, input: torch.Tensor, *, bits: A2aBits, bucket_size: int, group,
                async_op: bool, stochastic: bool, seed: Optional[int],
                layers: Optional[Sequence[Tuple[int, int, int, int]]], overlapped: bool,
                output_scales: Optional[torch.Tensor] = None):
    bits = _sharded_bits(bits, stochastic, layers, "all_gather")
    kw = {}
    if output_scales is not None:
        _check_ag_codes_output(output, input, output_scales, bits, int(bucket_size), layers)
        kw["output_scales"] = output_scales
    return _sharded("all_gather_compressed", "all_gather_into_tensor", output, input, (bits, int(bucket_size)),
                    group=group, async_op=async_op, stochastic=stochastic, seed=seed, layers=layers,
                    overlapped=overlapped, **kw)


def all_gather_into_tensor(output: torch.Tensor, input: torch.Tensor, bits: A2aBits = 4, bucket_size: int = 512,
                           group=None, async_op: bool = False, stochastic: bool = False, seed: Optional[int] = None,
                           layers: Optional[Sequence[Tuple[int, int, int, int]]] = None,
                           output_scales: Optional[torch.Tensor] = None):
    """Compressed ``dist.all_gather_into_tensor`` on a ``cgx`` group.

    ``output`` holds ``world * input.numel()`` elements; chunk q receives rank q's ``input``
    quantized once (``bits``, buckets of ``bucket_size`` counted from each shard's start) and
    decoded. The owner's own chunk is decoded from the same bytes, so every rank's ``output`` is
    identical (at world 1 it is the quantization round trip of ``input``). ``layers`` optionally
    gives one shard's quantization table as ``(elem_off, numel, bits, bucket_size)`` tuples
    (bits 32: copied unchanged). Round to nearest unless ``stochastic``; ``seed=None`` uses
    ``CGX_SEED``. ``input`` may be the rank's own chunk of ``output``. CUDA float32 / float16 /
    bfloat16.

    ``bits="e4m3"`` or ``"e5m2"`` sends the bytes of ``bits=8`` as FP8 (see ``all_to_all_single``),
    the usual choice for weights being ``e4m3``. Every rank, the owner included, writes the values
    decoded from the same codes, so at world 1 the output is ``ops.oracle.fp8_quantize_dequantize``
    of the input. A ``layers`` table may then hold bits 8 (FP8) and 32 (raw) only; FP8 rounds to
    nearest only. ``"e4m3_pow2"`` / ``"e5m2_pow2"`` use power-of-two scales, and ``"e4m3_sr"`` /
    ``"e5m2_sr"`` round stochastically whatever ``stochastic`` says (see ``all_to_all_single``).

    Over several nodes the owner's quantized bytes first go to the ranks of the same local rank on
    the other nodes, which decode them; each node then shares the decoded shards among its ranks
    uncompressed. Every shard is still quantized exactly once, so with round-to-nearest every
    rank's ``output`` is the same as on one node.

    FP8 codes for an FP8 GEMM on the gathered tensor: with ``output_scales`` (and an FP8 ``bits``)
    ``output`` is a ``torch.float8_e4m3fn`` / ``torch.float8_e5m2`` tensor (the format's) of ``world *
    input.numel()`` elements that receives the wire's codes undecoded, and ``output_scales`` (CUDA
    float32, contiguous, ``output.numel() // bucket_size`` elements, any shape) the fp32 unit of
    every bucket: the bucket starting at element ``e`` of ``output`` has the scale
    ``output_scales.view(-1)[e // bucket_size]``. ``input.numel() % bucket_size == 0`` and
    ``bucket_size <= 8192``, so every bucket lies inside one shard. Each owner's chunk holds the
    bytes it sent, and ``(codes.float() * scales.view(-1).repeat_interleave(bucket_size))``, one
    fp32 multiply, rounded to the input dtype is the decoded call's output bit for bit. With
    ``bucket_size`` equal to a row of ``H`` elements there is one scale per row, the row-wise scaling
    ``torch._scaled_mm`` takes (``scale_a`` ``[M, 1]`` for gathered activations, ``scale_b`` ``[1, N]``
    for a gathered weight ``[N, K]`` used as ``codes.view(N, K).t()``). No ``layers`` table, round to
    nearest, one node only (several nodes raise on every rank); not differentiable.
    """
    return _all_gather(output, input, bits=bits, bucket_size=bucket_size, group=group, async_op=async_op,
                       stochastic=stochastic, seed=seed, layers=layers, overlapped=False, output_scales=output_scales)


def _splits(s: Optional[Sequence[int]]) -> List[int]:
    return [] if s is None else [int(v) for v in s]


def _a2a_bits(bits: A2aBits, stochastic: bool) -> A2aBits:
    """``bits`` as the native all-to-all takes it: an int, or an FP8 format name. An unknown name, or
    a round-to-nearest FP8 format with ``stochastic``, raises ValueError (the native parser's check,
    run here so that it fires before anything is sent)."""
    if not isinstance(bits, str):
        return int(bits)
    from .. import _C

    _C.a2a_bits(bits, bool(stochastic))
    return bits


def all_to_all_single(output: torch.Tensor, input: torch.Tensor, output_split_sizes: Optional[Sequence[int]] = None,
                      input_split_sizes: Optional[Sequence[int]] = None, bits: A2aBits = 8, bucket_size: int = 512,
                      group=None, async_op: bool = False, stochastic: bool = False, seed: Optional[int] = None,
                      input_index: Optional[torch.Tensor] = None, output_index: Optional[torch.Tensor] = None,
                      output_scales: Optional[torch.Tensor] = None, input_scale: Optional[torch.Tensor] = None):
    """Compressed ``dist.all_to_all_single`` on a ``cgx`` group.

    Splits count dim-0 rows (``None``: equal splits). Rows ``input_split_sizes[q]`` of ``input`` go
    to rank q, and the chunk from rank q lands in the ``output_split_sizes[q]`` rows of ``output``.
    The rank's own chunk is copied bit for bit. Every other chunk is quantized once by the sender
    (``bits`` 1..8, max-min, buckets of ``bucket_size`` counted from the chunk's first element) and
    decoded by the receiver; ``bits=32`` moves every chunk unchanged. Round to nearest unless
    ``stochastic``; ``seed=None`` uses ``CGX_SEED``.

    ``bits="e4m3"`` or ``"e5m2"`` sends the same bytes as ``bits=8`` but as FP8: per bucket one fp32
    scale ``unit = max|x| / FMAX`` (448 or 57344) and one FP8 code of ``x / unit`` per element,
    converted by Hopper's FP8 instructions. Its relative error per element is at most 2^-4 (e4m3)
    or 2^-3 (e5m2) whatever else the bucket holds, so it suits rows with a few outlier channels;
    max-min 8-bit is more accurate on well-behaved data. A bucket holding a NaN or an Inf decodes to
    NaN in every element. These formats round to nearest only: ``stochastic=True`` raises
    ``ValueError``, as does any other string.

    ``bits="e4m3_sr"`` or ``"e5m2_sr"`` sends the records, scales and decoder of e4m3 / e5m2, but
    rounds every code stochastically, whatever ``stochastic`` says (both values give the same bytes):
    ``y = x / unit`` becomes one of its two neighbours on the format's grid, the one away from zero
    with probability equal to its distance from the other (in steps of 2^-16). The decoded value is
    then unbiased up to 2^-16 of a grid step, and values far below the bucket's maximum survive in
    expectation instead of flushing to zero. The random bits are those integer stochastic rounding
    uses for the same elements: ``seed`` (``None``: ``CGX_SEED``), the call sequence and the pair of
    ranks. They suit gradients, whose rounding errors then cancel across steps and ranks.

    ``bits="e4m3_pow2"`` or ``"e5m2_pow2"`` sends the same bytes with the codes of e4m3 / e5m2 and a
    power-of-two scale per bucket, ``unit = 2^k`` with k the smallest integer >= -126 such that
    ``max|x| <= FMAX * 2^k``. Encoding and decoding are then exact multiplications, so quantizing
    the decoded values again at the same buckets gives them back unchanged, and every unit is
    exactly representable as ``torch.float8_e8m0fnu``. A zero bucket has unit 2^-126.

    Routed form, for MoE token dispatch and combine without a permutation copy: ``input_index``
    (CUDA int64, ``sum(input_split_sizes)`` entries in ``[0, input.shape[0])``, repeats allowed)
    makes row i of the sent buffer ``input[input_index[i]]``; ``output_index`` (``sum(output_split_sizes)``
    entries in ``[0, output.shape[0])``) writes row j of the received buffer to
    ``output[output_index[j]]`` and leaves the other rows of ``output`` unchanged (duplicates: unspecified,
    as with ``index_copy_``). The result is bitwise that of ``input.index_select(0, input_index)``,
    the plain call, then ``output.index_copy_(0, output_index, received)``; on the P2P transport,
    when every quantization item lies inside one row, the gather and the scatter happen inside the
    kernel. With an index, ``None`` splits divide the index's entries equally. An index value out of
    range is not checked on the host: the kernel skips that row and the call fails (``work.wait()``
    raises, naming the index), after which the group refuses further collectives.

    FP8 codes for an FP8 expert GEMM: with ``output_scales`` (and an FP8 ``bits``) ``output`` is a
    ``torch.float8_e4m3fn`` (e4m3, e4m3_pow2, e4m3_sr) / ``torch.float8_e5m2`` (e5m2, e5m2_pow2, e5m2_sr) tensor of the input's shape per
    row that receives the wire's codes undecoded, and ``output_scales`` (CUDA float32, contiguous,
    ``[output.shape[0], H // bucket_size]`` with ``H`` the elements of a row) the fp32 unit of every
    bucket. ``H % bucket_size == 0`` and ``bucket_size <= 8192``, so every bucket lies inside one row;
    ``bucket_size == H`` gives one scale per row, the row-wise scaling ``torch._scaled_mm`` takes.
    ``codes[j, bB:(b+1)B].float() * output_scales[j, b]`` is the value the decoded call gives before
    its rounding to the input dtype. The own chunk is encoded too, with the peers' encoder. The index
    keywords route codes and scales rows alike. Not differentiable.

    Scaled rows on send, for the backward of an MoE combine: with ``input_index``, ``input_scale``
    (a contiguous CUDA float32 vector, one entry per ``input_index`` entry) makes sent row i
    ``(input[input_index[i]].float() * input_scale[i]).to(input.dtype)``: one fp32 multiply, rounded
    to nearest even (fp32 input: no second rounding). The call then behaves exactly like the routed
    call on those rows (quantization, stochastic rounding, every ``bits``, ``output_index``, the own
    chunk copied bit for bit as scaled). NaN, Inf, zero and negative scales follow from that
    arithmetic. ``ValueError`` before anything is sent without ``input_index``, for a scale of the
    wrong dtype, device, layout or length, with ``output_scales``, or for a scale overlapping
    ``output``.

    As with NCCL, the splits are the caller's contract: rank q's ``input_split_sizes[r]`` must equal
    rank r's ``output_split_sizes[q]``. Malformed splits on one rank (wrong length, sum or sign, or
    rows of another size than the output's) raise ``RuntimeError`` before anything is launched.
    CUDA float32 / float16 / bfloat16, contiguous, ``output`` not overlapping ``input``, at most 16
    ranks on one node, at most 256 over several nodes (each of at most 16 ranks), where the result is
    the same as on one node, bit for bit.
    """
    from .hooks import _native_backend

    bits = _a2a_bits(bits, stochastic)
    if input_scale is not None:
        _check_input_scale(output, input, input_index, input_scale, output_scales)
    if output_scales is not None:
        _check_codes_output(output, input, output_scales, bits, int(bucket_size))
    native = _native_backend(group if group is not None else dist.group.WORLD, input)
    if native is None:
        raise RuntimeError("cgx.all_to_all_single needs a process group with the cgx backend")
    work = native.all_to_all_compressed(output, input, _splits(output_split_sizes), _splits(input_split_sizes),
                                        bits, int(bucket_size), bool(stochastic), -1 if seed is None else int(seed),
                                        input_index, output_index, output_scales, None, None, input_scale)
    if async_op:
        return work
    work.wait()  # the current stream waits for the kernel; the host does not
    return None


def _check_input_scale(output: torch.Tensor, input: torch.Tensor, input_index: Optional[torch.Tensor],
                       scale: torch.Tensor, output_scales: Optional[torch.Tensor]) -> None:
    """ValueError unless ``scale`` can be the ``input_scale`` of ``all_to_all_single``; the checks that
    need no GPU come first, the device check last."""
    api = "cgx.all_to_all_single"
    if input_index is None:
        raise ValueError(f"{api}: input_scale needs an input_index (one scale per sent row)")
    if output_scales is not None:
        raise ValueError(f"{api}: input_scale has no codes output (output_scales)")
    n = int(input_index.shape[0]) if input_index.dim() == 1 else -1
    if scale.dtype != torch.float32 or scale.dim() != 1 or not scale.is_contiguous() or scale.shape[0] != n:
        raise ValueError(f"{api}: input_scale must be a contiguous float32 vector of one entry per input_index "
                         f"entry ({n}), got {scale.dtype} {list(scale.shape)}"
                         f"{'' if scale.is_contiguous() else ' (not contiguous)'}")
    if _overlaps(scale, output):
        raise ValueError(f"{api}: input_scale overlaps the output")
    if not scale.is_cuda or scale.device != input.device:
        raise ValueError(f"{api}: input_scale must be on the input's CUDA device, got {scale.device}")


def _check_codes_format(api: str, output: torch.Tensor, bits: A2aBits) -> None:
    """ValueError unless ``bits`` is an FP8 format and ``output`` a tensor of its float8 dtype (the
    codes output of ``api``)."""
    from ..ops.oracle import FP8_FORMATS, FP8_SR_FORMATS

    if not isinstance(bits, str):
        raise ValueError(f"cgx.{api}: output_scales needs bits='e4m3', 'e5m2', 'e4m3_pow2', 'e5m2_pow2', "
                         f"'e4m3_sr' or 'e5m2_sr', got bits={bits}")
    want = FP8_FORMATS[FP8_SR_FORMATS.get(bits, bits)][0]
    if output.dtype != want:
        raise ValueError(f"cgx.{api}: with bits={bits!r} and output_scales the output must be {want}, "
                         f"got {output.dtype}")


def _check_ag_codes_output(output: torch.Tensor, input: torch.Tensor, scales: torch.Tensor, bits: A2aBits,
                           bucket_size: int, layers) -> None:
    """ValueError unless (output, scales) can receive the codes output of ``all_gather_into_tensor``."""
    api = "all_gather_into_tensor"
    _check_codes_format(api, output, bits)
    if layers:
        raise ValueError(f"cgx.{api}: output_scales takes no layers table (one FP8 layer per shard)")
    S = input.numel()
    if bucket_size < 1 or bucket_size > 8192 or S % bucket_size != 0:
        raise ValueError(f"cgx.{api}: output_scales needs a bucket_size <= 8192 that divides the input's {S} "
                         f"elements, got {bucket_size}")
    n = output.numel() // bucket_size
    if (scales.dtype != torch.float32 or not scales.is_cuda or scales.device != output.device
            or not scales.is_contiguous() or scales.numel() != n):
        raise ValueError(f"cgx.{api}: output_scales must be a contiguous float32 tensor of {n} elements on "
                         f"{output.device}, got {scales.dtype} {list(scales.shape)} on {scales.device}"
                         f"{'' if scales.is_contiguous() else ' (not contiguous)'}")


def _check_codes_output(output: torch.Tensor, input: torch.Tensor, scales: torch.Tensor, bits: A2aBits,
                        bucket_size: int) -> None:
    """ValueError unless (output, scales) can receive the codes output of ``all_to_all_single``."""
    _check_codes_format("all_to_all_single", output, bits)
    H = 1
    for d in input.shape[1:]:
        H *= int(d)
    if bucket_size < 1 or bucket_size > 8192 or H % bucket_size != 0:
        raise ValueError(f"cgx.all_to_all_single: output_scales needs a bucket_size <= 8192 that divides the row "
                         f"length {H}, got {bucket_size}")
    shape = (output.shape[0], H // bucket_size)
    if (scales.dtype != torch.float32 or not scales.is_cuda or scales.device != output.device
            or not scales.is_contiguous() or tuple(scales.shape) != shape):
        raise ValueError(f"cgx.all_to_all_single: output_scales must be a contiguous float32 tensor of shape "
                         f"{list(shape)} on {output.device}, got {scales.dtype} {list(scales.shape)} on "
                         f"{scales.device}{'' if scales.is_contiguous() else ' (not contiguous)'}")


def _a2a_output(input: torch.Tensor, output_split_sizes: Optional[Sequence[int]],
                input_index: Optional[torch.Tensor]) -> torch.Tensor:
    if output_split_sizes is not None:
        rows = sum(int(v) for v in output_split_sizes)
    else:
        rows = input_index.shape[0] if input_index is not None else input.shape[0]
    return input.new_empty((rows,) + tuple(input.shape[1:]))


def _routes(input_index: Optional[torch.Tensor], output_index: Optional[torch.Tensor]) -> dict:
    """the index keywords of all_to_all_single that are set"""
    kw = {"input_index": input_index, "output_index": output_index}
    return {k: v for k, v in kw.items() if v is not None}


class _AllToAll(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, output_split_sizes, input_split_sizes, bits, grad_bits, bucket_size, group, stochastic,
                input_index, output_index, output_rows):
        ctx.splits = (output_split_sizes, input_split_sizes)
        ctx.grad_bits, ctx.bucket_size, ctx.group, ctx.stochastic = grad_bits, bucket_size, group, stochastic
        ctx.in_shape = input.shape
        ctx.index = (input_index, output_index)
        input = input.contiguous()
        if output_index is None:
            out = _a2a_output(input, output_split_sizes, input_index)
        else:
            out = input.new_zeros((int(output_rows),) + tuple(input.shape[1:]))  # rows nobody names stay zero
        all_to_all_single(out, input, output_split_sizes, input_split_sizes, bits=bits, bucket_size=bucket_size,
                          group=group, stochastic=stochastic, **_routes(input_index, output_index))
        return out

    @staticmethod
    def backward(ctx, grad):
        out_splits, in_splits = ctx.splits
        input_index, output_index = ctx.index
        grad = grad.contiguous()
        # the gradient travels back: the forward's output splits are its input splits, and the rows
        # the forward scattered by output_index are gathered by it on the way back
        if input_index is None:
            gin = grad.new_empty(ctx.in_shape)
        else:
            rows = sum(int(v) for v in in_splits) if in_splits is not None else input_index.shape[0]
            gin = grad.new_empty((rows,) + tuple(ctx.in_shape[1:]))
        all_to_all_single(gin, grad, in_splits, out_splits, bits=ctx.grad_bits, bucket_size=ctx.bucket_size,
                          group=ctx.group, stochastic=ctx.stochastic, **_routes(output_index, None))
        if input_index is not None:
            # a row sent to several ranks collects every copy's gradient (index_select's backward)
            gin = grad.new_zeros(ctx.in_shape).index_add_(0, input_index, gin)
        return gin, None, None, None, None, None, None, None, None, None, None


def differentiable_all_to_all_single(input: torch.Tensor, output_split_sizes: Optional[Sequence[int]] = None,
                                     input_split_sizes: Optional[Sequence[int]] = None, bits: A2aBits = 8,
                                     grad_bits: Optional[A2aBits] = None, bucket_size: int = 512, group=None,
                                     stochastic: bool = False, input_index: Optional[torch.Tensor] = None,
                                     output_index: Optional[torch.Tensor] = None,
                                     output_rows: Optional[int] = None) -> torch.Tensor:
    """``all_to_all_single`` that returns its output and has a backward pass: the compressed
    all-to-all of the gradient with the splits swapped, at ``grad_bits`` (``None``: ``bits``; 32:
    exact). This is the form an MoE layer calls for its token dispatch and combine. Either may be an
    FP8 format; ``bits="e4m3", grad_bits="e5m2"`` is the usual FP8 recipe. Both are checked before
    the forward sends anything.

    ``input_index`` / ``output_index`` route rows as in ``all_to_all_single``. With ``output_index``
    the result has ``output_rows`` rows, and rows it does not name are zero. The backward gathers
    the gradient by ``output_index`` inside the exchange and, with ``input_index``, sums what
    comes back into a zero gradient with ``index_add_``, so a row sent to several ranks receives
    the sum of its copies' gradients."""
    if output_index is not None and output_rows is None:
        raise ValueError("cgx.differentiable_all_to_all_single: output_index needs output_rows")
    bits = _a2a_bits(bits, stochastic)
    gb = _a2a_bits(bits if grad_bits is None else grad_bits, stochastic)
    return _AllToAll.apply(input, None if output_split_sizes is None else _splits(output_split_sizes),
                           None if input_split_sizes is None else _splits(input_split_sizes), bits, gb,
                           int(bucket_size), group, bool(stochastic), input_index, output_index, output_rows)


def _overlaps(a: torch.Tensor, b: torch.Tensor) -> bool:
    """whether the bytes of two dense tensors overlap (same device)"""
    if a.device != b.device or a.numel() == 0 or b.numel() == 0:
        return False
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


def _check_combine(output: torch.Tensor, input: torch.Tensor, gate: torch.Tensor, output_index: torch.Tensor,
                   slots: Optional[torch.Tensor], input_index: Optional[torch.Tensor] = None) -> None:
    """ValueError unless the arguments of ``all_to_all_combine`` are well formed. The checks that need
    no GPU come first, the device checks last."""
    api = "cgx.all_to_all_combine"
    if output.dtype != input.dtype:
        raise ValueError(f"{api}: the output must have the input's dtype {input.dtype}, got {output.dtype} "
                         "(a codes output has no combine)")
    if gate.dtype != torch.float32 or gate.dim() != 2 or not gate.is_contiguous():
        raise ValueError(f"{api}: the gate must be a contiguous float32 tensor [T, k], got {gate.dtype} "
                         f"{list(gate.shape)}{'' if gate.is_contiguous() else ' (not contiguous)'}")
    T, k = int(gate.shape[0]), int(gate.shape[1])
    if not 1 <= k <= 32:
        raise ValueError(f"{api}: k = {k} choices per token, at most 32 are supported")
    rows = tuple(input.shape[1:])
    if tuple(output.shape) != (T,) + rows or not output.is_contiguous():
        raise ValueError(f"{api}: the output must be a contiguous tensor of shape {[T, *rows]}, got "
                         f"{list(output.shape)}")
    if output_index.dtype != torch.int64 or output_index.dim() != 1 or output_index.numel() != T * k:
        raise ValueError(f"{api}: output_index must be an int64 vector of T * k = {T * k} entries, got "
                         f"{output_index.dtype} {list(output_index.shape)}")
    if input_index is not None and (input_index.dtype != torch.int64 or input_index.dim() != 1
                                    or not input_index.is_contiguous()):
        raise ValueError(f"{api}: input_index must be a contiguous int64 vector, got {input_index.dtype} "
                         f"{list(input_index.shape)}")
    if slots is not None and (slots.dtype != input.dtype or tuple(slots.shape) != (T * k,) + rows
                              or not slots.is_contiguous()):
        raise ValueError(f"{api}: slots must be a contiguous {input.dtype} tensor of shape {[T * k, *rows]}, got "
                         f"{slots.dtype} {list(slots.shape)}")
    for name, t in (("the output", output), ("slots", slots), ("the gate", gate)):
        if t is not None and _overlaps(t, input):
            raise ValueError(f"{api}: {name} overlaps the input")
    if slots is not None and _overlaps(slots, output):
        raise ValueError(f"{api}: slots overlap the output")
    for name, t in (("input", input), ("output", output), ("gate", gate), ("output_index", output_index),
                    ("slots", slots), ("input_index", input_index)):
        if t is not None and (not t.is_cuda or t.device != input.device):
            raise ValueError(f"{api}: {name} must be on the input's CUDA device, got {t.device}")


def all_to_all_combine(output: torch.Tensor, input: torch.Tensor, gate: torch.Tensor, output_index: torch.Tensor,
                       output_split_sizes: Optional[Sequence[int]] = None,
                       input_split_sizes: Optional[Sequence[int]] = None, bits: A2aBits = 8, bucket_size: int = 512,
                       group=None, async_op: bool = False, stochastic: bool = False, seed: Optional[int] = None,
                       slots: Optional[torch.Tensor] = None, input_index: Optional[torch.Tensor] = None):
    """The routed compressed all-to-all of an MoE combine followed by the weighted top-k sum, in one call.

    ``gate`` is a contiguous CUDA float32 ``[T, k]`` (``1 <= k <= 32``), ``output`` ``[T, ...]`` in the
    input's dtype and row shape, ``output_index`` a CUDA int64 permutation of ``[0, T*k)`` with
    ``sum(output_split_sizes)`` entries. Slot ``s = t*k + c`` is choice ``c`` of token ``t``.
    ``input_index`` (optional, CUDA int64, ``sum(input_split_sizes)`` entries) gathers the sent rows
    from ``input`` as in ``all_to_all_single``, for an input whose rows are grouped otherwise (by
    local expert, say). The call is defined as the composition
      1. ``slots = all_to_all_single(slots, input, ..., input_index=input_index, output_index=output_index)``
         (any ``bits``, stochastic rounding included, the own chunk copied bit for bit), into a
         ``[T*k, ...]`` buffer;
      2. for every ``t`` and element ``h``, with ``x_c = float(slots[t*k + c, h])`` and
         ``g_c = gate[t, c]``: ``acc = fp32(g_0 * x_0)``, then ``acc = fma(g_c, x_c, acc)`` for
         ``c = 1 .. k-1`` in that order, and ``output[t, h] = acc`` rounded to nearest in the dtype.
    NaN and signed zeros follow from that arithmetic. With ``slots`` given, it receives exactly the
    routed call's rows; otherwise the buffer is scratch.

    On the P2P transport, when every quantization item lies inside one row, the sum happens inside
    the all-to-all kernel: the last warp to store a token's slot segment sums it, so the slots are
    read back while they are likely still in L2, with no extra launch. Elsewhere (NCCL transport,
    rows the kernel cannot route, world 1 without a heap) the routed composition runs, then one
    standalone combine kernel with the same arithmetic; both give the same bits.

    Raises ``ValueError`` before anything runs for a gate of the wrong dtype, device, layout or
    shape, ``k > 32``, an index length other than ``T*k``, an output, slots or gate that overlap the
    input, and a float8 output (a codes output has no combine). A repeated slot, like an index out
    of range, is found by the kernel: the call fails (``work.wait()`` raises, naming
    ``output_index``) and the group refuses further collectives. Dropped tokens (an index that is
    not a permutation) are not supported: call ``all_to_all_single`` and sum the rows yourself.
    """
    from .hooks import _native_backend

    bits = _a2a_bits(bits, stochastic)
    _check_combine(output, input, gate, output_index, slots, input_index)
    if slots is None:
        slots = input.new_empty((gate.shape[0] * gate.shape[1],) + tuple(input.shape[1:]))
    native = _native_backend(group if group is not None else dist.group.WORLD, input)
    if native is None:
        raise RuntimeError("cgx.all_to_all_combine needs a process group with the cgx backend")
    work = native.all_to_all_compressed(slots, input, _splits(output_split_sizes), _splits(input_split_sizes),
                                        bits, int(bucket_size), bool(stochastic), -1 if seed is None else int(seed),
                                        input_index, output_index, None, gate, output)
    if async_op:
        return work
    work.wait()
    return None


class _AllToAllCombine(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, gate, output_index, output_split_sizes, input_split_sizes, bits, grad_bits, bucket_size,
                group, stochastic, gate_grad):
        input, gate = input.contiguous(), gate.contiguous()
        T, k = gate.shape
        slots = input.new_empty((T * k,) + tuple(input.shape[1:]))
        out = input.new_empty((T,) + tuple(input.shape[1:]))
        all_to_all_combine(out, input, gate, output_index, output_split_sizes, input_split_sizes, bits=bits,
                           bucket_size=bucket_size, group=group, stochastic=stochastic, slots=slots)
        ctx.save_for_backward(gate, slots, output_index)
        ctx.splits = (output_split_sizes, input_split_sizes)
        ctx.grad_bits, ctx.bucket_size, ctx.group, ctx.stochastic = grad_bits, bucket_size, group, stochastic
        ctx.in_shape = input.shape
        ctx.gate_grad = gate_grad
        return out

    @staticmethod
    def backward(ctx, grad):
        gate, slots, output_index = ctx.saved_tensors
        out_splits, in_splits = ctx.splits
        T, k = gate.shape
        grad = grad.contiguous()
        gin = grad.new_empty(ctx.in_shape)
        # slot t*k + c goes back as grad[t] * gate[t, c], rounded to the dtype: scaled rows on send
        work = all_to_all_single(gin, grad, in_splits, out_splits, bits=ctx.grad_bits, bucket_size=ctx.bucket_size,
                                 group=ctx.group, async_op=True, stochastic=ctx.stochastic,
                                 input_index=torch.div(output_index, k, rounding_mode="floor"),
                                 input_scale=gate.reshape(-1)[output_index])
        # on the caller's stream, while the exchange runs on the group's
        if ctx.gate_grad == "fused":
            from .. import _C

            grad_gate = _C.combine_gate_grad(grad, slots, k)
        else:
            grad_gate = (grad.reshape(T, 1, -1).float() * slots.reshape(T, k, -1).float()).sum(-1)
        work.wait()
        return gin, grad_gate, None, None, None, None, None, None, None, None, None


def differentiable_all_to_all_combine(input: torch.Tensor, gate: torch.Tensor, output_index: torch.Tensor,
                                      output_split_sizes: Optional[Sequence[int]] = None,
                                      input_split_sizes: Optional[Sequence[int]] = None, bits: A2aBits = 8,
                                      grad_bits: Optional[A2aBits] = None, bucket_size: int = 512, group=None,
                                      stochastic: bool = False, gate_grad: str = "torch") -> torch.Tensor:
    """``all_to_all_combine`` that returns its ``[T, ...]`` output and has a backward pass, for the
    combine of an MoE layer. The gradients, from the slots the forward received:
      - input: ``grad_out[t] * gate[t, c]`` (one fp32 multiply, rounded to the dtype) for every slot
        ``t*k + c``, sent back by the routed ``all_to_all_single`` with ``input_index=output_index // k``
        and ``input_scale=gate.view(-1)[output_index]`` (splits swapped) at ``grad_bits`` (``None``:
        ``bits``), so no ``[T*k, ...]`` gradient is materialized;
      - gate: ``sum_h grad_out[t, h] * slots[t*k + c, h]`` in fp32. ``gate_grad="torch"`` computes it
        with torch's reduction, in torch's order. ``gate_grad="fused"`` reads ``grad_out`` and the slots
        once in one kernel, in a fixed order (DESIGN §2.13e): lane ``l = (h // V) % 32`` of a warp
        (``V`` = 16 bytes of the dtype) runs ``acc = fma(grad_out[t, h], slots[t*k + c, h], acc)`` from
        ``+0`` over its ``h`` in increasing order, then the 32 partial sums are added by an xor
        butterfly (16, 8, 4, 2, 1). The two differ in the last bits; any other value raises
        ``ValueError`` before the forward sends.
    The gate gradient runs on the caller's stream while the input gradient's exchange runs.
    """
    if gate_grad not in ("torch", "fused"):
        raise ValueError(f"cgx.differentiable_all_to_all_combine: gate_grad must be 'torch' or 'fused', got "
                         f"{gate_grad!r}")
    bits = _a2a_bits(bits, stochastic)
    gb = _a2a_bits(bits if grad_bits is None else grad_bits, stochastic)
    return _AllToAllCombine.apply(input, gate, output_index,
                                  None if output_split_sizes is None else _splits(output_split_sizes),
                                  None if input_split_sizes is None else _splits(input_split_sizes), bits, gb,
                                  int(bucket_size), group, bool(stochastic), gate_grad)


def _check_slot_index(input: torch.Tensor, slot_index: torch.Tensor) -> int:
    """``k``, the choices per token, if ``slot_index`` can be the slot index of
    ``differentiable_all_to_all_dispatch``; ValueError otherwise. The device check comes last."""
    api = "cgx.differentiable_all_to_all_dispatch"
    if slot_index.dtype != torch.int64 or slot_index.dim() != 1 or not slot_index.is_contiguous():
        raise ValueError(f"{api}: slot_index must be a contiguous int64 vector, got {slot_index.dtype} "
                         f"{list(slot_index.shape)}{'' if slot_index.is_contiguous() else ' (not contiguous)'}")
    T, n = int(input.shape[0]), int(slot_index.numel())
    if T < 1 or n % T != 0 or not 1 <= n // T <= 32:
        raise ValueError(f"{api}: slot_index must hold T * k entries with T = {T} tokens and k in 1..32, got {n}")
    if not slot_index.is_cuda or slot_index.device != input.device:
        raise ValueError(f"{api}: slot_index must be on the input's CUDA device, got {slot_index.device}")
    return n // T


class _AllToAllDispatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, slot_index, k, output_split_sizes, input_split_sizes, bits, grad_bits, bucket_size,
                group, stochastic, output_index, output_rows):
        ctx.slot_index, ctx.k = slot_index, k
        return _AllToAll.forward(ctx, input, output_split_sizes, input_split_sizes, bits, grad_bits, bucket_size,
                                 group, stochastic, torch.div(slot_index, k, rounding_mode="floor"), output_index,
                                 output_rows)

    @staticmethod
    def backward(ctx, grad):
        out_splits, in_splits = ctx.splits
        _, output_index = ctx.index
        grad = grad.contiguous()
        gin = grad.new_empty(ctx.in_shape)
        # the combine with unit gates: slot t*k + c comes back to row slot_index^-1, and each token's
        # k slots are summed in fp32 in choice order, rounded once
        unit = torch.ones(ctx.in_shape[0], ctx.k, dtype=torch.float32, device=grad.device)
        all_to_all_combine(gin, grad, unit, ctx.slot_index, in_splits, out_splits, bits=ctx.grad_bits,
                           bucket_size=ctx.bucket_size, group=ctx.group, stochastic=ctx.stochastic,
                           input_index=output_index)
        return gin, None, None, None, None, None, None, None, None, None, None, None


def differentiable_all_to_all_dispatch(input: torch.Tensor, slot_index: torch.Tensor,
                                       output_split_sizes: Optional[Sequence[int]] = None,
                                       input_split_sizes: Optional[Sequence[int]] = None, bits: A2aBits = 8,
                                       grad_bits: Optional[A2aBits] = None, bucket_size: int = 512, group=None,
                                       stochastic: bool = False, output_index: Optional[torch.Tensor] = None,
                                       output_rows: Optional[int] = None) -> torch.Tensor:
    """The token dispatch of an MoE layer, with a backward that sums each token's k gradients inside
    the exchange (DESIGN §2.13i).

    ``input`` holds ``T`` tokens. ``slot_index`` is a contiguous CUDA int64 permutation of ``[0, T*k)``
    (``1 <= k <= 32``), slot ``s = t*k + c`` being choice ``c`` of token ``t``, listed in the order the
    rows are sent (``argsort`` of the flattened destinations, say): sent row ``i`` is token
    ``slot_index[i] // k``. The forward is bit for bit ``differentiable_all_to_all_single(input, ...,
    input_index=slot_index // k, output_index=output_index, output_rows=output_rows)``.

    The backward is one ``all_to_all_combine`` with gates of one: the gradient travels back at
    ``grad_bits`` (``None``: ``bits``) with the splits swapped, gathered by ``output_index`` if the
    forward had one, returned row ``i`` lands in slot ``slot_index[i]``, and for every token ``t`` and
    element ``h``, with ``x_c`` the fp32 value of slot ``t*k + c``, ``acc = x_0``, then ``acc = acc + x_c``
    for ``c = 1 .. k-1`` in fp32, and ``grad_input[t, h] = acc`` rounded once to the dtype. A unit gate
    is exact (``1 * x = x``, ``fma(1, x, acc) = x + acc``), so this is that sum bit for bit. Compared
    with the ``index_add_`` backward of ``differentiable_all_to_all_single``, the order is fixed, so
    two runs give the same bits; bf16 and fp16 are rounded once instead of once per choice; and a token
    whose k gradients are all ``-0`` gets ``-0`` instead of ``+0`` (``index_add_`` starts from ``+0``).

    ``ValueError`` before the forward sends anything for a ``slot_index`` of the wrong dtype, device,
    layout or length, for ``output_index`` without ``output_rows``, and for an FP8 ``bits`` or
    ``grad_bits`` with ``stochastic=True``. A repeated slot is found by the kernel in the backward: its
    call fails with the combine's message, which names ``output_index`` (the combine's name for
    ``slot_index``), and the group refuses further collectives.
    """
    if output_index is not None and output_rows is None:
        raise ValueError("cgx.differentiable_all_to_all_dispatch: output_index needs output_rows")
    bits = _a2a_bits(bits, stochastic)
    gb = _a2a_bits(bits if grad_bits is None else grad_bits, stochastic)
    k = _check_slot_index(input, slot_index)
    return _AllToAllDispatch.apply(input, slot_index, k,
                                   None if output_split_sizes is None else _splits(output_split_sizes),
                                   None if input_split_sizes is None else _splits(input_split_sizes), bits, gb,
                                   int(bucket_size), group, bool(stochastic), output_index, output_rows)
