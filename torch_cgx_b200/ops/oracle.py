"""Pure-PyTorch/NumPy reference ("oracle") of the quantization numerics and of the
whole compressed allreduce, SURVEY.md §2.7 and DESIGN §2.3:

    unit_k = (max_k - min_k) * fp32(1 / (2^b - 1))
    q_i    = min(floor((x_i - min_k) * fp32(1 / unit_k) + r), 2^b - 1),  r = 0.5 ; unit_k < 1e-10 => 1/unit := 0
    x^_i   = min_k + unit_k * q_i

computed per bucket of ``bucket_size`` consecutive elements of each layer, all
arithmetic in fp32 with IEEE rules (fused multiply-adds emulated exactly in
fp64).  Non-finite values follow the specification: min/max propagate NaN, a
NaN ``t`` becomes the top level (the ``fminf`` of ``encode_level``) and
``unit * q + min`` follows IEEE (``inf * 0 = NaN``).

It is independent of the C++/CUDA numerics: the only native call is
``build_plan`` (which rank owns which block), and the plan is checked on its
own by the plan property tests.  The CPU simulators and every kernel are judged
against it.  Reference kernels: /root/reference/src/common/compression/
cuda_compression_operations.cu:68-153 (encode/decode/meta).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

EPS = 1e-10
MAX_BUCKET = 8192  # larger quantization buckets are clamped to this size (one block holds a bucket)
RAW_BITS = 32

_F32 = np.float32
_EPS32 = _F32(EPS)
_DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
# (mantissa bits, smallest normal exponent) of each output dtype: half-ulp of the final rounding
_DTYPE_FMT = {torch.float32: (23, -126), torch.float16: (10, -14), torch.bfloat16: (7, -126)}

Layer = Tuple[int, int, int, int]  # (elem_off, numel, bits, bucket_size)


# ---- fp32 arithmetic -----------------------------------------------------------------------
def _fma32_np(a, b, c) -> np.ndarray:
    """round_fp32(a*b + c) with a single rounding, for fp32 inputs (numpy arrays or scalars).

    The product is exact in fp64; the fp64 sum is exact up to a residual found with
    TwoSum. Rounding the fp64 sum to fp32 is then correct unless that sum lies exactly
    half way between two fp32 values and the residual is not zero: the residual then
    decides the direction (this is the double-rounding case).
    """
    a, b, c = (np.asarray(v, dtype=np.float64) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bv = s - p
        lo = (p - (s - bv)) + (c - bv)
        r = s.astype(_F32)
        fix = np.isfinite(s) & np.isfinite(r) & (lo != 0)
        if np.any(fix):
            r64 = r.astype(np.float64)
            d = s - r64
            away = np.nextafter(r, np.where(d > 0, _F32(np.inf), _F32(-np.inf)).astype(_F32))
            tie = (d != 0) & (s == (r64 + away.astype(np.float64)) * 0.5)
            take = fix & tie & (np.sign(lo) == np.sign(d))
            r = np.where(take, away, r)
    return r


def _fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """round_fp32(a*b + c) for fp32 tensors, correctly rounded (see ``_fma32_np``)."""
    return torch.from_numpy(np.ascontiguousarray(_fma32_np(a.double().numpy(), b.double().numpy(),
                                                           c.double().numpy())))


def _ordered(x: np.ndarray) -> np.ndarray:
    """fp32 -> int32 keys with the float order and -0 < +0 (what min.f32 / max.f32 use)."""
    k = x.view(np.int32)
    return k ^ ((k >> 31) & np.int32(0x7FFFFFFF))


def _from_ordered(k: np.ndarray) -> np.ndarray:
    return (k ^ ((k >> 31) & np.int32(0x7FFFFFFF))).astype(np.int32).view(_F32)


def _nan_minmax(b: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Per-row NaN-propagating (min, max) of a 2-D fp32 array, -0 < +0."""
    k = _ordered(np.ascontiguousarray(b))
    mn = _from_ordered(k.min(axis=1, keepdims=True))
    mx = _from_ordered(k.max(axis=1, keepdims=True))
    nan = np.isnan(b).any(axis=1, keepdims=True)
    return np.where(nan, _F32(np.nan), mn), np.where(nan, _F32(np.nan), mx)


def round_to_dtype(v: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    """fp32 values as they are after a store to / load from ``dtype`` (round to nearest even)."""
    v = np.ascontiguousarray(v, dtype=_F32)
    if dtype == torch.float32:
        return v
    return torch.from_numpy(v).to(dtype).float().numpy()


def _levels(bits: int) -> _F32:
    return _F32((1 << bits) - 1)


# ---- one quantization round -----------------------------------------------------------------
def _qdq_buckets(v: np.ndarray, bits: int, bucket: int):
    """Round trip of a flat fp32 array whose buckets start at index 0.

    Returns (decoded fp32, levels, per-element unit of its bucket)."""
    assert 1 <= bits <= 8 and bucket >= 1
    n = v.size
    if n == 0:
        e = np.zeros(0, _F32)
        return e, e.copy(), e.copy()
    nb = -(-n // bucket)
    pad = nb * bucket - n
    # pad with the last element: it lies in the last bucket, so its min and max do not change
    vp = np.concatenate([v, np.repeat(v[-1:], pad)]) if pad else v
    b = vp.reshape(nb, bucket)
    levels = _levels(bits)
    with np.errstate(all="ignore"):
        mn, mx = _nan_minmax(b)
        unit = (mx - mn) * (_F32(1.0) / levels)
        inv = np.where(unit < _EPS32, _F32(0.0), _F32(1.0) / unit).astype(_F32)
        t = _fma32_np(b - mn, inv, _F32(0.5))
        q = np.floor(np.fmin(t, levels)).astype(_F32)  # fmin: a NaN t becomes the top level
        dec = _fma32_np(unit, q, mn)
    unit_e = np.broadcast_to(unit, b.shape)
    return (dec.reshape(-1)[:n].astype(_F32), q.reshape(-1)[:n].astype(_F32),
            np.ascontiguousarray(unit_e).reshape(-1)[:n])


def quantize_dequantize(x: torch.Tensor, bits: int, bucket_size: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Deterministic max-min quantization round trip of a flat tensor (one layer).

    Returns ``(decoded fp32 values, integer levels)``; the decoded values are NOT
    yet rounded to the tensor dtype. ``bucket_size`` is used as given (no clamp).
    """
    assert 1 <= bits <= 8
    flat = x.detach().reshape(-1).float().cpu().numpy()
    dec, q, _ = _qdq_buckets(flat, bits, bucket_size)
    return torch.from_numpy(dec.copy()), torch.from_numpy(q.astype(np.int64))


def quantize_dequantize_like(x: torch.Tensor, bits: int, bucket_size: int) -> torch.Tensor:
    """Round trip with the result rounded to ``x.dtype`` and reshaped like ``x``."""
    dec, _ = quantize_dequantize(x, bits, bucket_size)
    return dec.to(x.dtype).view_as(x)


def error_bound(x: torch.Tensor, bits: int, bucket_size: int) -> float:
    """Worst-case absolute error of one deterministic quantization: unit/2 of the widest bucket."""
    flat = x.detach().reshape(-1).float().cpu()
    n = flat.numel()
    nb = (n + bucket_size - 1) // bucket_size
    worst = 0.0
    for k in range(nb):
        seg = flat[k * bucket_size : (k + 1) * bucket_size]
        worst = max(worst, float(seg.max() - seg.min()))
    return worst / ((1 << bits) - 1) / 2.0


# ---- layer tables -----------------------------------------------------------------------------
def effective_bucket(bucket: int) -> int:
    """The bucket size a layer is quantized with: at least 1, at most ``MAX_BUCKET``."""
    return min(max(1, int(bucket)), MAX_BUCKET)


def layer_segments(layers: Sequence[Layer], skip_incomplete: bool) -> List[Tuple[int, int, int, int]]:
    """(elem_off, n, bits, bucket) runs of the buffer; bits == RAW_BITS means uncompressed.

    A compressed layer's buckets start at its first element. With ``skip_incomplete`` the
    last partial bucket (counted with the requested, unclamped size) travels uncompressed."""
    out = []
    for off, n, bits, bucket in layers:
        off, n, bits = int(off), int(n), int(bits)
        if bits >= RAW_BITS:
            out.append((off, n, RAW_BITS, 0))
            continue
        req = max(1, int(bucket))
        main = n // req * req if skip_incomplete else n
        if main:
            out.append((off, main, bits, effective_bucket(req)))
        if n - main:
            out.append((off + main, n - main, RAW_BITS, 0))
    return out


def block_owners(layers: Sequence[Layer], numel: int, world: int, lanes: int, dtype: torch.dtype,
                 skip_incomplete: bool, min_lane_elems: int) -> np.ndarray:
    """Per element: the rank that owns (reduces) it in the SRA plan, -1 outside every layer."""
    from .. import _C

    plan = _C.build_plan([tuple(int(v) for v in l) for l in layers], world=world, lanes=lanes,
                         dtype=_DTYPE_CODE[dtype], skip_incomplete=skip_incomplete,
                         min_lane_elems=min_lane_elems)
    owner = np.full(numel, -1, np.int64)
    blocks = plan["blocks"].tolist()
    lf, G = plan["lane_first"], plan["lanes"]
    for k in range(world * G):
        for b in range(lf[k], lf[k + 1]):
            off, n = blocks[b][0], blocks[b][1]
            owner[off:off + n] = k // G
    return owner


def _prescale(world: int, average: bool) -> _F32:
    return _F32(1.0) / _F32(world) if average else _F32(1.0)


def _scaled_inputs(inputs: Sequence[torch.Tensor], ps: _F32) -> List[np.ndarray]:
    with np.errstate(all="ignore"):
        return [t.detach().reshape(-1).float().cpu().numpy() * ps for t in inputs]


def _contribution(v: np.ndarray, bits: int, bucket: int, dtype: torch.dtype) -> np.ndarray:
    """What a receiver decodes of one sent contribution: one quantization round, or the value
    rounded to the dtype for raw runs."""
    if bits >= RAW_BITS:
        return round_to_dtype(v, dtype)
    return _qdq_buckets(v, bits, bucket)[0]


def quantize_dequantize_layers(x: torch.Tensor, layers: Sequence[Layer], *, skip_incomplete: bool = False,
                               prescale: float = 1.0) -> torch.Tensor:
    """One quantize -> dequantize round trip of ``prescale * x`` through a layer table, in
    ``x.dtype`` (raw runs: the value rounded to the dtype). Elements outside every layer are 0,
    as in a freshly dequantized tensor."""
    v = _scaled_inputs([x], _F32(prescale))[0]
    out = np.zeros(v.size, _F32)
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        out[off:off + m] = _contribution(v[off:off + m], bits, bucket, x.dtype)
    return _to_tensors([out], x.dtype)[0].view_as(x)


def _to_tensors(outs: Sequence[np.ndarray], dtype: torch.dtype) -> List[torch.Tensor]:
    return [torch.from_numpy(np.ascontiguousarray(o, dtype=_F32)).to(dtype) for o in outs]


def _sra_acc(xs: Sequence[np.ndarray], sl: slice, own: np.ndarray, bits: int, bucket: int,
             dtype: torch.dtype) -> np.ndarray:
    """The owner's fp32 accumulator of one run of the SRA: its own value, then every peer's
    decoded contribution in rank order."""
    acc = np.choose(own, [x[sl] for x in xs]).astype(_F32)
    with np.errstate(all="ignore"):
        for q in range(len(xs)):
            acc = np.where(own != q, acc + _contribution(xs[q][sl], bits, bucket, dtype), acc)
    return acc


def sra_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, world: int | None = None,
                  lanes: int = 1, min_lane_elems: int = 2048, average: bool = False,
                  skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's result of the deterministic compressed SRA allreduce (DESIGN §2.3).

    For each bucket, the owner c (the rank whose chunk holds it) forms in fp32
        acc = prescale*x_c  (kept unquantized)  +  sum over q != c, in rank order, of Q(prescale*x_q)
    where Q is one quantization round with buckets counted from the layer start; the result
    is Q(acc), the owner's self-decoded copy, stored in the input dtype on every rank.
    Raw runs (uncompressed layers, skip_incomplete tails) replace Q by a rounding to the
    dtype, per peer contribution and once at the end. Elements outside every layer are kept.
    """
    W = len(inputs)
    assert world is None or world == W
    dtype = inputs[0].dtype
    n = inputs[0].numel()
    xs = _scaled_inputs(inputs, _prescale(W, average))
    owner = block_owners(layers, n, W, lanes, dtype, skip_incomplete, min_lane_elems)
    outs = [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        sl = slice(off, off + m)
        res = _contribution(_sra_acc(xs, sl, owner[sl], bits, bucket, dtype), bits, bucket, dtype)
        for o in outs:
            o[sl] = res
    return _to_tensors(outs, dtype)


def oneshot_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                      skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's result of the one-shot allreduce: each contribution, the own one included,
    is quantized once (raw runs: rounded to the dtype) and the decoded values are summed in
    fp32 in rank order starting from +0; no second quantization, one rounding to the dtype."""
    W = len(inputs)
    dtype = inputs[0].dtype
    xs = _scaled_inputs(inputs, _prescale(W, average))
    outs = [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        sl = slice(off, off + m)
        acc = np.zeros(m, _F32)
        with np.errstate(all="ignore"):
            for q in range(W):
                acc = acc + _contribution(xs[q][sl], bits, bucket, dtype)
        res = round_to_dtype(acc, dtype)
        for o in outs:
            o[sl] = res
    return _to_tensors(outs, dtype)


# ---- the generic reducers (reduce/reducers.cc): rank chunks of the lanes = 1 plan ------------------
GENERIC_MIN_LANE_ELEMS = 2048  # Reducer::plan_for: one lane per rank chunk, default min_lane_elems


def _quantized(v: np.ndarray, segs, dtype: torch.dtype) -> np.ndarray:
    """``_contribution`` of every layer run of a whole-buffer fp32 array, buckets counted from
    each run's start; elements outside every run are returned unchanged."""
    out = v.copy()
    for off, m, bits, bucket in segs:
        out[off:off + m] = _contribution(v[off:off + m], bits, bucket, dtype)
    return out


def _own_values(inputs: Sequence[torch.Tensor]) -> List[np.ndarray]:
    return [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]


def ring_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                   skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's result of the compressed Ring allreduce (``RingReducer``, deterministic rounding).

    Chunk c is rank c's chunk of the lanes = 1 plan. Rank r starts with acc_r = prescale*x_r in fp32.
    At hop s = 0 .. W-2 every rank r sends Q(acc_r) restricted to chunk (r - s) mod W to rank r+1,
    which adds the decoded values to its own accumulator in fp32. Chunk c is then complete on rank
    (c - 1) mod W; every rank ends with Q(acc_{(c-1) mod W}) on chunk c, stored in the dtype (at
    W = 1: Q(prescale*x)). Q is one quantization round with buckets counted from the layer start;
    raw runs replace it by a rounding to the dtype. Elements outside every layer are kept.
    """
    W = len(inputs)
    dtype = inputs[0].dtype
    n = inputs[0].numel()
    segs = layer_segments(layers, skip_incomplete)
    chunk = block_owners(layers, n, W, 1, dtype, skip_incomplete, GENERIC_MIN_LANE_ELEMS)
    acc = _scaled_inputs(inputs, _prescale(W, average))
    with np.errstate(all="ignore"):
        for s in range(W - 1):
            sent = [_quantized(a, segs, dtype) for a in acc]  # every rank sends before it adds
            for r in range(W):
                sel = chunk == (r - s) % W
                dst = acc[(r + 1) % W]
                dst[sel] = dst[sel] + sent[r][sel]
    outs = _own_values(inputs)
    for c in range(W):
        sel = chunk == c
        final = _quantized(acc[(c - 1) % W], segs, dtype)
        for o in outs:
            o[sel] = final[sel]
    return _to_tensors(outs, dtype)


def alltoall_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                       skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's result of the debug all-to-all allreduce (``AllToAllReducer``, deterministic):
    rank r keeps prescale*x_r unquantized and adds, in fp32 and in ascending rank order, every
    peer's Q(prescale*x_q); the sum is stored in the dtype once. The ranks' results differ.
    Elements outside every layer are kept."""
    W = len(inputs)
    dtype = inputs[0].dtype
    segs = layer_segments(layers, skip_incomplete)
    xs = _scaled_inputs(inputs, _prescale(W, average))
    qs = [_quantized(x, segs, dtype) for x in xs]
    outs = _own_values(inputs)
    with np.errstate(all="ignore"):
        for r in range(W):
            acc = xs[r].copy()
            for q in range(W):
                if q != r:
                    acc = acc + qs[q]
            for off, m, _, _ in segs:
                outs[r][off:off + m] = acc[off:off + m]
    return _to_tensors(outs, dtype)


def broadcast_compressed_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, root: int,
                                   skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's result of ``Reducer::broadcast_compressed``: one quantization round of the
    root's values (prescale 1, one chunk, buckets from the layer start; a ``skip_incomplete`` tail
    stays raw), the root included so that all ranks agree. Elements outside every layer keep each
    rank's own values. With one rank nothing is sent and the values are unchanged."""
    W = len(inputs)
    dtype = inputs[0].dtype
    outs = _own_values(inputs)
    if W > 1:
        segs = layer_segments(layers, skip_incomplete)
        q = _quantized(_own_values([inputs[root]])[0], segs, dtype)
        for o in outs:
            for off, m, _, _ in segs:
                o[off:off + m] = q[off:off + m]
    return _to_tensors(outs, dtype)


def _shards(inputs: Sequence[torch.Tensor], r: int) -> List[torch.Tensor]:
    W = len(inputs)
    n = inputs[0].numel()
    assert n % W == 0, "a reduce-scatter input holds world x shard elements"
    S = n // W
    return [t.detach().reshape(-1)[r * S:(r + 1) * S] for t in inputs]


def reduce_scatter_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *,
                             world: int | None = None, average: bool = False,
                             skip_incomplete: bool = False) -> List[torch.Tensor]:
    """Every rank's output of the compressed reduce-scatter (deterministic rounding).

    ``inputs[r]`` holds W shards of S elements; ``shard_layers`` is one shard's table (offsets from
    the shard start), the same for every shard, so buckets are counted from each shard's start.
    Rank r receives, per element of shard r, in fp32:
        prescale*x_r  (kept unquantized)  +  sum over q != r, in rank order, of Q(prescale*x_q)
    rounded once to the dtype: the SRA's phase-B accumulator without the requantization. Raw runs
    round each peer contribution to the dtype. Elements outside every layer are 0.
    """
    W = len(inputs)
    assert world is None or world == W
    dtype = inputs[0].dtype
    ps = _prescale(W, average)
    outs = []
    for r in range(W):
        xs = _scaled_inputs(_shards(inputs, r), ps)
        out = np.zeros(xs[0].size, _F32)
        for off, m, bits, bucket in layer_segments(shard_layers, skip_incomplete):
            sl = slice(off, off + m)
            out[sl] = _sra_acc(xs, sl, np.full(m, r), bits, bucket, dtype)
        outs.append(out)
    return _to_tensors(outs, dtype)


def all_gather_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer]) -> torch.Tensor:
    """Every rank's output of the compressed all-gather (deterministic rounding): the concatenation
    over q of ``quantize_dequantize_layers(inputs[q], shard_layers)``. ``shard_layers`` is one
    shard's table (offsets from the shard start), so buckets are counted from each shard's start;
    the owner's shard is quantized like every other. Raw runs are the value in the dtype."""
    return torch.cat([quantize_dequantize_layers(t.detach().reshape(-1).cpu(), shard_layers) for t in inputs])


def reduce_scatter_exact_and_bound(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *,
                                   average: bool = False, skip_incomplete: bool = False,
                                   stochastic: bool = False) -> List[Tuple[np.ndarray, np.ndarray]]:
    """Per rank r: the fp64 exact sum of shard r and a per-element bound on the reduce-scatter's
    error (``exact_sum_and_bound`` of one quantization round, rank r's own values exact)."""
    return [exact_sum_and_bound(_shards(inputs, r), shard_layers, average=average, skip_incomplete=skip_incomplete,
                                stochastic=stochastic, oneshot=True, exact_rank=r) for r in range(len(inputs))]


def _half_ulp(v: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    """Half an ulp of ``dtype`` at magnitude |v| (subnormal spacing below the normal range)."""
    mant, emin = _DTYPE_FMT[dtype]
    with np.errstate(all="ignore"):
        _, e = np.frexp(np.abs(v))
        e = np.maximum(e - 1, emin)
        return np.ldexp(1.0, e - mant - 1)


def _round_err(unit: np.ndarray, h: float, levels: float) -> np.ndarray:
    """Error of one quantization round: h units, or the whole span of a bucket whose unit is
    below kQuantEps (all its levels are 0, it decodes to its min)."""
    return np.where(unit < float(_EPS32), unit * levels, h * unit)


def exact_sum_and_bound(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, lanes: int = 1,
                        min_lane_elems: int = 2048, average: bool = False, skip_incomplete: bool = False,
                        stochastic: bool = False, oneshot: bool = False,
                        exact_rank: int | None = None) -> Tuple[np.ndarray, np.ndarray]:
    """fp64 exact sum  sum_q prescale*x_q  and a per-element bound on |result - exact|.

    Compressed runs: for every quantized contribution unit/2 of its bucket (a full unit with
    stochastic rounding; the whole span max - min when unit < kQuantEps); for the SRA the
    owner's contribution is exact and the requantized sum adds the same for its own unit (with
    stochastic rounding, for a bound of that unit). Every run adds the
    fp32 slack of the prescale products, decodes and the accumulation, and half an ulp of
    the output dtype; raw runs add half an ulp of the dtype per rounded contribution.
    The bound is meaningful where the exact sum and the inputs are finite. Elements outside
    every layer (each rank keeps its own) have a NaN exact sum.
    ``oneshot`` with ``exact_rank``: that rank's contribution is added unquantized (the
    compressed reduce-scatter, one quantization round per peer).
    """
    W = len(inputs)
    dtype = inputs[0].dtype
    n = inputs[0].numel()
    ps = _prescale(W, average)
    xs = _scaled_inputs(inputs, ps)
    x64 = [t.detach().reshape(-1).double().cpu().numpy() for t in inputs]
    total = np.zeros(n)
    for x in x64:
        total += float(ps) * x
    exact = np.full(n, np.nan)
    bound = np.full(n, np.nan)
    owner = None if oneshot else block_owners(layers, n, W, lanes, dtype, skip_incomplete, min_lane_elems)
    h = 1.0 if stochastic else 0.5
    u32 = 2.0 ** -24    # relative error of one fp32 rounding ...
    tiny = 2.0 ** -150  # ... plus this absolute one in the subnormal range

    def _sent(q: int, sl: slice) -> np.ndarray:  # elements where rank q's contribution is quantized
        if oneshot:
            return np.full(sl.stop - sl.start, q != exact_rank)
        return owner[sl] != q

    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        sl = slice(off, off + m)
        exact[sl] = total[sl]
        mag = sum(np.abs(x[sl].astype(np.float64)) for x in xs)
        if bits >= RAW_BITS:
            err = np.zeros(m)
            for q in range(W):
                hu = _half_ulp(xs[q][sl], dtype) if dtype != torch.float32 else 0.0
                err += np.where(_sent(q, sl), hu, 0.0)
            b = err + (W + 2) * (u32 * (mag + err) + tiny)
        else:
            levels = float((1 << bits) - 1)
            qerr = np.zeros(m)
            span = np.zeros(m)
            for q in range(W):
                unit = _qdq_buckets(xs[q][sl], bits, bucket)[2].astype(np.float64)
                sent = _sent(q, sl)
                qerr += np.where(sent, _round_err(unit, h, levels), 0.0)
                span += unit * levels
            b = qerr
            if not oneshot:
                acc = _sra_acc(xs, sl, owner[sl], bits, bucket, dtype)
                unit_s = _qdq_buckets(acc, bits, bucket)[2].astype(np.float64)
                if stochastic:
                    # the stochastic sum differs from the deterministic one by at most qerr per
                    # element, so its bucket span by at most twice the largest qerr of the bucket
                    nb = -(-m // bucket)
                    pad = nb * bucket - m
                    qe = np.concatenate([qerr, np.zeros(pad)]).reshape(nb, bucket).max(axis=1)
                    unit_s = unit_s + np.repeat(2.0 * qe / levels, bucket)[:m] * (1 + 1e-6)
                b = b + _round_err(unit_s, h, levels)
                span = span + unit_s * levels
            b = b + (W + 4) * (u32 * (mag + span + np.abs(exact[sl])) + tiny)
        b = b + _half_ulp(np.abs(exact[sl]) + b, dtype)
        bound[sl] = b
    return exact, bound
