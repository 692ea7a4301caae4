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


def _prescale(world: int, average: bool, prescale: float | None = None) -> _F32:
    """The factor every contribution is multiplied by first: ``prescale`` when given, else 1/world
    when averaging, else 1."""
    if prescale is not None:
        return _F32(prescale)
    return _F32(1.0) / _F32(world) if average else _F32(1.0)


def _scaled_inputs(inputs: Sequence[torch.Tensor], ps: _F32) -> List[np.ndarray]:
    with np.errstate(all="ignore"):
        return [t.detach().reshape(-1).float().cpu().numpy() * ps for t in inputs]


def _contribution(v: np.ndarray, bits: int, bucket: int, dtype: torch.dtype, fmt: str | None = None,
                  sr_key: Tuple[int, int, int, int] | None = None) -> np.ndarray:
    """What a receiver decodes of one sent contribution: one quantization round (in the FP8 format
    ``fmt`` when given), or the value rounded to the dtype for raw runs. An ``_sr`` format needs
    ``sr_key = (seed, seq, stream, first_elem)``: the key and the element index of ``v[0]``."""
    if bits >= RAW_BITS:
        return round_to_dtype(v, dtype)
    if fmt in FP8_SR_FORMATS:
        if sr_key is None:
            raise ValueError(f"the FP8 format {fmt!r} rounds stochastically: this reference has no random stream")
        return _fp8_sr_qdq_buckets(v, fmt, bucket, _sr_words(*sr_key, v.size, bucket))
    if fmt is not None:
        return _fp8_qdq_buckets(v, fmt, bucket)
    return _qdq_buckets(v, bits, bucket)[0]


def quantize_dequantize_layers(x: torch.Tensor, layers: Sequence[Layer], *, skip_incomplete: bool = False,
                               prescale: float = 1.0, fmt: str | None = None,
                               sr_stream: Tuple[int, int, int, int] | None = None) -> torch.Tensor:
    """One quantize -> dequantize round trip of ``prescale * x`` through a layer table, in
    ``x.dtype`` (raw runs: the value rounded to the dtype). Elements outside every layer are 0,
    as in a freshly dequantized tensor. ``fmt`` (a name of ``FP8_FORMATS``): the compressed layers (bits 8)
    take the FP8 round trip of ``fp8_quantize_dequantize`` instead of max-min's. An ``_sr`` format
    needs ``sr_stream = (seed, seq, stream, base)``: element i of ``x`` has element index base + i."""
    _check_fp8_table(layers, fmt)
    v = _scaled_inputs([x], _F32(prescale))[0]
    out = np.zeros(v.size, _F32)
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        key = None if sr_stream is None else (*sr_stream[:3], sr_stream[3] + off)
        out[off:off + m] = _contribution(v[off:off + m], bits, bucket, x.dtype, fmt, key)
    return _to_tensors([out], x.dtype)[0].view_as(x)


def _to_tensors(outs: Sequence[np.ndarray], dtype: torch.dtype) -> List[torch.Tensor]:
    return [torch.from_numpy(np.ascontiguousarray(o, dtype=_F32)).to(dtype) for o in outs]


def _sra_acc(xs: Sequence[np.ndarray], sl: slice, own: np.ndarray, bits: int, bucket: int,
             dtype: torch.dtype, fmt: str | None = None) -> np.ndarray:
    """The owner's fp32 accumulator of one run of the SRA: its own value, then every peer's
    decoded contribution in rank order (each an fp32 add of its own)."""
    acc = np.choose(own, [x[sl] for x in xs]).astype(_F32)
    with np.errstate(all="ignore"):
        for q in range(len(xs)):
            acc = np.where(own != q, acc + _contribution(xs[q][sl], bits, bucket, dtype, fmt), acc)
    return acc


def _check_fp8_table(layers: Sequence[Layer], fmt: str | None) -> None:
    if fmt is None:
        return
    if fmt not in FP8_FORMATS and fmt not in FP8_SR_FORMATS:
        raise ValueError(f"unknown FP8 format {fmt!r}")
    for l in layers:
        if int(l[2]) != 8 and int(l[2]) < RAW_BITS:
            raise ValueError(f"an FP8 format needs layers of bits 8 or {RAW_BITS}, got {l[2]}")


def sra_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, world: int | None = None,
                  lanes: int = 1, min_lane_elems: int = 2048, average: bool = False,
                  skip_incomplete: bool = False, prescale: float | None = None,
                  fmt: str | None = None) -> List[torch.Tensor]:
    """Every rank's result of the deterministic compressed SRA allreduce (DESIGN §2.3).

    For each bucket, the owner c (the rank whose chunk holds it) forms in fp32
        acc = prescale*x_c  (kept unquantized)  +  sum over q != c, in rank order, of Q(prescale*x_q)
    where Q is one quantization round with buckets counted from the layer start; the result
    is Q(acc), the owner's self-decoded copy, stored in the input dtype on every rank.
    Raw runs (uncompressed layers, skip_incomplete tails) replace Q by a rounding to the
    dtype, per peer contribution and once at the end. Elements outside every layer are kept.
    ``fmt`` (a name of ``FP8_FORMATS``): Q is the FP8 round trip of ``fp8_quantize_dequantize``, for the
    peers' contributions and for the fp32 sum alike; the table may hold bits 8 and 32 only.
    """
    _check_fp8_table(layers, fmt)
    W = len(inputs)
    assert world is None or world == W
    dtype = inputs[0].dtype
    n = inputs[0].numel()
    xs = _scaled_inputs(inputs, _prescale(W, average, prescale))
    owner = block_owners(layers, n, W, lanes, dtype, skip_incomplete, min_lane_elems)
    outs = [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        sl = slice(off, off + m)
        res = _contribution(_sra_acc(xs, sl, owner[sl], bits, bucket, dtype, fmt), bits, bucket, dtype, fmt)
        for o in outs:
            o[sl] = res
    return _to_tensors(outs, dtype)


def oneshot_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                      skip_incomplete: bool = False, prescale: float | None = None,
                      fmt: str | None = None, seed: int = 0, seq: int = 0) -> List[torch.Tensor]:
    """Every rank's result of the one-shot allreduce: each contribution, the own one included,
    is quantized once (raw runs: rounded to the dtype) and the decoded values are summed in
    fp32 in rank order starting from +0; no second quantization, one rounding to the dtype.
    ``fmt``: the contributions take the FP8 round trip instead (as in ``sra_reference``); an ``_sr``
    format rounds rank q's with stream q * 2 of (``seed``, ``seq``), elements indexed from the buffer start."""
    _check_fp8_table(layers, fmt)
    W = len(inputs)
    dtype = inputs[0].dtype
    xs = _scaled_inputs(inputs, _prescale(W, average, prescale))
    outs = [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]
    for off, m, bits, bucket in layer_segments(layers, skip_incomplete):
        sl = slice(off, off + m)
        acc = np.zeros(m, _F32)
        with np.errstate(all="ignore"):
            for q in range(W):
                acc = acc + _contribution(xs[q][sl], bits, bucket, dtype, fmt, (seed, seq, 2 * q, off))
        res = round_to_dtype(acc, dtype)
        for o in outs:
            o[sl] = res
    return _to_tensors(outs, dtype)


# ---- the generic reducers (reduce/reducers.cc): rank chunks of the lanes = 1 plan ------------------
GENERIC_MIN_LANE_ELEMS = 2048  # Reducer::plan_for: one lane per rank chunk, default min_lane_elems


def _quantized(v: np.ndarray, segs, dtype: torch.dtype, fmt: str | None = None) -> np.ndarray:
    """``_contribution`` of every layer run of a whole-buffer fp32 array, buckets counted from
    each run's start; elements outside every run are returned unchanged."""
    out = v.copy()
    for off, m, bits, bucket in segs:
        out[off:off + m] = _contribution(v[off:off + m], bits, bucket, dtype, fmt)
    return out


def _own_values(inputs: Sequence[torch.Tensor]) -> List[np.ndarray]:
    return [t.detach().reshape(-1).float().cpu().numpy().copy() for t in inputs]


def ring_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                   skip_incomplete: bool = False, prescale: float | None = None,
                   fmt: str | None = None) -> List[torch.Tensor]:
    """Every rank's result of the compressed Ring allreduce (``RingReducer``, deterministic rounding).

    Chunk c is rank c's chunk of the lanes = 1 plan. Rank r starts with acc_r = prescale*x_r in fp32.
    At hop s = 0 .. W-2 every rank r sends Q(acc_r) restricted to chunk (r - s) mod W to rank r+1,
    which adds the decoded values to its own accumulator in fp32. Chunk c is then complete on rank
    (c - 1) mod W; every rank ends with Q(acc_{(c-1) mod W}) on chunk c, stored in the dtype (at
    W = 1: Q(prescale*x)). Q is one quantization round with buckets counted from the layer start;
    raw runs replace it by a rounding to the dtype. Elements outside every layer are kept.
    ``fmt``: Q is the FP8 round trip (as in ``sra_reference``).
    """
    _check_fp8_table(layers, fmt)
    W = len(inputs)
    dtype = inputs[0].dtype
    n = inputs[0].numel()
    segs = layer_segments(layers, skip_incomplete)
    chunk = block_owners(layers, n, W, 1, dtype, skip_incomplete, GENERIC_MIN_LANE_ELEMS)
    acc = _scaled_inputs(inputs, _prescale(W, average, prescale))
    with np.errstate(all="ignore"):
        for s in range(W - 1):
            sent = [_quantized(a, segs, dtype, fmt) for a in acc]  # every rank sends before it adds
            for r in range(W):
                sel = chunk == (r - s) % W
                dst = acc[(r + 1) % W]
                dst[sel] = dst[sel] + sent[r][sel]
    outs = _own_values(inputs)
    for c in range(W):
        sel = chunk == c
        final = _quantized(acc[(c - 1) % W], segs, dtype, fmt)
        for o in outs:
            o[sel] = final[sel]
    return _to_tensors(outs, dtype)


def alltoall_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, average: bool = False,
                       skip_incomplete: bool = False, prescale: float | None = None) -> List[torch.Tensor]:
    """Every rank's result of the debug all-to-all allreduce (``AllToAllReducer``, deterministic):
    rank r keeps prescale*x_r unquantized and adds, in fp32 and in ascending rank order, every
    peer's Q(prescale*x_q); the sum is stored in the dtype once. The ranks' results differ.
    Elements outside every layer are kept."""
    W = len(inputs)
    dtype = inputs[0].dtype
    segs = layer_segments(layers, skip_incomplete)
    xs = _scaled_inputs(inputs, _prescale(W, average, prescale))
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
                                   skip_incomplete: bool = False, fmt: str | None = None) -> List[torch.Tensor]:
    """Every rank's result of ``Reducer::broadcast_compressed``: one quantization round of the
    root's values (prescale 1, one chunk, buckets from the layer start; a ``skip_incomplete`` tail
    stays raw), the root included so that all ranks agree. Elements outside every layer keep each
    rank's own values. With one rank nothing is sent and the values are unchanged. ``fmt``: the
    FP8 round trip instead of max-min's."""
    _check_fp8_table(layers, fmt)
    W = len(inputs)
    dtype = inputs[0].dtype
    outs = _own_values(inputs)
    if W > 1:
        segs = layer_segments(layers, skip_incomplete)
        q = _quantized(_own_values([inputs[root]])[0], segs, dtype, fmt)
        for o in outs:
            for off, m, _, _ in segs:
                o[off:off + m] = q[off:off + m]
    return _to_tensors(outs, dtype)


# ---- the allreduce engine (engine/engine.cc): stages composed from the references above ------------
ENGINE_DEFAULTS = dict(fusion_bytes=64 << 20, oneshot_max_bytes=2 << 20, min_lane_elems=4096, min_compress_elems=16,
                       inner_reduction="SRA", cross_reduction="RING", intra_broadcast=True, intra_compress=True,
                       dummy_compression=False, overlap_lanes=64, p2p=True)
ONESHOT_MAX_EGRESS = 4 << 20  # a one-shot rank pushes its packed image to every peer: at most this many bytes
_U32 = 0xFFFFFFFF
_ELSIZE = {torch.float32: 4, torch.float16: 2, torch.bfloat16: 2}
ENGINE_PERTURBATIONS = ("prescale_local", "raw_broadcast", "cross_seq_unmarked", "oneshot_shifted")


def _generic_allreduce(kind, ins, layers, *, prescale, skip_incomplete, stochastic, seed, seq, fmt=None):
    """One generic reducer's allreduce over ``ins`` (one tensor per rank of its group)."""
    if stochastic:
        from .. import _C

        out = [t.clone() for t in ins]
        _C.LocalReducerGroup(len(ins), kind, 20_000).allreduce(out, layers, False, skip_incomplete, True, seed, seq,
                                                               prescale=float(prescale))
        return out
    kw = dict(skip_incomplete=skip_incomplete, prescale=prescale)
    if fmt is not None:
        if kind == "ALLTOALL":
            raise ValueError("the debug all-to-all reduction has no FP8 formats")
        kw["fmt"] = fmt
    if kind == "SRA":
        return sra_reference(ins, layers, lanes=1, min_lane_elems=GENERIC_MIN_LANE_ELEMS, **kw)
    if kind == "RING":
        return ring_reference(ins, layers, **kw)
    return alltoall_reference(ins, layers, **kw)


def engine_reference(inputs: Sequence[torch.Tensor], layers: Sequence[Layer], *, local_size: int, config: dict,
                     lanes: int, slot_bytes: Tuple[int, int] = (0, 0), average: bool = False, call_seq: int = 1,
                     cuda: bool = True, overlapped: bool = False, skip_incomplete: bool = False,
                     stochastic: bool = False, seed: int = 0, perturb: str | None = None, fmt: str | None = None):
    """Every rank's result of one ``AllreduceEngine`` allreduce over ``layers`` and the stages each
    rank issues, ``(outputs, stages)``; ``stages[r]`` is a list of dicts (kind, layers, lanes, numel,
    seed, seq, stochastic, scale) in the order rank r issues them.

    The stages follow engine.cc, written out here from the configuration (keys of
    ``ENGINE_DEFAULTS``) rather than read from a run. ``local_size`` consecutive ranks form a node.
    Layers are cut into fusion groups (``split_for_fusion``); group g of call ``call_seq`` runs with
    RNG sequence ``call_seq << 4 | (g & 15)`` and, per group:
      1. inside the node (skipped when nodes have one rank and there are several nodes): with every
         rank's contribution prescaled by 1/W when averaging. With ``cuda`` and heaps (``p2p``), and
         the SRA or no intra-node reducer, the fused kernel: the one-shot kernel when the group
         fits ``oneshot_max_bytes``, its single-chunk plan the one-shot slot and its egress 4 MiB;
         otherwise the three-phase SRA of each piece of the group, halving (by layers, then at
         bucket boundaries) every piece whose plan does not fit the slot, pieces numbered in launch
         order into the low 3 bits of ``seq << 3``. Else the generic ``inner_reduction``. With
         several nodes and no ``intra_compress`` this stage sends every layer raw.
      2. across nodes, between the ranks of one local rank, with ``seq ^ 0x40000000`` and scale 1
         (1/W when nodes have one rank): the node leaders only with ``intra_broadcast``, which then
         hand the result to their node, compressed from root 0 with ``seq ^ 0x20000000`` when the
         intra-node stage compresses and the group has a compressed layer, else as raw bytes of
         the group's span.
    ``stochastic`` composes the CPU simulators (``C.sra_simulate``, ``C.oneshot_simulate`` and
    ``C.LocalReducerGroup``) with these sequence numbers instead of the deterministic references.
    ``perturb`` (one of ``ENGINE_PERTURBATIONS``) switches on a wrong semantics, for the tests that
    show the reference tells it apart.
    ``fmt`` (a name of ``FP8_FORMATS``): every compressed stage uses that FP8 format (deterministic only).
    """
    from .. import _C

    _check_fp8_table(layers, fmt)
    if fmt is not None and stochastic:
        raise ValueError("the FP8 formats round to nearest only")

    cfg = dict(ENGINE_DEFAULTS, **config)
    W, L = len(inputs), local_size
    nodes = W // L
    multi = nodes > 1
    dtype = inputs[0].dtype
    es = _ELSIZE[dtype]
    dt = _DTYPE_CODE[dtype]
    layers = [tuple(int(v) for v in l) for l in layers]
    if cfg["dummy_compression"]:
        layers = [(o, n, RAW_BITS, b) for o, n, _, b in layers]
    ps = _prescale(W, average)
    ps1 = _prescale(L, average) if perturb == "prescale_local" else ps
    cap = cfg["overlap_lanes"] if overlapped else 0
    plan_lanes = cap if 0 < cap < lanes else lanes
    slot, os_slot = slot_bytes
    fused = cuda and cfg["p2p"] and (cfg["inner_reduction"] == "SRA" or L == 1)
    groups = _C.split_for_fusion(layers, es, cfg["fusion_bytes"])
    oneshot_limit = cfg["oneshot_max_bytes"]
    if perturb == "oneshot_shifted":  # the largest group that takes the one-shot kernel takes the SRA instead
        fits = [sum(l[1] for l in g) * es for g in groups if sum(l[1] for l in g) * es <= oneshot_limit]
        oneshot_limit = max(fits) - 1 if fits else oneshot_limit
    state = [t.detach().reshape(-1).cpu().clone() for t in inputs]
    stages = [[] for _ in range(W)]

    def log(ranks, kind, ls, seq, scale, lanes_=0, numel=None):
        for r in ranks:
            stages[r].append(dict(kind=kind, layers=[tuple(l) for l in ls], lanes=lanes_,
                                  numel=sum(l[1] for l in ls) if numel is None else numel, seed=seed,
                                  seq=seq & _U32, stochastic=stochastic, scale=float(scale)))

    def node_ranks(nd):
        return list(range(nd * L, (nd + 1) * L))

    def setvals(ranks, outs):
        for r, o in zip(ranks, outs):
            state[r] = o.reshape(-1).clone()

    def fused_pieces(gl):
        """[(kind, layers, plan)] of one group's fused launches, in launch order."""
        n = sum(l[1] for l in gl)
        if L > 1 and oneshot_limit > 0 and n * es <= oneshot_limit:
            p = _C.build_plan(gl, world=1, lanes=plan_lanes, dtype=dt, skip_incomplete=skip_incomplete,
                              min_lane_elems=cfg["min_lane_elems"])
            if p["max_chunk_wire"] <= os_slot and p["total_wire"] * (L - 1) <= ONESHOT_MAX_EGRESS:
                return [("oneshot", gl, p)]
        out, todo = [], [list(gl)]
        while todo:
            cur = todo.pop()
            p = _C.build_plan(cur, world=L, lanes=plan_lanes, dtype=dt, skip_incomplete=skip_incomplete,
                              min_lane_elems=cfg["min_lane_elems"])
            if p["max_chunk_wire"] <= slot:
                out.append(("sra", cur, p))
                continue
            if len(cur) > 1:
                h = len(cur) // 2
                todo += [cur[h:], cur[:h]]
                continue
            off, m, bits, bucket = cur[0]
            gran = 512 if bits >= RAW_BITS else max(1, bucket)
            assert m > gran, "fusion buffer too small for a single quantization bucket"
            h = max(gran, (m // 2) // gran * gran)
            todo += [[(off + h, m - h, bits, bucket)], [(off, h, bits, bucket)]]
        return out

    for g, group in enumerate(groups):
        seq = ((call_seq << 4) | (g & 15)) & _U32
        intra = [(o, n, RAW_BITS, b) for o, n, _, b in group] if (multi and not cfg["intra_compress"]) else group
        if L > 1 or not multi:
            for nd in range(nodes):
                rk = node_ranks(nd)
                ins = [state[r] for r in rk]
                if fused:
                    for sub, (kind, gl, p) in enumerate(fused_pieces(intra)):
                        s3 = ((seq << 3) | (sub & 7)) & _U32
                        log(rk, kind, gl, s3, ps1, p["lanes"], p["numel"])
                        if stochastic:
                            outs = [t.clone() for t in ins]
                            sim = _C.oneshot_simulate if kind == "oneshot" else _C.sra_simulate
                            sim(outs, gl, plan_lanes, False, skip_incomplete, True, seed, s3, cfg["min_lane_elems"],
                                prescale=float(ps1))
                        elif kind == "oneshot":
                            outs = oneshot_reference(ins, gl, skip_incomplete=skip_incomplete, prescale=ps1, fmt=fmt)
                        else:
                            outs = sra_reference(ins, gl, lanes=plan_lanes, min_lane_elems=cfg["min_lane_elems"],
                                                 skip_incomplete=skip_incomplete, prescale=ps1, fmt=fmt)
                        ins = [o.reshape(-1) for o in outs]
                else:
                    log(rk, "generic_intra", intra, seq, ps1)
                    ins = _generic_allreduce(cfg["inner_reduction"], ins, intra, prescale=ps1,
                                             skip_incomplete=skip_incomplete, stochastic=stochastic, seed=seed,
                                             seq=seq, fmt=fmt)
                setvals(rk, ins)
        if not multi:
            continue
        cseq = seq if perturb == "cross_seq_unmarked" else seq ^ 0x40000000
        cscale = _F32(1.0) if L > 1 else ps
        leaders_only = cfg["intra_broadcast"] and L > 1
        for lr in range(1 if leaders_only else L):
            rk = [nd * L + lr for nd in range(nodes)]
            log(rk, "cross", group, cseq, cscale)
            setvals(rk, _generic_allreduce(cfg["cross_reduction"], [state[r] for r in rk], group, prescale=cscale,
                                           skip_incomplete=skip_incomplete, stochastic=stochastic, seed=seed,
                                           seq=cseq, fmt=fmt))
        if not leaders_only:
            continue
        compressed = (cfg["intra_compress"] and any(l[2] < RAW_BITS for l in group)
                      and perturb != "raw_broadcast")
        for nd in range(nodes):
            rk = node_ranks(nd)
            if compressed:
                bseq = seq ^ 0x20000000
                log(rk, "bcast_compressed", group, bseq, 1.0)
                ins = [state[r] for r in rk]
                if stochastic:
                    outs = [t.clone() for t in ins]
                    _C.LocalReducerGroup(L, "SRA", 20_000).broadcast_compressed(outs, group, 0, skip_incomplete,
                                                                                True, seed, bseq)
                else:
                    outs = broadcast_compressed_reference(ins, group, root=0, skip_incomplete=skip_incomplete,
                                                          fmt=fmt)
                setvals(rk, outs)
            else:
                log(rk, "bcast_raw", group, seq, 1.0)
                lo = min(l[0] for l in group)
                hi = max(l[0] + l[1] for l in group)
                for r in rk[1:]:
                    state[r][lo:hi] = state[rk[0]][lo:hi]
    return [s.view_as(t).to(t.dtype) for s, t in zip(state, inputs)], stages


def _shards(inputs: Sequence[torch.Tensor], r: int) -> List[torch.Tensor]:
    W = len(inputs)
    n = inputs[0].numel()
    assert n % W == 0, "a reduce-scatter input holds world x shard elements"
    S = n // W
    return [t.detach().reshape(-1)[r * S:(r + 1) * S] for t in inputs]


def reduce_scatter_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *,
                             world: int | None = None, average: bool = False,
                             skip_incomplete: bool = False, prescale: float | None = None,
                             fmt: str | None = None) -> List[torch.Tensor]:
    """Every rank's output of the compressed reduce-scatter (deterministic rounding).

    ``inputs[r]`` holds W shards of S elements; ``shard_layers`` is one shard's table (offsets from
    the shard start), the same for every shard, so buckets are counted from each shard's start.
    Rank r receives, per element of shard r, in fp32:
        prescale*x_r  (kept unquantized)  +  sum over q != r, in rank order, of Q(prescale*x_q)
    rounded once to the dtype: the SRA's phase-B accumulator without the requantization. Raw runs
    round each peer contribution to the dtype. Elements outside every layer are 0. The prescale is
    ``prescale`` when given, else 1/W when averaging, else 1. ``fmt`` (a name of ``FP8_FORMATS``): Q is
    the FP8 round trip (``fp8_quantize_dequantize`` of the prescaled values), and the table's
    compressed layers have bits 8.
    """
    _check_fp8_table(shard_layers, fmt)
    W = len(inputs)
    assert world is None or world == W
    dtype = inputs[0].dtype
    ps = _prescale(W, average, prescale)
    outs = []
    for r in range(W):
        xs = _scaled_inputs(_shards(inputs, r), ps)
        out = np.zeros(xs[0].size, _F32)
        for off, m, bits, bucket in layer_segments(shard_layers, skip_incomplete):
            sl = slice(off, off + m)
            out[sl] = _sra_acc(xs, sl, np.full(m, r), bits, bucket, dtype, fmt)
        outs.append(out)
    return _to_tensors(outs, dtype)


def all_gather_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer],
                         fmt: str | None = None, seed: int = 0, seq: int = 0) -> torch.Tensor:
    """Every rank's output of the compressed all-gather (deterministic rounding): the concatenation
    over q of ``quantize_dequantize_layers(inputs[q], shard_layers, fmt=fmt)``. ``shard_layers`` is
    one shard's table (offsets from the shard start), so buckets are counted from each shard's
    start; the owner's shard is quantized like every other. Raw runs are the value in the dtype. An
    ``_sr`` format rounds shard q with stream q * 2 + 1 of (``seed``, ``seq``), its element i having
    index q * S + i (S the shard's size), as the all-gather publishes it."""
    return torch.cat([quantize_dequantize_layers(t.detach().reshape(-1).cpu(), shard_layers, fmt=fmt,
                                                 sr_stream=(seed, seq, 2 * q + 1, q * t.numel()))
                      for q, t in enumerate(inputs)])


# ---- FP8 wire formats of the all-to-all (common/quant_math.h, DESIGN §2.13b) ------------------------
# name -> (torch dtype, largest finite value). The "_pow2" formats have their base format's codes
# with a power-of-two unit per bucket (DESIGN §2.13g).
FP8_FORMATS = {"e4m3": (torch.float8_e4m3fn, 448.0), "e5m2": (torch.float8_e5m2, 57344.0),
               "e4m3_pow2": (torch.float8_e4m3fn, 448.0), "e5m2_pow2": (torch.float8_e5m2, 57344.0)}
# The "_sr" formats: the records, units and decoder of their base format, rounded stochastically
# (DESIGN §2.13h) with 16 random bits per element.
FP8_SR_FORMATS = {"e4m3_sr": "e4m3", "e5m2_sr": "e5m2"}
_FP8_MIN_UNIT = _F32(2.0 ** -126)


def _fp8_pow2_units(a: np.ndarray, fmax: float) -> Tuple[np.ndarray, np.ndarray]:
    """The power-of-two unit 2^k of buckets whose max |x| is ``a`` (fp32, >= +0 or NaN), k the smallest
    integer >= -126 with a <= fmax * 2^k, and its inverse 2^-k. With a = m * 2^e and fmax = fm * 2^fe
    (frexp, m and fm in [0.5, 1)), a <= fmax * 2^k holds from k = e - fe on when m <= fm, from
    e - fe + 1 otherwise. A NaN or Inf ``a`` is its own unit, with the fp32-scale formats' inverse."""
    finite = np.isfinite(a)
    m, e = np.frexp(np.where(finite, a, 0).astype(np.float64))
    fm, fe = np.frexp(fmax)
    k = e.astype(np.int64) - fe + (m > fm)
    k = np.where(a == 0, -126, np.maximum(k, -126))
    with np.errstate(all="ignore"):
        unit = np.where(finite, np.ldexp(1.0, k), a).astype(_F32)
        inv = np.where(finite, np.ldexp(1.0, -k), _F32(1.0) / unit).astype(_F32)
    return unit, inv


def _fp8_units(b: np.ndarray, fmt: str) -> Tuple[np.ndarray, np.ndarray]:
    """unit and inverse of every row of ``b`` (buckets, fp32) in the FP8 format ``fmt``"""
    fmax = FP8_FORMATS[fmt][1]
    with np.errstate(all="ignore"):
        mn, mx = _nan_minmax(b)
        a = np.maximum(-mn, mx)  # NaN propagates
        a = np.where(a == 0, _F32(0.0), a)  # +0, as max.NaN gives for a zero bucket
        if fmt.endswith("_pow2"):
            return _fp8_pow2_units(a, fmax)
        unit = (a * (_F32(1.0) / _F32(fmax))).astype(_F32)
        inv = np.where(unit < _FP8_MIN_UNIT, _F32(0.0), _F32(1.0) / unit).astype(_F32)
    return unit, inv


def _fp8_code_buckets(v: np.ndarray, fmt: str, bucket: int) -> Tuple[torch.Tensor, np.ndarray]:
    """FP8 codes of a flat fp32 array whose buckets start at index 0, in numpy fp32 arithmetic and
    torch's float8 casts: unit = max|x| * fp32(1/FMAX), inv = 1/unit (0 below 2^-126), or for the
    "_pow2" formats the unit of ``_fp8_pow2_units``; code = float8(clamp(x * inv, ±FMAX)). The clamp stands for the hardware's saturation: torch's
    casts give NaN / Inf past the largest finite value. Returns the codes as a [buckets, bucket]
    float8 tensor (the last bucket padded with its last value) and the units, fp32 [buckets]."""
    tdt, fmax = FP8_FORMATS[fmt]
    n = v.size
    nb = -(-n // bucket)
    pad = nb * bucket - n
    vp = np.concatenate([v, np.repeat(v[-1:], pad)]) if pad else v
    b = vp.reshape(nb, bucket)
    unit, inv = _fp8_units(b, fmt)
    with np.errstate(all="ignore"):
        t = np.clip((b * inv).astype(_F32), _F32(-fmax), _F32(fmax))
    return torch.from_numpy(np.ascontiguousarray(t)).to(tdt), unit.reshape(-1).astype(_F32)


def _fp8_qdq_buckets(v: np.ndarray, fmt: str, bucket: int) -> np.ndarray:
    """FP8 round trip of a flat fp32 array whose buckets start at index 0: the codes of
    ``_fp8_code_buckets`` decoded as float(code) * unit."""
    n = v.size
    if n == 0:
        return np.zeros(0, _F32)
    code, unit = _fp8_code_buckets(v, fmt, bucket)
    with np.errstate(all="ignore"):
        dec = (code.float().numpy() * unit[:, None]).astype(_F32)  # one fp32 multiply
    return dec.reshape(-1)[:n]


def fp8_quantize(x: torch.Tensor, fmt: str, bucket_size: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """FP8 (``fmt`` a name of ``FP8_FORMATS``) codes and per-bucket units of a flat tensor, buckets of
    ``bucket_size`` (clamped as every bucket) from its first element: ``(codes, units)``, the codes
    a float8 tensor of ``x.numel()`` elements, the units fp32, one per bucket. ``codes.float() *
    units`` (bucket-wise, one fp32 multiply) is ``fp8_quantize_dequantize`` before its rounding to
    ``x.dtype``."""
    if fmt not in FP8_FORMATS:
        raise ValueError(f"unknown FP8 format {fmt!r}")
    v = x.detach().reshape(-1).float().cpu().numpy()
    if v.size == 0:
        return torch.empty(0, dtype=FP8_FORMATS[fmt][0]), torch.empty(0, dtype=torch.float32)
    code, unit = _fp8_code_buckets(v, fmt, effective_bucket(bucket_size))
    return code.reshape(-1)[:v.size].clone(), torch.from_numpy(unit)


def fp8_quantize_dequantize(x: torch.Tensor, fmt: str, bucket_size: int) -> torch.Tensor:
    """FP8 (``fmt`` a name of ``FP8_FORMATS``) round trip of a flat tensor, buckets of ``bucket_size``
    (clamped as every bucket) from its first element, rounded to ``x.dtype``."""
    if fmt not in FP8_FORMATS:
        raise ValueError(f"unknown FP8 format {fmt!r}")
    v = x.detach().reshape(-1).float().cpu().numpy()
    dec = _fp8_qdq_buckets(v, fmt, effective_bucket(bucket_size))
    return _to_tensors([dec], x.dtype)[0].view_as(x)


def _sr_words(seed: int, seq: int, stream: int, first: int, n: int, bucket: int) -> np.ndarray:
    """The 16 random bits of n elements from element index ``first`` on, whose buckets of ``bucket``
    start at ``first``: every bucket's pack groups start at its first element (``_C.philox_u16``)."""
    from .. import _C

    parts = [_C.philox_u16(int(seed), int(seq), int(stream), int(first) + b, min(bucket, n - b)).numpy()
             for b in range(0, n, bucket)]
    return np.concatenate(parts).astype(np.int64) if parts else np.zeros(0, np.int64)


def _fp8_sr_round(y: np.ndarray, base: str, h: np.ndarray) -> np.ndarray:
    """The SR rule on y = fp32(x * inv) (DESIGN §2.13h), in float64 and frexp: with s = 2^(max(floor(log2
    |y|), emin) - mb) the grid spacing at |y|, t = |y| / s = n + f, |y| becomes (n + 1) * s when h +
    floor(2^16 f) >= 2^16 and n * s otherwise, saturated to FMAX; y's sign is kept, NaN stays NaN and
    Inf saturates."""
    emin, mb = (-6, 3) if base == "e4m3" else (-14, 2)
    fmax = FP8_FORMATS[base][1]
    ay = np.abs(y.astype(np.float64))
    finite = np.isfinite(ay)
    m, e = np.frexp(np.where(finite, ay, 1.0))
    se = np.maximum(e.astype(np.int64) - 1, emin) - mb
    t = np.ldexp(np.where(finite, ay, 0.0), -se)  # exact: a power-of-two scaling of a 24-bit value
    n = np.floor(t)
    up = (h + np.floor((t - n) * 65536.0)) >= 65536.0
    mag = np.where(finite, np.minimum(np.ldexp(n + up, se), fmax), fmax)
    return np.where(np.isnan(y), np.nan, np.copysign(mag, y)).astype(_F32)


def _fp8_sr_code_buckets(v: np.ndarray, fmt: str, bucket: int, words: np.ndarray) -> Tuple[torch.Tensor, np.ndarray]:
    """``_fp8_code_buckets`` of an ``_sr`` format: the units of its base format, and the codes of the SR
    rule with element i's random bits ``words[i]``."""
    base = FP8_SR_FORMATS[fmt]
    n = v.size
    nb = -(-n // bucket)
    pad = nb * bucket - n
    vp = np.concatenate([v, np.repeat(v[-1:], pad)]) if pad else v
    hp = np.concatenate([words, np.zeros(pad, np.int64)]) if pad else words
    b = vp.reshape(nb, bucket)
    unit, inv = _fp8_units(b, base)
    with np.errstate(all="ignore"):
        y = (b * inv).astype(_F32)
    g = _fp8_sr_round(y, base, hp.reshape(nb, bucket))
    return torch.from_numpy(np.ascontiguousarray(g)).to(FP8_FORMATS[base][0]), unit.reshape(-1).astype(_F32)


def _fp8_sr_qdq_buckets(v: np.ndarray, fmt: str, bucket: int, words: np.ndarray) -> np.ndarray:
    n = v.size
    if n == 0:
        return np.zeros(0, _F32)
    code, unit = _fp8_sr_code_buckets(v, fmt, bucket, words)
    with np.errstate(all="ignore"):
        dec = (code.float().numpy() * unit[:, None]).astype(_F32)
    return dec.reshape(-1)[:n]


def _sr_input(x: torch.Tensor, fmt: str, words) -> Tuple[np.ndarray, np.ndarray]:
    if fmt not in FP8_SR_FORMATS:
        raise ValueError(f"unknown stochastic FP8 format {fmt!r}")
    v = x.detach().reshape(-1).float().cpu().numpy()
    h = np.asarray(words.numpy() if isinstance(words, torch.Tensor) else words, dtype=np.int64).reshape(-1)
    if h.size != v.size:
        raise ValueError(f"need one random word per element: {h.size} words for {v.size} elements")
    return v, h & 0xFFFF


def fp8_sr_quantize(x: torch.Tensor, fmt: str, bucket: int, words) -> Tuple[torch.Tensor, torch.Tensor]:
    """Codes and units of ``x`` (flat, buckets of ``bucket`` from its first element) in the stochastic
    FP8 format ``fmt`` ("e4m3_sr" / "e5m2_sr"), element i rounded with the 16-bit word ``words[i]``:
    ``(codes, units)`` as ``fp8_quantize`` gives them. Computed from the rule of DESIGN §2.13h, not
    by the encoder; the words of a collective come from ``_C.philox_u16``."""
    v, h = _sr_input(x, fmt, words)
    if v.size == 0:
        return torch.empty(0, dtype=FP8_FORMATS[FP8_SR_FORMATS[fmt]][0]), torch.empty(0, dtype=torch.float32)
    code, unit = _fp8_sr_code_buckets(v, fmt, effective_bucket(bucket), h)
    return code.reshape(-1)[:v.size].clone(), torch.from_numpy(unit)


def fp8_sr_quantize_dequantize(x: torch.Tensor, fmt: str, bucket: int, words) -> torch.Tensor:
    """The round trip of ``fp8_sr_quantize``: float(code) * unit, rounded to ``x.dtype``."""
    v, h = _sr_input(x, fmt, words)
    dec = _fp8_sr_qdq_buckets(v, fmt, effective_bucket(bucket), h)
    return _to_tensors([dec], x.dtype)[0].view_as(x)


def _a2a_chunk_fp8(chunk: torch.Tensor, fmt: str, bucket_size: int, seed: int, seq: int, q: int, r: int,
                   codes: bool):
    """The FP8 record of the chunk rank q sends rank r: decoded, or (codes, units) with ``codes``"""
    if fmt in FP8_SR_FORMATS:
        from .. import _C

        n = chunk.numel()
        w = _sr_words(seed, seq, _C.a2a_rng_stream(q, r), 0, n, effective_bucket(bucket_size))
        return fp8_sr_quantize(chunk, fmt, bucket_size, w) if codes else fp8_sr_quantize_dequantize(
            chunk, fmt, bucket_size, w)
    return fp8_quantize(chunk, fmt, bucket_size) if codes else fp8_quantize_dequantize(chunk, fmt, bucket_size)


def all_to_all_reference(inputs: Sequence[torch.Tensor], counts: Sequence[Sequence[int]], *, bits: int | str,
                         bucket_size: int, seed: int = 0, seq: int = 0) -> List[torch.Tensor]:
    """Every rank's output of the compressed all-to-all (round to nearest). ``counts[q][r]`` elements
    go from rank q to rank r; rank q's input holds its chunks in destination order and rank r's
    output the chunks it receives in source order. The own chunk, and every chunk when ``bits`` is
    32, is the input unchanged; every other chunk is ``quantize_dequantize_layers`` of one layer, so
    buckets are counted from the chunk's first element. ``bits`` an FP8 format: every other chunk
    is ``fp8_quantize_dequantize`` instead; an ``_sr`` format rounds the chunk from q to r with the
    stream ``a2a_rng_stream(q, r)`` of (``seed``, ``seq``), elements indexed from the chunk's start."""
    if isinstance(bits, str) and bits not in FP8_FORMATS and bits not in FP8_SR_FORMATS:
        raise ValueError(f"unknown FP8 format {bits!r}")
    fp8 = isinstance(bits, str)
    W = len(inputs)
    flat = [t.detach().reshape(-1).cpu() for t in inputs]
    outs = []
    for r in range(W):
        parts = []
        for q in range(W):
            a = sum(int(c) for c in counts[q][:r])
            n = int(counts[q][r])
            chunk = flat[q][a:a + n].clone()
            if q != r and n > 0 and fp8:
                chunk = _a2a_chunk_fp8(chunk, bits, bucket_size, seed, seq, q, r, False)
            elif q != r and n > 0 and bits < RAW_BITS:
                chunk = quantize_dequantize_layers(chunk, [(0, n, int(bits), int(bucket_size))])
            parts.append(chunk)
        outs.append(torch.cat(parts) if parts else flat[r].new_empty(0))
    return outs


def all_to_all_codes_reference(inputs: Sequence[torch.Tensor], counts: Sequence[Sequence[int]], *, fmt: str,
                               bucket_size: int, seed: int = 0,
                               seq: int = 0) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """Every rank's codes output of the FP8 all-to-all (``output_scales``): rank r's codes are, in
    source order, ``fp8_quantize`` of every chunk it receives, its own chunk included, and its scales
    the units of those chunks' buckets, concatenated (flat; every count a multiple of
    ``bucket_size``, so the scales of a row-major ``[rows, H / bucket_size]`` matrix). An ``_sr``
    format rounds as in ``all_to_all_reference``, the own chunk with the stream ``a2a_rng_stream(r, r)``."""
    W = len(inputs)
    flat = [t.detach().reshape(-1).cpu() for t in inputs]
    codes, scales = [], []
    for r in range(W):
        cs, us = [], []
        for q in range(W):
            a = sum(int(c) for c in counts[q][:r])
            c, u = _a2a_chunk_fp8(flat[q][a:a + int(counts[q][r])], fmt, bucket_size, seed, seq, q, r, True)
            cs.append(c)
            us.append(u)
        codes.append(torch.cat(cs))
        scales.append(torch.cat(us))
    return codes, scales


def all_gather_codes_reference(inputs: Sequence[torch.Tensor], fmt: str, bucket_size: int, seed: int = 0,
                               seq: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """The codes output of the FP8 all-gather (``output_scales``), the same on every rank: codes
    ``fp8_quantize`` of every rank's shard concatenated in rank order (float8, flat), and the units
    of their buckets likewise (fp32, flat; every shard a multiple of ``bucket_size``). An ``_sr``
    format rounds shard q as ``all_gather_reference`` does."""
    if fmt in FP8_SR_FORMATS:
        B = effective_bucket(bucket_size)
        parts = [fp8_sr_quantize(t.detach().reshape(-1).cpu(), fmt, bucket_size,
                                 _sr_words(seed, seq, 2 * q + 1, q * t.numel(), t.numel(), B))
                 for q, t in enumerate(inputs)]
    else:
        parts = [fp8_quantize(t.detach().reshape(-1).cpu(), fmt, bucket_size) for t in inputs]
    return torch.cat([c for c, _ in parts]), torch.cat([u for _, u in parts])


def routed_all_to_all_codes_reference(inputs: Sequence[torch.Tensor], counts: Sequence[Sequence[int]],
                                      input_index: Sequence[torch.Tensor | None],
                                      output_index: Sequence[torch.Tensor | None], row: int, *, fmt: str,
                                      bucket_size: int, outputs: Sequence[torch.Tensor] | None = None,
                                      output_scales: Sequence[torch.Tensor] | None = None
                                      ) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """The routed codes output as the composition that defines it: ``index_select`` of the sent rows,
    ``all_to_all_codes_reference``, then ``index_copy_`` of the received rows' codes (as bytes) and
    scales into copies of ``outputs[r]`` / ``output_scales[r]`` (``None``: the received rows are the
    output). Outputs are flat: codes as float8, scales fp32."""
    W = len(inputs)
    send = []
    for q in range(W):
        x = inputs[q].detach().cpu().reshape(-1, row)
        ix = input_index[q]
        send.append((x if ix is None else x.index_select(0, ix.cpu())).reshape(-1))
    codes, scales = all_to_all_codes_reference(send, counts, fmt=fmt, bucket_size=bucket_size)
    nsr = row // bucket_size
    out_c, out_s = [], []
    for r in range(W):
        ix = output_index[r]
        if ix is None:
            out_c.append(codes[r])
            out_s.append(scales[r])
            continue
        base = outputs[r].detach().cpu().reshape(-1, row).view(torch.uint8).clone()
        base.index_copy_(0, ix.cpu(), codes[r].view(torch.uint8).reshape(-1, row))
        out_c.append(base.reshape(-1).view(codes[r].dtype))
        sb = output_scales[r].detach().cpu().reshape(-1, nsr).clone()
        out_s.append(sb.index_copy_(0, ix.cpu(), scales[r].reshape(-1, nsr)).reshape(-1))
    return out_c, out_s


def routed_all_to_all_reference(inputs: Sequence[torch.Tensor], counts: Sequence[Sequence[int]],
                                input_index: Sequence[torch.Tensor | None],
                                output_index: Sequence[torch.Tensor | None], row: int, *, bits: int | str,
                                bucket_size: int, outputs: Sequence[torch.Tensor] | None = None,
                                input_scale: Sequence[torch.Tensor | None] | None = None, seed: int = 0,
                                seq: int = 0) -> List[torch.Tensor]:
    """Every rank's output of the routed all-to-all, as the composition that defines it: rank q sends
    ``inputs[q].index_select(0, input_index[q])`` (rows of ``row`` elements; ``None``: the input
    itself), ``all_to_all_reference`` exchanges the rows (``counts[q][r]`` elements, whole rows), and
    rank r writes what it receives with ``index_copy_(0, output_index[r], ...)`` into a copy of
    ``outputs[r]`` (``None``: the received rows are the output). Outputs are flat.
    ``input_scale[q]`` (fp32, one entry per ``input_index[q]`` entry; ``None``: unscaled) scales the
    selected rows first: ``(selected.float() * input_scale[q][:, None]).to(dtype)``, one fp32 multiply
    rounded to nearest even in the dtype. ``seed`` / ``seq``: the random bits of an ``_sr`` format, as
    in ``all_to_all_reference``."""
    W = len(inputs)
    send = []
    for q in range(W):
        x = inputs[q].detach().cpu().reshape(-1, row)
        ix = input_index[q]
        sel = x if ix is None else x.index_select(0, ix.cpu())
        sc = None if input_scale is None else input_scale[q]
        if sc is not None:
            sel = (sel.float() * sc.detach().cpu().float()[:, None]).to(x.dtype)
        send.append(sel.reshape(-1))
    recv = all_to_all_reference(send, counts, bits=bits, bucket_size=bucket_size, seed=seed, seq=seq)
    outs = []
    for r in range(W):
        ix = output_index[r]
        if ix is None:
            outs.append(recv[r])
            continue
        base = outputs[r].detach().cpu().reshape(-1, row).clone()
        outs.append(base.index_copy_(0, ix.cpu(), recv[r].reshape(-1, row)).reshape(-1))
    return outs


def combine_rows_reference(slots: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
    """The weighted top-k combine of slot rows: ``slots`` ``[T*k, H]`` (any float dtype), ``gate``
    ``[T, k]`` fp32. For every ``t, h``, with ``x_c = float(slots[t*k + c, h])`` and ``g_c = gate[t, c]``:
    ``acc = fp32(g_0 * x_0)``, then ``acc = fma(g_c, x_c, acc)`` for ``c = 1 .. k-1`` in that order,
    rounded once each (``_fma32_np``); the result is ``acc`` rounded to nearest in the slots' dtype."""
    T, k = gate.shape
    x = slots.detach().cpu().float().reshape(T, k, -1).numpy()
    g = gate.detach().cpu().float().numpy()
    with np.errstate(all="ignore"):
        acc = (g[:, 0, None].astype(np.float64) * x[:, 0].astype(np.float64)).astype(_F32)
    for c in range(1, k):
        acc = _fma32_np(g[:, c, None], x[:, c], acc)
    return torch.from_numpy(np.ascontiguousarray(acc, dtype=_F32)).to(slots.dtype)


def combine_gate_grad_reference(grad_out: torch.Tensor, slots: torch.Tensor) -> torch.Tensor:
    """The gate gradient of the weighted top-k combine in the order of ``combine_gate_grad_kernel``:
    ``grad_out`` ``[T, H]``, ``slots`` ``[T*k, H]`` of one float dtype; returns fp32 ``[T, k]`` with
    ``out[t, c] = sum_h float(grad_out[t, h]) * float(slots[t*k + c, h])``, summed as follows. With
    ``V = 16 // element_size``, element ``h`` belongs to lane ``l = (h // V) % 32``; every lane starts
    at ``+0`` and runs ``acc = fma(go_h, x_h, acc)`` (``_fma32_np``, one rounding) over its elements
    in increasing ``h``; then ``acc += acc[lane ^ m]`` in fp32 for ``m = 16, 8, 4, 2, 1``, which leaves
    the same value in every lane."""
    T = grad_out.shape[0]
    V = 16 // grad_out.element_size()
    go = grad_out.detach().cpu().float().reshape(T, 1, -1).numpy()
    H = go.shape[-1]
    x = slots.detach().cpu().float().reshape(T, -1, H).numpy()
    k = x.shape[1]
    acc = np.zeros((T, k, 32), dtype=_F32)
    lanes = np.arange(32)
    # step j of every lane: its (j // V)-th group of V elements, element j % V of it
    for j in range((H + 32 * V - 1) // (32 * V) * V):
        h = ((j // V) * 32 + lanes) * V + j % V
        ok = h < H
        hc = np.where(ok, h, 0)
        acc = np.where(ok, _fma32_np(go[:, :, hc], x[:, :, hc], acc), acc).astype(_F32)
    with np.errstate(all="ignore"):
        for m in (16, 8, 4, 2, 1):
            acc = (acc + acc[:, :, lanes ^ m]).astype(_F32)
    return torch.from_numpy(np.ascontiguousarray(acc[:, :, 0]))


def routed_all_to_all_combine_reference(inputs: Sequence[torch.Tensor], counts: Sequence[Sequence[int]],
                                        output_index: Sequence[torch.Tensor], gates: Sequence[torch.Tensor],
                                        row: int, *, bits: int | str, bucket_size: int, seed: int = 0,
                                        seq: int = 0) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """Every rank's weighted top-k combine as the composition that defines it: ``routed_all_to_all_reference``
    into slots (rank r's ``output_index[r]`` a permutation of ``[0, T_r * k_r)``), then
    ``combine_rows_reference`` with ``gates[r]`` (``[T_r, k_r]``). Returns (slots, outputs), flat.
    ``seed`` / ``seq``: the random bits of an ``_sr`` format."""
    W = len(inputs)
    bases = [inputs[r].new_zeros(output_index[r].numel() * row) for r in range(W)]
    slots = routed_all_to_all_reference(inputs, counts, [None] * W, output_index, row, bits=bits,
                                        bucket_size=bucket_size, outputs=bases, seed=seed, seq=seq)
    outs = [combine_rows_reference(slots[r].reshape(-1, row), gates[r]).reshape(-1) for r in range(W)]
    return slots, outs


def dispatch_sum_reference(slots: torch.Tensor, k: int) -> torch.Tensor:
    """The sum of each token's k slot rows, as the backward of an MoE dispatch defines it: ``slots``
    ``[T*k, H]`` (any float dtype); for every ``t, h``, with ``x_c = float(slots[t*k + c, h])``,
    ``acc = x_0``, then ``acc = acc + x_c`` for ``c = 1 .. k-1`` in that order, each add an IEEE fp32
    add (numpy float32); the result is ``acc`` rounded to nearest in the slots' dtype. NaN, Inf and
    signed zeros follow from IEEE addition: k slots of -0 sum to -0."""
    x = slots.detach().cpu().float().reshape(slots.shape[0] // k, k, -1).numpy()
    acc = x[:, 0].copy()
    with np.errstate(all="ignore"):
        for c in range(1, k):
            acc = np.add(acc, x[:, c], dtype=_F32)
    return torch.from_numpy(np.ascontiguousarray(acc, dtype=_F32)).to(slots.dtype)


def dispatch_backward_reference(grads: Sequence[torch.Tensor], counts: Sequence[Sequence[int]],
                                slot_index: Sequence[torch.Tensor], k: int, row: int, *, bits: int | str,
                                bucket_size: int, input_index: Sequence[torch.Tensor | None] | None = None,
                                seed: int = 0, seq: int = 0) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """Every rank's input gradient of ``differentiable_all_to_all_dispatch``, as the composition that
    defines it: ``routed_all_to_all_reference`` of the gradients ``grads`` (rank q's rows gathered by
    ``input_index[q]``, the forward's output index; ``None``: in order; ``counts[q][r]`` elements go
    back from rank q to rank r) into zeroed slots scattered by ``slot_index[r]`` (a permutation of
    ``[0, T_r * k)``), then ``dispatch_sum_reference`` of each token's k slots. Returns (slots,
    gradients), flat."""
    W = len(grads)
    bases = [grads[r].new_zeros(slot_index[r].numel() * row) for r in range(W)]
    slots = routed_all_to_all_reference(grads, counts, input_index or [None] * W, slot_index, row, bits=bits,
                                        bucket_size=bucket_size, outputs=bases, seed=seed, seq=seq)
    outs = [dispatch_sum_reference(slots[r].reshape(-1, row), k).reshape(-1) for r in range(W)]
    return slots, outs


# ---- the sharded collectives over several nodes (AllreduceEngine::sharded, DESIGN §2.9b) -----------
SHARDED_PERTURBATIONS = ("prescale_local", "requantized_gather", "quantized_own_partial", "transposed_ranks")
_CROSS_SEQ = 0x40000000  # the allreduce's cross-node marker


def _hier_rank(n: int, l: int, nodes: int, local_size: int, perturb: str | None) -> int:
    """The rank of local rank l on node n: n*L + l (l*N + n under ``transposed_ranks``)."""
    return l * nodes + n if perturb == "transposed_ranks" else n * local_size + l


def _raw_table(layers: Sequence[Layer]) -> List[Layer]:
    return [(int(o), int(n), RAW_BITS, int(b)) for o, n, _, b in layers]


def _rs_quantized_own(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *, prescale: float,
                      skip_incomplete: bool) -> List[torch.Tensor]:
    """``reduce_scatter_reference`` with each rank's own contribution quantized like its peers' (the
    wrong semantics ``quantized_own_partial``)."""
    dtype = inputs[0].dtype
    segs = layer_segments(shard_layers, skip_incomplete)
    outs = []
    for r in range(len(inputs)):
        xs = _scaled_inputs(_shards(inputs, r), _F32(prescale))
        xs[r] = _quantized(xs[r], segs, dtype)
        out = np.zeros(xs[0].size, _F32)
        for off, m, bits, bucket in segs:
            sl = slice(off, off + m)
            out[sl] = _sra_acc(xs, sl, np.full(m, r), bits, bucket, dtype)
        outs.append(out)
    return _to_tensors(outs, dtype)


def _rs_hier(inputs, shard_layers, local_size, *, average, intra_compress, perturb, stage, seq=0):
    """The two-stage reduce-scatter, each flat reduce-scatter computed by
    ``stage(ins, table, prescale, seq, cross)``."""
    W, L = len(inputs), local_size
    N = W // L
    assert N * L == W, "the local size divides the world"
    dtype = inputs[0].dtype
    ps = _prescale(W, average)
    full = [t.detach().reshape(-1).cpu() for t in inputs]
    S = full[0].numel() // W
    shard_layers = [tuple(int(v) for v in l) for l in shard_layers]
    if L > 1 or N == 1:
        # 1. inside node n, for every node block b: the local reduce-scatter of in[b*L*S, (b+1)*L*S)
        ps1 = _prescale(L, average) if perturb == "prescale_local" else ps
        t1 = _raw_table(shard_layers) if (N > 1 and not intra_compress) else shard_layers
        partial = [torch.empty(N * S, dtype=dtype) for _ in range(W)]
        for n in range(N):
            rk = [_hier_rank(n, l, N, L, perturb) for l in range(L)]
            for b in range(N):
                outs = stage([full[r][b * L * S:(b + 1) * L * S] for r in rk], t1, ps1, seq ^ b, False)
                for r, o in zip(rk, outs):
                    partial[r][b * S:(b + 1) * S] = o.reshape(-1)
        if N == 1:
            return partial
        ps2 = _F32(1.0)
    else:
        partial, ps2 = full, ps
    # 2. across nodes, among the ranks of local rank l: node n's partial P[n] unquantized, Q of the others
    result = [None] * W
    for l in range(L):
        rk = [_hier_rank(n, l, N, L, perturb) for n in range(N)]
        for r, o in zip(rk, stage([partial[r] for r in rk], shard_layers, ps2, seq ^ _CROSS_SEQ, True)):
            result[r] = o.reshape(-1)
    return result


def reduce_scatter_hier_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *,
                                  local_size: int, average: bool = False, skip_incomplete: bool = False,
                                  intra_compress: bool = True, perturb: str | None = None,
                                  fmt: str | None = None) -> List[torch.Tensor]:
    """Every rank's output of the compressed reduce-scatter over N = W / L nodes of L = ``local_size``
    consecutive ranks (deterministic rounding); rank r = n*L + l, ``inputs[r]`` holds W shards of S.

    1. Inside node n (skipped when L = 1), for each node block b: ``reduce_scatter_reference`` of the
       L local ranks' in[b*L*S, (b+1)*L*S) with the shard table (raw when N > 1 and not
       ``intra_compress``) and prescale 1/W when averaging; local rank l keeps P[b] = the node's
       partial of chunk b*L + l, stored in the dtype.
    2. Across nodes, among the N ranks of local rank l: ``reduce_scatter_reference`` of the N
       partial buffers with prescale 1 (with L = 1: of the inputs, prescale 1/W when averaging):
       rank (n, l) gets P[n] unquantized plus Q of every other node's P[n], in node order.
    With N = 1 this is ``reduce_scatter_reference``, and with L = 1 bitwise the same over W ranks.
    ``perturb`` (one of ``SHARDED_PERTURBATIONS``) switches on a wrong semantics for the tests.
    ``fmt`` (a name of ``FP8_FORMATS``): both stages use that FP8 format (``reduce_scatter_reference``).
    """
    def stage(ins, table, prescale, _seq, cross):
        if cross and perturb == "quantized_own_partial":
            return _rs_quantized_own(ins, table, prescale=prescale, skip_incomplete=skip_incomplete)
        return reduce_scatter_reference(ins, table, prescale=prescale, skip_incomplete=skip_incomplete, fmt=fmt)

    return _rs_hier(inputs, shard_layers, local_size, average=average, intra_compress=intra_compress,
                    perturb=perturb, stage=stage)


def _ag_hier(inputs, shard_layers, local_size, *, perturb, stage, seq=0):
    """The two-stage all-gather, each flat compressed all-gather computed by ``stage(ins, table, seq)``
    (one tensor, every rank's output)."""
    W, L = len(inputs), local_size
    N = W // L
    assert N * L == W, "the local size divides the world"
    shards = [t.detach().reshape(-1).cpu() for t in inputs]
    shard_layers = [tuple(int(v) for v in l) for l in shard_layers]
    if N == 1:
        return [stage(shards, shard_layers, seq)] * W
    S = shards[0].numel()
    # 1. across nodes: the ranks of local rank l gather Q of each other's shard, G = N shards
    gathered = [None] * W
    for l in range(L):
        rk = [_hier_rank(n, l, N, L, perturb) for n in range(N)]
        g = stage([shards[r] for r in rk], shard_layers, seq ^ _CROSS_SEQ)
        for r in rk:
            gathered[r] = g
    # 2. inside node n, for every n2: local rank l2's G[n2] travels raw (re-quantized under
    #    ``requantized_gather``) to out[(n2*L + l2)*S]
    result = [None] * W
    for n in range(N):
        out = torch.empty(W * S, dtype=shards[0].dtype)
        for n2 in range(N):
            for l2 in range(L):
                piece = gathered[_hier_rank(n, l2, N, L, perturb)][n2 * S:(n2 + 1) * S]
                if perturb == "requantized_gather" and L > 1:
                    piece = quantize_dequantize_layers(piece, shard_layers)
                out[(n2 * L + l2) * S:(n2 * L + l2 + 1) * S] = piece
        for l in range(L):
            result[_hier_rank(n, l, N, L, perturb)] = out
    return result


def all_gather_hier_reference(inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *, local_size: int,
                              perturb: str | None = None) -> List[torch.Tensor]:
    """Every rank's output of the compressed all-gather over N = W / L nodes of L = ``local_size``
    consecutive ranks (deterministic rounding); ``inputs[r]`` is rank r's shard of S elements.

    1. Across nodes (skipped when N = 1), among the N ranks of local rank l: ``all_gather_reference``
       of their shards, G = Q of each, node by node.
    2. Inside node n (with N = 1 the compressed all-gather itself): local rank l2's G[n2] is copied
       unchanged (a raw table) to out[(n2*L + l2)*S, ...) of every rank of the node.
    Every shard gets exactly one quantization round trip, so every rank's output is
    ``all_gather_reference`` of all W inputs, for every (N, L).
    """
    return _ag_hier(inputs, shard_layers, local_size, perturb=perturb,
                    stage=lambda ins, table, _seq: all_gather_reference(ins, table))


def _replicated(window: Sequence[Layer], world: int, S: int) -> List[Layer]:
    return [(o + c * S, n, b, k) for c in range(world) for o, n, b, k in window]


def sharded_engine_reference(op: str, inputs: Sequence[torch.Tensor], shard_layers: Sequence[Layer], *,
                             local_size: int, config: dict, lanes: int, slot_bytes: Tuple[int, int] = (0, 0),
                             average: bool = False, call_seq: int = 1, cuda: bool = True,
                             skip_incomplete: bool = False, stochastic: bool = False, seed: int = 0):
    """Every rank's output of one ``AllreduceEngine::sharded`` call and the stages each rank issues,
    ``(outputs, stages)``, stages as in ``engine_reference``; ``op`` is "reduce_scatter" or
    "all_gather" (which runs without ``skip_incomplete``).

    The call runs with RNG sequence ``call_seq << 4``. Node-local stages (every node block b, or
    every gathered node n2) run with ``seq ^ b``, the cross-node stage with ``seq ^ 0x40000000``.
    A node-local stage is the fused kernel with ``cuda`` and heaps (``p2p``): one "rs" / "ag" launch
    per window of ``C.reduce_scatter_windows`` at the heap's slot size, logged with the window's
    table; otherwise one "generic_rs" / "generic_ag" stage with the whole table. The cross-node
    stage is "cross_rs" / "cross_ag". Scales: 1/W when averaging for the reduce-scatter's first
    stage (the cross one when L = 1), else 1. ``stochastic`` composes ``C.reduce_scatter_simulate``
    and ``C.all_gather_simulate`` with these sequence numbers; otherwise the values are
    ``reduce_scatter_hier_reference`` / ``all_gather_hier_reference``.
    """
    from .. import _C

    cfg = dict(ENGINE_DEFAULTS, **config)
    W, L = len(inputs), local_size
    N = W // L
    rs = op == "reduce_scatter"
    assert rs or op == "all_gather"
    skip = skip_incomplete and rs
    dtype = inputs[0].dtype
    dt = _DTYPE_CODE[dtype]
    table = [tuple(int(v) for v in l) for l in shard_layers]
    S = sum(l[1] for l in table)
    ps = _prescale(W, average)
    seq = (call_seq << 4) & _U32
    intra_table = _raw_table(table) if N > 1 and (not rs or not cfg["intra_compress"]) else table

    stages = [[] for _ in range(W)]

    def log(r, kind, ls, s, scale, lanes_=0, numel=None):
        stages[r].append(dict(kind=kind, layers=[tuple(l) for l in ls], lanes=lanes_,
                              numel=sum(l[1] for l in ls) if numel is None else numel, seed=seed,
                              seq=s & _U32, stochastic=stochastic, scale=float(scale)))

    def intra(r, s, scale):
        if not (cuda and cfg["p2p"]):
            log(r, "generic_rs" if rs else "generic_ag", intra_table, s, scale)
            return
        for w in _C.reduce_scatter_windows(intra_table, world=L, lanes=lanes, dtype=dt, skip_incomplete=skip,
                                           min_lane_elems=cfg["min_lane_elems"], slot_bytes=slot_bytes[0]):
            p = _C.build_plan(_replicated(w, L, S), world=L, lanes=lanes, dtype=dt, skip_incomplete=skip,
                              min_lane_elems=cfg["min_lane_elems"])
            log(r, "rs" if rs else "ag", w, s, scale, p["lanes"], p["numel"])

    local = L > 1 or N == 1
    for r in range(W):
        if rs:
            for b in range(N if local else 0):
                intra(r, seq ^ b, ps)
            if N > 1:
                log(r, "cross_rs", table, seq ^ _CROSS_SEQ, _F32(1.0) if L > 1 else ps)
        else:
            if N > 1:
                log(r, "cross_ag", table, seq ^ _CROSS_SEQ, 1.0)
            for n in range(N if local else 0):
                intra(r, seq ^ n, 1.0)

    if not stochastic:
        if rs:
            outs = reduce_scatter_hier_reference(inputs, table, local_size=L, average=average, skip_incomplete=skip,
                                                 intra_compress=cfg["intra_compress"])
        else:
            outs = all_gather_hier_reference(inputs, table, local_size=L)
        return outs, stages

    def rs_stage(ins, t, prescale, s, _cross):
        outs = [torch.empty(ins[0].numel() // len(ins), dtype=dtype) for _ in ins]
        _C.reduce_scatter_simulate([x.contiguous() for x in ins], outs, t, 1, False, skip, True, seed, s,
                                   cfg["min_lane_elems"], prescale=float(prescale))
        return outs

    def ag_stage(ins, t, s):
        outs = [torch.empty(ins[0].numel() * len(ins), dtype=dtype) for _ in ins]
        _C.all_gather_simulate([x.contiguous() for x in ins], outs, t, True, seed, s)
        return outs[0]

    if rs:
        return _rs_hier(inputs, table, L, average=average, intra_compress=cfg["intra_compress"], perturb=None,
                        stage=rs_stage, seq=seq), stages
    return _ag_hier(inputs, table, L, perturb=None, stage=ag_stage, seq=seq), stages


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


# ---- bit allocation ------------------------------------------------------------------------------
def _layer_wire_bytes(numel: int, bits: int, bucket_size: int) -> int:
    """Wire bytes of one layer (ops.wire_bytes) with the bucket clamped as the plan clamps it."""
    from .quantization import wire_bytes

    return wire_bytes(int(numel), int(bits), effective_bucket(bucket_size))


def allocate_bits_reference(errors, numels: Sequence[int], bucket_sizes: Sequence[int], candidates: Sequence[int],
                            budget_bytes: int, current=None, resolution: int = 4096, *, target_bits=None) -> List[int]:
    """NumPy dynamic program of ``ops.allocate_bits`` (same arguments, same result for every input)."""
    err = np.asarray(errors, dtype=np.float64)
    cands = [int(c) for c in candidates]
    L, K = len(numels), len(cands)
    if err.shape != (L, K):
        raise ValueError(f"allocate_bits: errors has shape {err.shape}, expected ({L}, {K})")
    if K == 0 or resolution < 1:
        raise ValueError("allocate_bits: need at least one candidate and resolution >= 1")
    cost = np.array([[_layer_wire_bytes(n, b, bs) for b in cands] for n, bs in zip(numels, bucket_sizes)],
                    dtype=np.int64).reshape(L, K)
    if target_bits is None:
        fits = [k for k in range(K) if cost[:, k].sum() <= budget_bytes]
        target_bits = max(cands[k] for k in fits) if fits else min(cands)
    keep = [int(c) for c in current] if current is not None else [int(target_bits)] * L
    out = list(keep)
    finite = np.isfinite(err).all(axis=1)
    free = [l for l in range(L) if finite[l]]
    fixed_bytes = sum(_layer_wire_bytes(numels[l], keep[l], bucket_sizes[l]) for l in range(L) if not finite[l])
    room = int(budget_bytes) - fixed_bytes
    k_t = cands.index(target_bits) if target_bits in cands else None
    uniform = list(out)
    for l in free:
        uniform[l] = int(target_bits)
    if not free or room <= 0:
        return uniform

    # bins[l, k] = ceil(cost * resolution / room): any choice with sum(bins) <= resolution fits
    R = int(resolution)
    bins = (cost[free] * R + room - 1) // room
    e = err[free]
    # candidates visited in (bytes, index) order with strict improvement: ties keep fewer bytes
    order = np.lexsort((np.arange(K)[None, :].repeat(len(free), 0), cost[free]), axis=1)
    dp = np.zeros(R + 1)  # least error of the layers so far within c bins
    choice = np.zeros((len(free), R + 1), dtype=np.int16)
    for i in range(len(free)):
        best = np.full(R + 1, np.inf)
        pick = np.zeros(R + 1, dtype=np.int16)
        for k in order[i]:
            c = int(bins[i, k])
            if c > R:
                continue
            cand = np.full(R + 1, np.inf)
            cand[c:] = dp[: R + 1 - c] + e[i, k]
            better = cand < best
            best[better] = cand[better]
            pick[better] = k
        dp, choice[i] = best, pick
    if not np.isfinite(dp[R]):
        return uniform
    c = int(np.argmax(dp == dp[R]))  # fewest bins that reach the least error (dp is non-increasing)
    total = dp[R]
    for i in range(len(free) - 1, -1, -1):
        k = int(choice[i, c])
        out[free[i]] = cands[k]
        c -= int(bins[i, k])
    if k_t is not None and cost[free, k_t].sum() <= room and total > e[:, k_t].sum():
        return uniform
    return out
