"""Power-of-two FP8 scales ("e4m3_pow2" / "e5m2_pow2") without a GPU: the unit against its definition
(smallest k >= -126 with max|x| <= FMAX * 2^k, brute force over k), the properties the formats promise
(units in [2^-126, 2^120] and E8M0-exact, max |code| in [FMAX/2, FMAX], decode(quantize(.)) a
projection, the base format's relative error), the simulators against the oracle bit for bit for
every collective (all-to-all plain, across nodes and codes output, routed compositions,
reduce-scatter, all-gather and its codes output, SRA, one-shot, Ring, compressed broadcast, the
engine's stages and the two-stage sharded path), and the front ends' acceptance and refusals."""
from __future__ import annotations

import math
import os

import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import fsdp as FS
from torch_cgx_b200.parallel import hooks as H

import _a2a_cases as A
from _bitwise import assert_same
from _edge_inputs import edge_inputs
from _engine_cases import TIMEOUT_MS, assert_results, clean_environment, inputs_for, mixed_table  # noqa: F401

FMTS = ("e4m3_pow2", "e5m2_pow2")
BASE = {"e4m3_pow2": "e4m3", "e5m2_pow2": "e5m2"}
FMAX = {"e4m3_pow2": 448.0, "e5m2_pow2": 57344.0}
TDT = {"e4m3_pow2": torch.float8_e4m3fn, "e5m2_pow2": torch.float8_e5m2}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
WORLDS = (2, 3, 8)
H_ROW = 1536  # the row length of the "H" bucket
BUCKETS = (7, 128, 512, 1024, 8192, "H")
MIXED = [(0, 37, 32, 512), (37, 3000, 8, 100), (3037, 301, 32, 512), (3338, 1501, 8, 7), (4839, 700, 8, 1024)]
S_MIXED = 5539


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)


def _b(bucket):
    return H_ROW if bucket == "H" else bucket


def _unit_by_definition(a: float, fmax: float) -> float:
    """2^k for the smallest integer k >= -126 with a <= fmax * 2^k, by search (exact in float64)"""
    if math.isnan(a) or math.isinf(a):
        return a
    k = -126
    while a > fmax * 2.0 ** k:
        k += 1
    return 2.0 ** k


def _hostile(n: int, seed: int) -> torch.Tensor:
    """buckets spanning the fp32 range: gaussians scaled by 2^e for e in [-140, 120], plus zeros, a
    bucket far below FMAX * 2^-126, FLT_MAX and values at, just below and just above FMAX * 2^k"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g, dtype=torch.float64)
    e = torch.randint(-140, 120, (n // 64 + 1,), generator=g).repeat_interleave(64)[:n]
    x = (x * torch.pow(2.0, e.double())).float()
    x[:64] = 0.0
    x[64:128] = -0.0
    x[128:192] = 2.0 ** -130 * torch.arange(64)
    x[192] = 3.4028234663852886e38
    x[256] = 448.0 * 2.0 ** 3
    x[320] = float(np.nextafter(np.float32(448.0 * 2.0 ** 3), np.float32(np.inf)))
    x[384] = 57344.0 * 2.0 ** -20
    x[448] = float(np.nextafter(np.float32(57344.0 * 2.0 ** -20), np.float32(0)))
    return x


# ---- the unit and the properties ------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_unit_is_its_definition(fmt):
    x = _hostile(64 * 200, 1)
    codes, units = O.fp8_quantize(x, fmt, 64)
    a = x.reshape(-1, 64).abs().amax(1).double().tolist()
    want = torch.tensor([_unit_by_definition(v, FMAX[fmt]) for v in a], dtype=torch.float32)
    assert_same(units, want, fmt)
    # the simulator's units (the C++ bit arithmetic) are the oracle's
    c = [[0, x.numel()], [0, 0]]
    outs = [torch.empty(0, dtype=TDT[fmt]), torch.empty(x.numel(), dtype=TDT[fmt])]
    scales = [torch.empty(0), torch.full((x.numel() // 64,), float("nan"))]
    _C.all_to_all_simulate([x, x.new_zeros(0)], outs, c, bits=fmt, bucket_size=64, output_scales=scales)
    assert_same(scales[1], units, f"{fmt} simulator")
    assert torch.equal(outs[1].view(torch.uint8), codes.view(torch.uint8))


@pytest.mark.parametrize("fmt", FMTS)
def test_unit_properties(fmt):
    x = _hostile(64 * 300, 2)
    codes, units = O.fp8_quantize(x, fmt, 64)
    m, e = np.frexp(units.numpy().astype(np.float64))
    assert (m == 0.5).all() and (e - 1 >= -126).all() and (e - 1 <= 120).all()
    assert torch.equal(units.to(torch.float8_e8m0fnu).float(), units)
    amax = x.reshape(-1, 64).abs().amax(1)
    cmax = codes.float().reshape(-1, 64).abs().amax(1)
    big = amax >= FMAX[fmt] * 2.0 ** -126
    assert big.sum() > 100
    assert ((cmax[big] >= FMAX[fmt] / 2) & (cmax[big] <= FMAX[fmt])).all()
    # zero buckets: unit 2^-126 and signed zero codes
    assert units[0] == 2.0 ** -126 and units[1] == 2.0 ** -126
    assert (codes[:64].view(torch.uint8) == 0).all() and (codes[64:128].view(torch.uint8) == 0x80).all()
    # a tiny bucket is encoded on the FP8 grid at 2^-126, not flushed
    dec = codes[128:192].float().double() * float(units[2])
    assert units[2] == 2.0 ** -126 and (dec[1:] != 0).all()
    bound = 2.0 ** -4 if fmt == "e4m3_pow2" else 2.0 ** -3
    assert ((dec - x[128:192].double()).abs() <= bound * x[128:192].double()).all()
    # FLT_MAX: unit 2^120 for e4m3, 2^113 for e5m2
    assert units[3] == 2.0 ** (120 if fmt == "e4m3_pow2" else 113)


@pytest.mark.parametrize("fmt", FMTS)
def test_nonfinite_bucket_unit_and_nan_decode(fmt):
    x = torch.randn(256)
    x[3], x[70], x[140:150] = float("nan"), float("inf"), float("-inf")
    codes, units = O.fp8_quantize(x, fmt, 64)
    assert math.isnan(units[0]) and units[1] == math.inf and units[2] == math.inf and torch.isfinite(units[3])
    dec = O.fp8_quantize_dequantize(x, fmt, 64)
    assert torch.isnan(dec[:192]).all() and torch.isfinite(dec[192:]).all()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [7, 64, 512, 8192])
def test_quantize_is_a_projection(fmt, bucket):
    g = torch.Generator().manual_seed(bucket)
    x = torch.randn(3 * 8192 + 5, generator=g) * torch.exp(torch.randn(3 * 8192 + 5, generator=g) * 3)
    once = O.fp8_quantize_dequantize(x, fmt, bucket)
    twice = O.fp8_quantize_dequantize(once, fmt, bucket)
    assert torch.equal(once.view(torch.int32), twice.view(torch.int32))
    # the fp32-scale format is not a projection on the same data
    b1 = O.fp8_quantize_dequantize(x, BASE[fmt], bucket)
    b2 = O.fp8_quantize_dequantize(b1, BASE[fmt], bucket)
    assert not torch.equal(b1.view(torch.int32), b2.view(torch.int32))


@pytest.mark.parametrize("fmt", FMTS)
def test_relative_error_bound(fmt):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(512 * 64, generator=g) * torch.exp(torch.randn(512 * 64, generator=g))
    x[::512] *= 1000.0  # one outlier per bucket
    codes, units = O.fp8_quantize(x, fmt, 512)
    dec = O.fp8_quantize_dequantize(x, fmt, 512)
    bound = 2.0 ** -4 if fmt == "e4m3_pow2" else 2.0 ** -3
    # the base format's normal range: |x| / unit >= 2^-6 (e4m3) / 2^-14 (e5m2)
    normal = x.abs() >= units.repeat_interleave(512) * (2.0 ** -6 if fmt == "e4m3_pow2" else 2.0 ** -14)
    assert normal.sum() > 0.9 * x.numel()
    assert ((dec - x).abs()[normal] <= bound * x.abs()[normal]).all()


# ---- simulators against the oracle, bit for bit ------------------------------------------------------
def _a2a_inputs(world, dtype, bucket, seed):
    B = _b(bucket)
    c = [[v * H_ROW for v in row] for row in A.counts(world, "uneven", 2, seed)] if bucket == "H" else \
        A.counts(world, "uneven", A.base_elems(B), seed)
    return c, A.inputs(c, dtype, seed)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_all_to_all_simulator(bucket, world, fmt, dtype):
    B = _b(bucket)
    c, xs = _a2a_inputs(world, dtype, bucket, 7 * world + B)
    outs = A.outputs(c, dtype)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=B)
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=B)
    for r in range(world):
        assert_same(outs[r], ref[r], f"rank {r}")


@pytest.mark.parametrize("world", (17, 24))
@pytest.mark.parametrize("fmt", FMTS)
def test_all_to_all_simulator_across_nodes(world, fmt):
    c = A.counts(world, "uneven", 70, seed=world)
    xs = A.inputs(c, torch.bfloat16, seed=3)
    outs = A.outputs(c, torch.bfloat16)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=64)
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=64)
    for r in range(world):
        assert_same(outs[r], ref[r], f"rank {r}")


def _codes_buffers(c, B, fmt):
    W = len(c)
    outs, scales = [], []
    for r in range(W):
        n = sum(c[q][r] for q in range(W))
        outs.append(torch.full((n,), 0x55, dtype=torch.uint8).view(TDT[fmt]))
        scales.append(torch.full((n // B,), float("nan")))
    return outs, scales


def _assert_codes(got, ref, what):
    gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
    assert torch.equal(gn, rn), what
    assert torch.equal(got.view(torch.uint8)[~gn], ref.view(torch.uint8)[~rn]), what


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("bucket", [128, 512, 1024, "H"])
def test_all_to_all_codes_simulator(bucket, world, fmt, dtype):
    B = _b(bucket)
    H_ = max(B, 1024)
    c = [[v * H_ for v in row] for row in A.counts(world, "uneven", 2, world)]
    xs = A.inputs(c, dtype, B)
    outs, scales = _codes_buffers(c, B, fmt)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=B, output_scales=scales)
    rc, rs = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=B)
    for r in range(world):
        _assert_codes(outs[r], rc[r], f"rank {r} codes")
        assert_same(scales[r], rs[r], f"rank {r} scales")
        finite = torch.isfinite(scales[r])
        assert torch.equal(scales[r][finite].to(torch.float8_e8m0fnu).float(), scales[r][finite])


@pytest.mark.parametrize("fmt", FMTS)
def test_routed_scaled_and_combine_references_compose_the_simulator(fmt):
    W, Hh, B = 3, 1024, 512
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(6, Hh, generator=g).bfloat16() for _ in range(W)]
    rows = [[1, 2, 1], [2, 0, 2], [1, 1, 1]]
    c = [[v * Hh for v in row] for row in rows]
    ii = [torch.randint(0, 6, (sum(rows[q]),), generator=g) for q in range(W)]
    n_out = [sum(rows[q][r] for q in range(W)) for r in range(W)]
    oi = [torch.randperm(n_out[r], generator=g) for r in range(W)]
    sc = [torch.rand(sum(rows[q]), generator=g) * 2 for q in range(W)]
    base = [torch.zeros(n_out[r] * Hh, dtype=torch.bfloat16) for r in range(W)]
    got = O.routed_all_to_all_reference(xs, c, ii, oi, Hh, bits=fmt, bucket_size=B, outputs=base, input_scale=sc)
    send = [(xs[q].index_select(0, ii[q]).float() * sc[q][:, None]).bfloat16().reshape(-1) for q in range(W)]
    outs = A.outputs(c, torch.bfloat16)
    _C.all_to_all_simulate(send, outs, c, bits=fmt, bucket_size=B)
    for r in range(W):
        want = torch.empty(n_out[r], Hh, dtype=torch.bfloat16).index_copy_(0, oi[r], outs[r].reshape(-1, Hh))
        assert_same(got[r].reshape(-1), want.reshape(-1), f"routed rank {r}")
    # the combine: k = 1 slots per token, gate 1 -> the slots themselves
    gates = [torch.ones(n_out[r], 1) for r in range(W)]
    slots, comb = O.routed_all_to_all_combine_reference(xs, c, oi, gates, Hh, bits=fmt, bucket_size=B)
    plain = O.routed_all_to_all_reference(xs, c, [None] * W, oi, Hh, bits=fmt, bucket_size=B, outputs=base)
    for r in range(W):
        assert_same(slots[r].reshape(-1), plain[r].reshape(-1), f"combine slots rank {r}")


def _rs(full, table, fmt, **kw):
    W = len(full)
    outs = [torch.empty(full[0].numel() // W, dtype=full[0].dtype) for _ in range(W)]
    _C.reduce_scatter_simulate(full, outs, table, bits=fmt, **kw)
    return outs


def _ag(shards, table, fmt, **kw):
    W = len(shards)
    outs = [torch.empty(W * shards[0].numel(), dtype=shards[0].dtype) for _ in range(W)]
    _C.all_gather_simulate(shards, outs, table, bits=fmt, **kw)
    return outs


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_sharded_simulators(bucket, world, fmt, dtype):
    B = _b(bucket)
    S = 3 * 8192 + 37
    g = torch.Generator().manual_seed(world + B)
    full = [(torch.randn(world * S, generator=g) * (r + 1)).to(dtype) for r in range(world)]
    table = [(0, S, 8, B)]
    assert_results(_rs(full, table, fmt, average=True), O.reduce_scatter_reference(full, table, average=True, fmt=fmt),
                   "rs")
    own = [full[r][r * S:(r + 1) * S].clone() for r in range(world)]
    assert_results(_ag(own, table, fmt), [O.all_gather_reference(own, table, fmt)] * world, "ag")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("bucket", [128, 1024, 8192, "H"])
def test_all_gather_codes_simulator(bucket, world, fmt):
    B = _b(bucket)
    S = 2 * max(B, 1024)
    g = torch.Generator().manual_seed(B)
    xs = [(torch.randn(S, generator=g) * torch.exp(torch.randn(S, generator=g) * 2)) for _ in range(world)]
    codes = [torch.full((world * S,), 0x55, dtype=torch.uint8).view(TDT[fmt]) for _ in range(world)]
    scales = [torch.full((world * S // B,), float("nan")) for _ in range(world)]
    _C.all_gather_simulate(xs, codes, [(0, S, 8, B)], bits=fmt, output_scales=scales)
    rc, rs = O.all_gather_codes_reference(xs, fmt, B)
    for r in range(world):
        _assert_codes(codes[r], rc, f"rank {r}")
        assert_same(scales[r], rs, f"rank {r}")


def _inputs(world, n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def _allreduce_check(xs, layers, fmt, what, **kw):
    sra = [x.clone() for x in xs]
    _C.sra_simulate(sra, layers, bits=fmt, **kw)
    assert_results(sra, O.sra_reference(xs, layers, fmt=fmt, **kw), f"sra {what}")
    one = [x.clone() for x in xs]
    _C.oneshot_simulate(one, layers, bits=fmt, **kw)
    assert_results(one, O.oneshot_reference(xs, layers, fmt=fmt, **kw), f"oneshot {what}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_allreduce_simulators(bucket, world, fmt, dtype):
    n = 9000
    table = [(0, n, 8, _b(bucket))]
    xs = _inputs(world, n, dtype, 13 * world + _b(bucket))
    _allreduce_check(xs, table, fmt, f"B={bucket}", average=True)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("where", ["owner", "peer"])
def test_edge_inputs_every_op(where, fmt, dtype):
    world, bucket, n = 3, 64, 64 * 90
    table = [(0, n, 8, bucket)]
    owners = O.block_owners(table, n, world, 1, dtype, False, 2048)
    xs, planted = edge_inputs(dtype, n, bucket, 5, world=world, bits=8, owners=owners, where=where)
    assert planted
    _allreduce_check(xs, table, fmt, f"edge {where}")
    S = n // world
    stab = [(0, S, 8, bucket)]
    assert_results(_rs(xs, stab, fmt), O.reduce_scatter_reference(xs, stab, fmt=fmt), "edge rs")
    own = [xs[r][r * S:(r + 1) * S].clone() for r in range(world)]
    assert_results(_ag(own, stab, fmt), [O.all_gather_reference(own, stab, fmt)] * world, "edge ag")
    c = [[S] * world for _ in range(world)]
    outs = A.outputs(c, dtype)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=bucket)
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=bucket)
    for r in range(world):
        assert_same(outs[r], ref[r], f"edge a2a rank {r}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [2, 3])
def test_host_generic_reducers(world, fmt, dtype):
    xs = _inputs(world, S_MIXED, dtype, 3 + world)
    for kind, ref in (("SRA", O.sra_reference), ("RING", O.ring_reference)):
        out = [x.clone() for x in xs]
        _C.LocalReducerGroup(world, kind, 5000).allreduce(out, MIXED, bits=fmt, average=True)
        kw = dict(lanes=1, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS) if kind == "SRA" else {}
        assert_results(out, ref(xs, MIXED, fmt=fmt, average=True, **kw), f"generic {kind}")
    for root in {0, world - 1}:
        out = [x.clone() for x in xs]
        _C.LocalReducerGroup(world, "SRA", 5000).broadcast_compressed(out, MIXED, root, bits=fmt)
        assert_results(out, O.broadcast_compressed_reference(xs, MIXED, root=root, fmt=fmt), f"bcast root {root}")
    full = [x.repeat(world) for x in xs]
    g = _C.LocalReducerGroup(world, "SRA", 5000)
    outs = [torch.empty(S_MIXED, dtype=dtype) for _ in range(world)]
    g.reduce_scatter(full, outs, MIXED, average=True, bits=fmt)
    assert_results(outs, _rs(full, MIXED, fmt, average=True), "generic rs")


ENGINE = [dict(world=4, local=2, inner="SRA", cross="RING", bcast=True, icomp=True),
          dict(world=6, local=3, inner="RING", cross="SRA", bcast=True, icomp=True),
          dict(world=8, local=4, inner="SRA", cross="SRA", bcast=True, icomp=False)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("h", ENGINE, ids=lambda h: f"w{h['world']}l{h['local']}")
def test_engine_stages(h, fmt):
    cfg = dict(inner_reduction=h["inner"], cross_reduction=h["cross"], intra_broadcast=h["bcast"],
               intra_compress=h["icomp"], p2p=False, fusion_bytes=8192)
    layers, total = mixed_table([(37, 32, 512), (9000, 8, 512), (2001, 8, 64), (700, 8, 100), (513, 8, 1)])
    world, local = h["world"], h["local"]
    g = _C.LocalEngineGroup(world, local, cfg, 1, 1 << 16, TIMEOUT_MS)
    state = inputs_for(world, total, torch.bfloat16, world * 7 + local)
    want, _ = O.engine_reference(state, layers, local_size=local, config=cfg, lanes=1, call_seq=1, cuda=False,
                                 fmt=fmt)
    g.allreduce_layers(state, layers, False, bits=fmt)
    assert_results(state, want, "engine")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,local", [(4, 1), (4, 2), (6, 3)])
def test_two_stage_sharded(world, local, fmt):
    g = _C.LocalEngineGroup(world, local, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    xs = _inputs(world, world * S_MIXED, torch.bfloat16, world + local)
    own = [xs[r][r * S_MIXED:(r + 1) * S_MIXED].clone() for r in range(world)]
    outs = [torch.empty(world * S_MIXED, dtype=torch.bfloat16) for _ in range(world)]
    g.all_gather(own, outs, MIXED, bits=fmt)
    assert_results(outs, [O.all_gather_reference(own, MIXED, fmt)] * world, "two-stage ag")
    outs = [torch.empty(S_MIXED, dtype=torch.bfloat16) for _ in range(world)]
    g.reduce_scatter(xs, outs, True, MIXED, bits=fmt)
    if local == 1:
        assert_results(outs, O.reduce_scatter_reference(xs, MIXED, average=True, fmt=fmt), "two-stage rs")
    else:
        want = O.reduce_scatter_hier_reference(xs, MIXED, local_size=local, average=True, fmt=fmt)
        assert_results(outs, want, "two-stage rs")


# ---- the front ends --------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_names_accepted_everywhere(fmt, monkeypatch):
    for op in ("all_to_all", "allreduce", "reduce_scatter", "all_gather"):
        assert tuple(_C.a2a_bits(fmt, False, op)) == (8, 3 if fmt == "e4m3_pow2" else 4)
    with cgx.compression(bits=fmt):
        assert os.environ["CGX_COMPRESSION_FORMAT"] == fmt
        assert os.environ["CGX_COMPRESSION_QUANTIZATION_BITS"] == "8"
    st = cgx.CGXState(None, compression_params={"bits": fmt, "bucket_size": 256})
    assert (st.quantization_bits, st.quantization_format) == (8, fmt)
    assert H._width_and_format(fmt) == (8, fmt)
    params = [((16, 8), 128), ((16,), 16)]
    assert FS.fsdp_shard_table(params, fmt, 64) == [(0, 128, 8, 64), (128, 16, 32, 64)]
    assert FS.CGXReduceScatter(fmt).bits == fmt and FS.CGXAllGather(fmt).bits == fmt
    # CGX_COMPRESSION_FORMAT selects the format in the engine
    layers, total = mixed_table([(9000, 8, 512), (700, 8, 100)])
    eg = _C.LocalEngineGroup(2, 2, dict(p2p=False, fusion_bytes=8192), 1, 1 << 16, TIMEOUT_MS)
    state = inputs_for(2, total, torch.float16, 1)
    want, _ = O.engine_reference(state, layers, local_size=2, config=dict(p2p=False, fusion_bytes=8192), lanes=1,
                                 cuda=False, fmt=fmt)
    monkeypatch.setenv("CGX_COMPRESSION_FORMAT", fmt)
    eg.allreduce_layers(state, layers, False)
    assert_results(state, want, f"CGX_COMPRESSION_FORMAT={fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_refusals_before_anything_is_sent(fmt, monkeypatch):
    xs = _inputs(2, 512, torch.float32, 0)
    before = [x.clone() for x in xs]
    with pytest.raises(ValueError, match="round"):
        _C.a2a_bits(fmt, True, "all_to_all")
    with pytest.raises(ValueError, match="round"):
        cgx.all_reduce(torch.ones(64), bits=fmt, stochastic=True)
    with pytest.raises(ValueError, match="round"):
        cgx.reduce_scatter_tensor(torch.empty(64), torch.empty(128), bits=fmt, stochastic=True)
    with pytest.raises(ValueError, match="round"):
        cgx.all_to_all_single(torch.empty(4, 512), torch.randn(4, 512), bits=fmt, stochastic=True)
    with pytest.raises(ValueError, match="round"):
        cgx.compression(bits=fmt, stochastic=True).__enter__()
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveCGXState(None, compression_params={"bits": fmt})
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveFSDPState(reduce_scatter_bits=fmt)
    with pytest.raises(ValueError, match="adaptive"):
        FS.CGXAllGather(fmt, adaptive=object())
    # codes of the other base format
    other = torch.float8_e5m2 if fmt == "e4m3_pow2" else torch.float8_e4m3fn
    x = torch.randn(4, 512)
    with pytest.raises(ValueError, match="float8"):
        cgx.all_to_all_single(torch.empty(4, 512, dtype=other), x, bits=fmt, bucket_size=128,
                              output_scales=torch.empty(4, 4))
    with pytest.raises(ValueError, match="float8"):
        cgx.all_gather_into_tensor(torch.empty(2048, dtype=other), x.reshape(-1), bits=fmt, bucket_size=128,
                                   output_scales=torch.empty(16))
    c = [[256, 256], [256, 256]]
    outs = [torch.empty(512, dtype=other) for _ in range(2)]
    with pytest.raises(RuntimeError):
        _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=128, output_scales=[torch.empty(4)] * 2)
    for kind in ("SRA", "RING"):
        g = _C.LocalReducerGroup(2, kind, 5000)
        with pytest.raises(ValueError, match="round"):
            g.allreduce(xs, [(0, 512, 8, 32)], stochastic=True, bits=fmt)
        with pytest.raises(ValueError, match="bits 8 or 32"):
            g.allreduce(xs, [(0, 256, 8, 32), (256, 256, 4, 32)], bits=fmt)
        assert g.bytes_sent() == [0, 0]
    eg = _C.LocalEngineGroup(2, 2, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    monkeypatch.setenv("CGX_STOCHASTIC_ROUNDING", "1")
    with pytest.raises((ValueError, RuntimeError), match="round"):
        eg.allreduce_layers(xs, [(0, 512, 8, 32)], False, bits=fmt)
    assert all(eg.stats(r)["calls"] == 0 and eg.stats(r)["wire_bytes"] == 0 for r in range(2))
    for o, b in zip(xs, before):
        assert torch.equal(o, b)
