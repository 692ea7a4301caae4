"""FP8 wire formats of the compressed all-to-all without a GPU: the host codec (the simulator's)
against the independent numpy / torch.float8 reference on every code, every rounding midpoint and
one fp32 ulp either side of it, the simulator against the reference over the shared case matrix and
the edge inputs, the error bounds, the generic reducer on host memory, and the argument checks."""
from __future__ import annotations

import itertools

import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import functional as F

from _a2a_cases import BUCKETS, DTYPES, SPLITS, WORLDS, base_elems, counts, inputs, outputs
from _bitwise import assert_same
from _edge_inputs import edge_inputs

FMTS = ("e4m3", "e5m2")
FMAX = {"e4m3": 448.0, "e5m2": 57344.0}
TDT = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
F32 = np.float32


def _simulate(xs, c, bits, bucket, **kw):
    outs = outputs(c, xs[0].dtype)
    _C.all_to_all_simulate(xs, outs, c, bits=bits, bucket_size=bucket, **kw)
    return outs


def _check(xs, c, bits, bucket, what):
    got = _simulate(xs, c, bits, bucket)
    ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket)
    for r in range(len(xs)):
        assert_same(got[r], ref[r], f"{what} rank {r}")
    return got


def _one_chunk(x, bits, bucket):
    """x travels from rank 0 to rank 1 (world 2): the simulator's decode of it, and the reference's"""
    n = x.numel()
    c = [[0, n], [0, 0]]
    xs = [x, x.new_zeros(0)]
    got = _simulate(xs, c, bits, bucket)[1]
    ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket)[1]
    return got, ref


# ---- the codec on crafted buckets --------------------------------------------------------------
def _codes(fmt):
    """the finite values of the format, ascending, one per magnitude and sign (-0 included)"""
    v = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(TDT[fmt]).float()
    v = v[torch.isfinite(v)]
    return np.unique(v.numpy().astype(F32))


def _unit_one_scale(fmt):
    """a bucket maximum a near FMAX for which unit = fp32(a * fp32(1/FMAX)) is exactly 1, so that the
    codes are x itself"""
    r = F32(1.0) / F32(FMAX[fmt])
    a = F32(FMAX[fmt])
    for _ in range(64):
        if F32(a * r) == F32(1.0):
            return a
        a = np.nextafter(a, F32(np.inf) if F32(a * r) < 1 else F32(0))
    raise AssertionError("no scale with unit 1")


def _targets(fmt):
    """every code, every midpoint between adjacent codes and one fp32 ulp either side of each, both
    signs, plus fp32 subnormals; all within [-FMAX, FMAX]"""
    pos = _codes(fmt)
    pos = pos[pos >= 0]
    mids = ((pos[:-1].astype(np.float64) + pos[1:]) / 2).astype(F32)
    around = np.concatenate([mids, np.nextafter(mids, F32(0)), np.nextafter(mids, F32(np.inf))])
    vals = np.concatenate([pos, around, np.array([1e-40, 1e-45, 2.0 ** -126], F32)])
    vals = vals[vals <= FMAX[fmt]]
    return np.concatenate([vals, -vals]).astype(F32)


@pytest.mark.parametrize("fmt", FMTS)
def test_codec_every_code_and_midpoint(fmt):
    a = _unit_one_scale(fmt)
    t = _targets(fmt)
    B = 512
    # every bucket starts with the scale value a, so unit = 1 and x * inv = x: the codes are the targets
    rows = [np.concatenate([[a], t[i:i + B - 1]]) for i in range(0, t.size, B - 1)]
    rows[-1] = np.concatenate([rows[-1], np.zeros(B - rows[-1].size, F32)])
    x = torch.from_numpy(np.concatenate(rows).astype(F32))
    got, ref = _one_chunk(x, fmt, B)
    assert_same(got, ref, fmt)
    # an exact code decodes to itself; the rest lands on one of the two neighbouring codes
    codes = _codes(fmt)
    xv, gv = x.numpy(), got.numpy()
    exact = np.isin(xv, codes) & (xv != a)
    assert np.array_equal(gv[exact].view(np.int32), xv[exact].view(np.int32))
    assert np.isin(np.abs(gv[xv != a]), np.abs(codes)).all()
    # a tie goes to the even code (the one whose last mantissa bit is 0)
    pos = codes[codes > 0]
    mids = ((pos[:-1].astype(np.float64) + pos[1:]) / 2).astype(F32)
    ties = torch.from_numpy(gv[np.isin(xv, mids)].copy()).to(TDT[fmt]).view(torch.uint8)
    assert ties.numel() > 0 and bool(((ties & 1) == 0).all())


@pytest.mark.parametrize("fmt", FMTS)
def test_codec_unit_threshold_and_saturation_edge(fmt):
    fm, B = FMAX[fmt], 64
    g = torch.Generator().manual_seed(7)
    rows = []
    # largest magnitude just below / above FMAX * 2^-126: unit on either side of the threshold
    for s in (0.97, 0.999, 1.001, 1.03):
        r = (torch.rand(B, generator=g, dtype=torch.float64) * 2 - 1) * (fm * 2.0 ** -126 * s)
        r[5] = fm * 2.0 ** -126 * s
        rows.append(r.float())
    # the FMAX edge: values at and one ulp below the bucket maximum, at every scale
    for top in (1.0, fm, 3.0e38, 1e-30):
        r = torch.tensor([top, -top, np.nextafter(F32(top), F32(0)), top * 0.999, top / fm], dtype=torch.float32)
        rows.append(torch.cat([r, torch.rand(B - r.numel(), generator=g) * top]))
    x = torch.cat(rows)
    got, ref = _one_chunk(x, fmt, B)
    assert_same(got, ref, fmt)
    below = got[:2 * B]
    assert bool((below == 0).all()), "a unit below 2^-126 decodes to zeros"
    assert bool((got[2 * B + 5: 4 * B] != 0).any())
    assert bool(torch.isfinite(got).all())


def test_codec_distinguishes_formats_and_max_min():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4096, generator=g)
    e4, _ = _one_chunk(x, "e4m3", 512)
    e5, _ = _one_chunk(x, "e5m2", 512)
    mm, _ = _one_chunk(x, 8, 512)
    assert not torch.equal(e4, e5) and not torch.equal(e4, mm) and not torch.equal(e5, mm)
    # the reference tells them apart too, so matching it is not vacuous
    ref = {b: O.all_to_all_reference([x, x[:0]], [[0, 4096], [0, 0]], bits=b, bucket_size=512)[1]
           for b in ("e4m3", "e5m2", 8)}
    assert not torch.equal(ref["e4m3"], ref["e5m2"]) and not torch.equal(ref["e4m3"], ref[8])


# ---- non-finite and zero buckets ---------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_poisoned_and_zero_buckets(fmt, dtype):
    B = 64
    g = torch.Generator().manual_seed(2)
    x = torch.randn(8 * B, generator=g).to(dtype)
    x[B + 3] = float("nan")
    x[2 * B + 9] = float("inf")
    x[3 * B:4 * B] = float("-inf")
    x[4 * B:5 * B] = 0.0
    x[5 * B:6 * B] = -0.0
    x[6 * B:7 * B] = torch.where(torch.arange(B) % 2 == 0, 0.0, -0.0).to(dtype)
    got, ref = _one_chunk(x, fmt, B)
    assert_same(got, ref, f"{fmt} {dtype}")
    for k in (1, 2, 3):
        assert bool(torch.isnan(got[k * B:(k + 1) * B]).all()), f"bucket {k} must decode to NaN"
    assert_same(got[4 * B:7 * B], x[4 * B:7 * B], "signed zeros survive")
    assert bool(torch.isfinite(got[:B]).all() & torch.isfinite(got[7 * B:]).all())


# ---- the simulator against the reference ------------------------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, BUCKETS)))
def test_simulator_matches_reference(dtype, fmt, bucket):
    i = DTYPES.index(dtype) * 5 + FMTS.index(fmt) * 3 + BUCKETS.index(bucket)
    W = WORLDS[i % len(WORLDS)]
    base = base_elems(bucket) if W <= 5 else max(300, min(base_elems(bucket), 2000))
    kind = SPLITS[i % len(SPLITS)]
    c = counts(W, kind, base, seed=i)
    _check(inputs(c, dtype, i), c, fmt, bucket, f"W={W} {kind}")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind", SPLITS)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_every_world_and_split(world, kind, fmt):
    c = counts(world, kind, 700, seed=world)
    _check(inputs(c, torch.bfloat16, world), c, fmt, 512, f"W={world} {kind}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_edge_inputs(dtype, fmt):
    W, bucket = 3, 64
    n = 40 * bucket
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=5, world=W, bits=8)
    assert planted
    _check(xs, [[n] * W for _ in range(W)], fmt, bucket, "edge")


# ---- error bounds ------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,rel", [("e4m3", 2.0 ** -4), ("e5m2", 2.0 ** -3)])
def test_relative_error_bound(fmt, rel):
    g = torch.Generator().manual_seed(11)
    B = 512
    x = torch.randn(64 * B, generator=g, dtype=torch.float64)
    x[::97] *= 50.0  # outlier channels: the bound holds whatever else the bucket holds
    x = x.float()
    got, _ = _one_chunk(x, fmt, B)
    xb, gb = x.reshape(-1, B).double(), got.reshape(-1, B).double()
    unit = xb.abs().amax(dim=1, keepdim=True) / FMAX[fmt]
    # normal range of the format: |x| / unit at least the smallest normal, 2^-6 (e4m3) / 2^-14 (e5m2)
    normal = xb.abs() / unit >= (2.0 ** -6 if fmt == "e4m3" else 2.0 ** -14)
    err = (gb - xb).abs()
    # half an ulp of the format (2^-4 / 2^-3 of the value at worst), plus the fp32 roundings of the scale
    bound = xb.abs() * rel * (1 + 2.0 ** -18)
    assert bool((err[normal] <= bound[normal]).all())
    assert bool((err[normal] > 0).any())  # not vacuous
    # max-min 8-bit loses far more on the small channels of a bucket with an outlier
    mm, _ = _one_chunk(x, 8, B)
    small = (xb.abs() < 1) & (xb.abs() > 0.1)
    mm_rel = ((mm.reshape(-1, B).double() - xb).abs() / xb.abs())[small].max()
    assert float(mm_rel) > rel


# ---- the generic reducer on host memory ---------------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 512), ("e5m2", 1024), ("e4m3", 7), ("e5m2", 10000)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_reducer_matches_simulator(fmt, bucket, dtype):
    W = 3
    c = counts(W, "uneven", 3000, seed=bucket)
    xs = inputs(c, dtype, bucket)
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    outs = outputs(c, dtype)
    red.all_to_all(xs, outs, c, bits=fmt, bucket_size=bucket)
    sim = _simulate(xs, c, fmt, bucket)
    for r in range(W):
        assert_same(outs[r], sim[r], f"rank {r}")


def test_generic_reducer_edge_inputs_and_messages():
    W, bucket, dtype = 3, 64, torch.float32
    n = 40 * bucket
    xs, _ = edge_inputs(dtype, n * W, bucket, seed=3, world=W, bits=8)
    c = [[n] * W for _ in range(W)]
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    red.set_recording(True)
    outs = outputs(c, dtype)
    red.all_to_all(xs, outs, c, bits="e4m3", bucket_size=bucket)
    sim = _simulate(xs, c, "e4m3", bucket)
    for r in range(W):
        assert_same(outs[r], sim[r], f"rank {r}")
    msgs = red.messages()
    assert len(msgs) == W * (W - 1)
    for _, src, dst, m in msgs:
        assert m.numel() == n + 8 * (n // bucket)  # the 8-bit record: one byte per element, 8 per bucket


# ---- arguments ----------------------------------------------------------------------------------
def test_bits_parser():
    assert _C.a2a_bits("e4m3") == (8, 1)
    assert _C.a2a_bits("e5m2") == (8, 2)
    assert _C.a2a_bits(8) == (8, 0) and _C.a2a_bits(32) == (32, 0)
    with pytest.raises(ValueError, match="e4m3"):
        _C.a2a_bits("fp8")
    with pytest.raises(ValueError, match="round"):
        _C.a2a_bits("e5m2", True)
    xs, c = [torch.zeros(4), torch.zeros(4)], [[2, 2], [2, 2]]
    for bad in ("E4M3", "int8", ""):
        with pytest.raises(ValueError):
            _C.all_to_all_simulate(xs, [torch.zeros(4)] * 2, c, bits=bad)
        with pytest.raises(ValueError):
            _C.LocalReducerGroup(2, "SRA", 5000).all_to_all(xs, [torch.zeros(4)] * 2, c, bits=bad)
    with pytest.raises(ValueError, match="round"):
        _C.all_to_all_simulate(xs, [torch.zeros(4)] * 2, c, bits="e4m3", stochastic=True)
    with pytest.raises(ValueError):
        O.all_to_all_reference(xs, c, bits="e3m4", bucket_size=64)


def test_public_api_rejects_before_sending(monkeypatch):
    sent = []
    monkeypatch.setattr(F, "all_to_all_single", lambda *a, **k: sent.append(k))
    x = torch.zeros(4, 2, requires_grad=True)
    with pytest.raises(ValueError):
        cgx.differentiable_all_to_all_single(x, bits="e4m3", stochastic=True)
    with pytest.raises(ValueError):
        cgx.differentiable_all_to_all_single(x, bits=8, grad_bits="e5m2", stochastic=True)
    with pytest.raises(ValueError):
        cgx.differentiable_all_to_all_single(x, bits=8, grad_bits="e6m1")
    with pytest.raises(ValueError):
        cgx.differentiable_all_to_all_single(x, bits="bf8")
    assert not sent
    # the public function itself checks before it looks for a process group
    with pytest.raises(ValueError):
        cgx.all_to_all_single(torch.zeros(4), torch.zeros(4), bits="e4m3", stochastic=True)


def test_differentiable_fp8_recipe_world1(monkeypatch):
    """at world 1 the exchange is the own chunk's copy: bits and grad_bits reach the forward and the
    backward calls unchanged, and the result is the identity"""
    calls = []

    def world1(output, input, output_split_sizes=None, input_split_sizes=None, bits=8, bucket_size=512,
               group=None, async_op=False, stochastic=False, seed=None, **kw):
        calls.append((bits, bucket_size))
        output.copy_(input)

    monkeypatch.setattr(F, "all_to_all_single", world1)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(6, 8, generator=g, requires_grad=True)
    y = cgx.differentiable_all_to_all_single(x, [6], [6], bits="e4m3", grad_bits="e5m2", bucket_size=128)
    w = torch.randn(6, 8, generator=g)
    (y * w).sum().backward()
    assert calls == [("e4m3", 128), ("e5m2", 128)]
    assert_same(y.detach(), x.detach())
    assert_same(x.grad, w)
    calls.clear()
    y = cgx.differentiable_all_to_all_single(x, [6], [6], bits="e5m2")
    y.sum().backward()
    assert calls == [("e5m2", 512), ("e5m2", 512)]  # grad_bits=None means bits
