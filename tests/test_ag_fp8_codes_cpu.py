"""The FP8 all-gather's codes output without a GPU: the simulator's codes and scales against the
oracle byte for byte (NaN-aware) over dtypes, formats, buckets, worlds and the edge inputs; the
decode identity against the decoded call; the host generic reducer against the simulator, with the
decoded call's wire; and every refusal of the public call, which fires before anything is sent."""
from __future__ import annotations

import itertools

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import DTYPES
from _ag_codes_cases import (BUCKET_SHARDS, FMTS, TDT, WORLDS, assert_codes, codes_buffers, decode, shards,
                             simulate_codes, table)
from _bitwise import assert_same
from _edge_inputs import edge_inputs


def check_against_oracle(xs, fmt, bucket, what):
    got_c, got_s = simulate_codes(xs, fmt, bucket)
    ref_c, ref_s = O.all_gather_codes_reference(xs, fmt, bucket)
    for r in range(len(xs)):
        assert_codes(got_c[r], ref_c, f"{what} rank {r} codes")
        assert_same(got_s[r], ref_s, f"{what} rank {r} scales")
    return got_c, got_s


# ---- the simulator against the oracle -----------------------------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, BUCKET_SHARDS)))
def test_simulator_matches_oracle(dtype, fmt, bucket):
    i = DTYPES.index(dtype) * 7 + FMTS.index(fmt) * 3 + list(BUCKET_SHARDS).index(bucket)
    W = WORLDS[i % len(WORLDS)]
    S = BUCKET_SHARDS[bucket] if W <= 3 else bucket * 2
    check_against_oracle(shards(W, S, dtype, i), fmt, bucket, f"W={W} S={S} B={bucket}")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_every_world(world, fmt):
    check_against_oracle(shards(world, 2048, torch.bfloat16, world), fmt, 128, f"W={world}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_edge_inputs(dtype, fmt):
    W, bucket = 3, 64
    xs, planted = edge_inputs(dtype, 40 * bucket, bucket, seed=5, world=W, bits=8)
    assert planted
    got_c, got_s = check_against_oracle(xs, fmt, bucket, "edge")
    # the rules of the wire format: zero buckets have unit +0, NaN / Inf buckets a NaN / Inf unit
    s = got_s[0]
    assert bool((s.isnan() | s.isinf()).any()) and bool((s == 0).any())
    assert not bool(torch.signbit(s[s == 0]).any()), "a zero bucket's unit is +0"


# ---- decoding the codes gives the decoded call, bit for bit ---------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [64, 100, 128, 7168])
@pytest.mark.parametrize("edge", [False, True])
def test_decode_identity(dtype, fmt, bucket, edge):
    W = 3
    S = BUCKET_SHARDS[bucket]
    if edge:
        S = 40 * bucket
        xs, _ = edge_inputs(dtype, S, bucket, seed=bucket, world=W, bits=8)
    else:
        xs = shards(W, S, dtype, bucket)
    codes, scales = simulate_codes(xs, fmt, bucket)
    dec = [torch.full((W * S,), float("nan"), dtype=dtype) for _ in range(W)]
    _C.all_gather_simulate(xs, dec, table(S, bucket), bits=fmt)
    for r in range(W):
        assert_same(decode(codes[r], scales[r], bucket, dtype), dec[r], f"rank {r}")


# ---- the host generic reducer -------------------------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", 7168),
                                        ("e4m3", 8192)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_reducer_matches_simulator(fmt, bucket, dtype):
    W, S = 3, BUCKET_SHARDS[bucket]
    xs = shards(W, S, dtype, bucket)
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    red.set_recording(True)
    codes, scales = codes_buffers(W, S, bucket, fmt)
    red.all_gather(xs, codes, table(S, bucket), bits=fmt, output_scales=scales)
    codes_msgs = red.messages()
    sim_c, sim_s = simulate_codes(xs, fmt, bucket)
    for r in range(W):
        assert_codes(codes[r], sim_c[r], f"rank {r}")
        assert_same(scales[r], sim_s[r], f"rank {r}")
    # the wire is the decoded FP8 call's, byte for byte
    red.all_gather(xs, [torch.empty(W * S, dtype=dtype) for _ in range(W)], table(S, bucket), bits=fmt)
    dec_msgs = red.messages()
    assert len(codes_msgs) == len(dec_msgs) == W * (W - 1)
    for (_, s1, d1, m1), (_, s2, d2, m2) in zip(codes_msgs, dec_msgs):
        assert (s1, d1) == (s2, d2) and torch.equal(m1, m2)


def test_generic_reducer_uint8_outputs_world1():
    x = torch.randn(4 * 256)
    codes, scales = [torch.zeros(x.numel(), dtype=torch.uint8)], [torch.zeros(x.numel() // 256)]
    _C.LocalReducerGroup(1, "SRA", 5000).all_gather([x], codes, table(x.numel(), 256), bits="e5m2",
                                                    output_scales=scales)
    ref_c, ref_s = O.fp8_quantize(x, "e5m2", 256)
    assert torch.equal(codes[0], ref_c.view(torch.uint8))
    assert_same(scales[0], ref_s)


# ---- refusals -----------------------------------------------------------------------------------
def test_native_refusals():
    W, S, B = 2, 512, 128
    xs = shards(W, S, torch.float32, 0)
    codes, scales = codes_buffers(W, S, B, "e4m3")
    sim = _C.all_gather_simulate
    with pytest.raises(ValueError, match="e4m3"):  # integer bits
        sim(xs, [c.view(torch.uint8) for c in codes], table(S, B), bits=8, output_scales=scales)
    with pytest.raises(ValueError, match="round"):
        sim(xs, codes, table(S, B), bits="e4m3", stochastic=True, output_scales=scales)
    with pytest.raises(ValueError, match="8192"):
        sim(xs, codes, table(S, 16384), bits="e4m3", output_scales=scales)
    with pytest.raises(ValueError, match="divides"):  # S % B != 0
        sim(xs, codes, table(S, 100), bits="e4m3", output_scales=scales)
    with pytest.raises(ValueError, match="bits 8"):  # a raw layer has no codes
        sim(xs, codes, [(0, 256, 8, B), (256, 256, 32, B)], bits="e4m3", output_scales=scales)
    with pytest.raises(RuntimeError):  # a float8 of the other format
        sim(xs, [c.view(torch.float8_e5m2) for c in codes], table(S, B), bits="e4m3", output_scales=scales)
    with pytest.raises(RuntimeError):  # scales of the wrong size
        sim(xs, codes, table(S, B), bits="e4m3", output_scales=[s[:1] for s in scales])
    with pytest.raises(RuntimeError):  # scales of the wrong dtype
        sim(xs, codes, table(S, B), bits="e4m3", output_scales=[s.double() for s in scales])
    # the generic reducer checks the same, and refuses codes and scales that overlap the input or each other
    red = _C.LocalReducerGroup(1, "SRA", 5000)
    y = torch.randn(1024)
    t = table(512, B)
    with pytest.raises((ValueError, RuntimeError), match="overlap"):
        red.all_gather([y[:512]], [y.view(torch.uint8)[1024:1536]], t, bits="e4m3", output_scales=[torch.zeros(4)])
    with pytest.raises((ValueError, RuntimeError), match="overlap"):
        red.all_gather([y[:512]], [torch.zeros(512, dtype=torch.uint8)], t, bits="e4m3", output_scales=[y[:4]])
    buf = torch.zeros(1024, dtype=torch.uint8)
    with pytest.raises((ValueError, RuntimeError), match="overlap"):
        red.all_gather([y[:512]], [buf[:512]], t, bits="e4m3", output_scales=[buf[256:272].view(torch.float32)])


def _public(out, x, scales, **kw):
    kw.setdefault("bits", "e4m3")
    kw.setdefault("bucket_size", 128)
    cgx.all_gather_into_tensor(out, x, output_scales=scales, **kw)


def test_public_api_refusals_before_sending():
    """every check the public call can make on its arguments raises ValueError before it looks for a
    process group (there is none here)"""
    x = torch.randn(4, 512)
    codes = torch.empty(4, 512, dtype=torch.float8_e4m3fn)
    scales = torch.empty(4, 4)
    cases = [
        dict(bits=8),                                                   # integer bits
        dict(bits=4, stochastic=True),
        dict(bits="e4m3", stochastic=True),                             # FP8 rounds to nearest only
        dict(bits="e5m2"),                                              # codes of the other format
        dict(bucket_size=3),                                            # S % bucket != 0
        dict(bucket_size=16384),                                        # bucket > 8192
        dict(layers=[(0, 2048, 8, 128)]),                               # any layers table
        dict(layers=[(0, 1024, 8, 128), (1024, 1024, 32, 128)]),
    ]
    for kw in cases:
        with pytest.raises(ValueError):
            _public(codes, x, scales, **kw)
    with pytest.raises(ValueError, match="output_scales"):  # host scales (the CUDA cases are in the GPU tier)
        _public(codes, x, scales)
    with pytest.raises(ValueError, match="float8"):
        _public(torch.empty(4, 512, dtype=torch.uint8), x, scales)
    with pytest.raises(ValueError, match="float8"):
        _public(torch.empty(4, 512, dtype=torch.bfloat16), x, scales)


def test_reference_is_fp8_quantize_of_each_shard():
    xs = shards(3, 1024, torch.float16, 9)
    c, u = O.all_gather_codes_reference(xs, "e5m2", 256)
    assert c.dtype == TDT["e5m2"] and c.numel() == 3 * 1024 and u.numel() == 3 * 4
    for q in range(3):
        rc, ru = O.fp8_quantize(xs[q], "e5m2", 256)
        assert torch.equal(c[q * 1024:(q + 1) * 1024].view(torch.uint8), rc.view(torch.uint8))
        assert_same(u[q * 4:(q + 1) * 4], ru)
