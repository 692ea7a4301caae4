"""The FP8 all-to-all's codes output without a GPU: the simulator's codes and scales against the
oracle byte for byte (NaN-aware) over dtypes, formats, buckets, worlds, splits and the edge inputs;
the decode of the peers' rows against the decoded call; the host generic reducer against the
simulator; and every refusal of the public call, which fires before anything is sent."""
from __future__ import annotations

import itertools

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import DTYPES, inputs
from _bitwise import assert_same
from _edge_inputs import edge_inputs

FMTS = ("e4m3", "e5m2")
TDT = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
# bucket -> row length H (a multiple of it); "H" is one bucket per row
BUCKET_ROWS = {64: 512, 100: 1000, 128: 1024, 512: 1536, 1024: 2048, "H": 7168}
CODES_WORLDS = (1, 2, 3, 8, 16)
CODES_SPLITS = ("equal", "uneven", "empty")


def row_counts(world: int, kind: str, rows: int, H: int, seed: int):
    """counts of whole rows of H elements: rows each, random in [0, 2 rows], or none"""
    g = torch.Generator().manual_seed(seed)
    if kind == "equal":
        m = [[rows] * world for _ in range(world)]
    elif kind == "empty":
        m = [[0] * world for _ in range(world)]
    else:
        m = torch.randint(0, 2 * rows + 1, (world, world), generator=g).tolist()
    return [[v * H for v in row] for row in m]


def codes_outputs(c, bucket, fmt, device="cpu"):
    """per rank: codes (the format's float8, filled with 0x55) and scales (NaN)"""
    W = len(c)
    outs, scales = [], []
    for r in range(W):
        n = sum(c[q][r] for q in range(W))
        outs.append(torch.full((n,), 0x55, dtype=torch.uint8, device=device).view(TDT[fmt]))
        scales.append(torch.full((n // bucket,), float("nan"), dtype=torch.float32, device=device))
    return outs, scales


def simulate_codes(xs, c, fmt, bucket):
    outs, scales = codes_outputs(c, bucket, fmt)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=bucket, output_scales=scales)
    return outs, scales


def assert_codes(got, ref, what=""):
    """FP8 codes byte for byte, except that any NaN code equals any other"""
    got, ref = got.detach().cpu().reshape(-1), ref.detach().cpu().reshape(-1)
    assert got.dtype == ref.dtype and got.numel() == ref.numel(), f"{what}: {got.dtype}/{got.numel()} vs {ref.dtype}/{ref.numel()}"
    gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
    assert torch.equal(gn, rn), f"{what}: NaN codes differ at {int((gn != rn).nonzero()[0])}"
    diff = (got.view(torch.uint8) != ref.view(torch.uint8)) & ~gn
    assert not diff.any(), f"{what}: {int(diff.sum())} codes differ, first at {int(diff.nonzero()[0])}"


def check_against_oracle(xs, c, fmt, bucket, what):
    got_c, got_s = simulate_codes(xs, c, fmt, bucket)
    ref_c, ref_s = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=bucket)
    for r in range(len(xs)):
        assert_codes(got_c[r], ref_c[r], f"{what} rank {r} codes")
        assert_same(got_s[r], ref_s[r], f"{what} rank {r} scales")
    return got_c, got_s


def _bucket(b):
    return BUCKET_ROWS["H"] if b == "H" else b


# ---- the simulator against the oracle -----------------------------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, BUCKET_ROWS)))
def test_simulator_matches_oracle(dtype, fmt, bucket):
    H, B = BUCKET_ROWS[bucket], _bucket(bucket)
    i = DTYPES.index(dtype) * 7 + FMTS.index(fmt) * 3 + list(BUCKET_ROWS).index(bucket)
    W = CODES_WORLDS[i % len(CODES_WORLDS)]
    c = row_counts(W, CODES_SPLITS[i % len(CODES_SPLITS)], 3 if W <= 3 else 1, H, seed=i)
    check_against_oracle(inputs(c, dtype, i), c, fmt, B, f"W={W} H={H} B={B}")


@pytest.mark.parametrize("world", CODES_WORLDS)
@pytest.mark.parametrize("kind", CODES_SPLITS)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_every_world_and_split(world, kind, fmt):
    c = row_counts(world, kind, 2, 1024, seed=world)
    check_against_oracle(inputs(c, torch.bfloat16, world), c, fmt, 128, f"W={world} {kind}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_simulator_edge_inputs(dtype, fmt):
    W, bucket = 3, 64
    n = 40 * bucket
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=5, world=W, bits=8)
    assert planted
    got_c, got_s = check_against_oracle(xs, [[n] * W for _ in range(W)], fmt, bucket, "edge")
    # the rules of the wire format: zero buckets have unit +0, NaN / Inf buckets a NaN / Inf unit
    s = torch.cat(got_s)
    assert bool((s.isnan() | s.isinf()).any()) and bool((s == 0).any())
    assert not bool(torch.signbit(s[s == 0]).any()), "a zero bucket's unit is +0"


# ---- decoding the codes gives the decoded call ---------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [128, "H"])
def test_decoded_codes_equal_decoded_call(dtype, fmt, bucket):
    H, B = BUCKET_ROWS[bucket], _bucket(bucket)
    W = 3
    c = row_counts(W, "uneven", 2, H, seed=B)
    xs = inputs(c, dtype, B)
    codes, scales = simulate_codes(xs, c, fmt, B)
    dec = [torch.full((codes[r].numel(),), float("nan"), dtype=dtype) for r in range(W)]
    _C.all_to_all_simulate(xs, dec, c, bits=fmt, bucket_size=B)
    for r in range(W):
        mine = (codes[r].float().reshape(-1, B) * scales[r][:, None]).reshape(-1).to(dtype)
        off = 0
        for q in range(W):
            n = c[q][r]
            if q != r:  # the decoded call copies the own chunk; the codes output encodes it
                assert_same(mine[off:off + n], dec[r][off:off + n], f"rank {r} from {q}")
            off += n


def test_fp8_quantize_is_the_round_trip():
    g = torch.Generator().manual_seed(3)
    for fmt, B, dtype in itertools.product(FMTS, (7, 64, 100, 8192, 10000), DTYPES):
        x = (torch.randn(3000, generator=g) * 40).to(dtype)
        codes, units = O.fp8_quantize(x, fmt, B)
        b = min(B, 8192)
        assert codes.dtype == TDT[fmt] and codes.numel() == 3000 and units.numel() == -(-3000 // b)
        pad = torch.zeros(units.numel() * b - 3000)
        dec = (torch.cat([codes.float(), pad]).reshape(-1, b) * units[:, None]).reshape(-1)[:3000]
        assert_same(dec.to(dtype), O.fp8_quantize_dequantize(x, fmt, B), f"{fmt} B={B} {dtype}")


def test_routed_oracle_is_the_composition():
    W, H, B, fmt = 2, 512, 128, "e4m3"
    g = torch.Generator().manual_seed(1)
    xs = [torch.randn(5, H, generator=g) for _ in range(W)]
    ii = [torch.tensor([4, 0, 4]), torch.tensor([1, 2, 3])]
    oi = [torch.tensor([3, 1, 0]), torch.tensor([2, 0, 5])]
    c = [[H, 2 * H], [2 * H, H]]
    base = [torch.full((6 * H,), 0x11, dtype=torch.uint8).view(TDT[fmt]) for _ in range(W)]
    bs = [torch.full((6 * H // B,), -1.0) for _ in range(W)]
    got_c, got_s = O.routed_all_to_all_codes_reference(xs, c, ii, oi, H, fmt=fmt, bucket_size=B, outputs=base,
                                                       output_scales=bs)
    send = [xs[q].index_select(0, ii[q]).reshape(-1) for q in range(W)]
    rc, rs = O.all_to_all_codes_reference(send, c, fmt=fmt, bucket_size=B)
    for r in range(W):
        exp_c = base[r].view(torch.uint8).reshape(-1, H).clone()
        exp_c.index_copy_(0, oi[r], rc[r].view(torch.uint8).reshape(-1, H))
        assert torch.equal(got_c[r].view(torch.uint8), exp_c.reshape(-1))
        exp_s = bs[r].reshape(-1, H // B).clone().index_copy_(0, oi[r], rs[r].reshape(-1, H // B))
        assert_same(got_s[r], exp_s.reshape(-1))


# ---- the host generic reducer -------------------------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", "H")])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_reducer_matches_simulator(fmt, bucket, dtype):
    H, B = BUCKET_ROWS[bucket], _bucket(bucket)
    W = 3
    c = row_counts(W, "uneven", 2, H, seed=B)
    xs = inputs(c, dtype, B)
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    red.set_recording(True)
    outs, scales = codes_outputs(c, B, fmt)
    red.all_to_all(xs, outs, c, bits=fmt, bucket_size=B, output_scales=scales)
    codes_msgs = red.messages()
    sim_c, sim_s = simulate_codes(xs, c, fmt, B)
    for r in range(W):
        assert_codes(outs[r], sim_c[r], f"rank {r}")
        assert_same(scales[r], sim_s[r], f"rank {r}")
    # the wire is the decoded FP8 call's, byte for byte
    red.all_to_all(xs, [torch.empty(o.numel(), dtype=dtype) for o in outs], c, bits=fmt, bucket_size=B)
    dec_msgs = red.messages()
    assert len(codes_msgs) == len(dec_msgs)
    for (_, s1, d1, m1), (_, s2, d2, m2) in zip(codes_msgs, dec_msgs):
        assert (s1, d1) == (s2, d2) and torch.equal(m1, m2)


def test_generic_reducer_uint8_outputs_world1():
    x = torch.randn(4 * 256)
    outs = [torch.zeros(x.numel(), dtype=torch.uint8)]
    scales = [torch.zeros(x.numel() // 256)]
    _C.LocalReducerGroup(1, "SRA", 5000).all_to_all([x], outs, [[x.numel()]], bits="e5m2", bucket_size=256,
                                                      output_scales=scales)
    ref_c, ref_s = O.fp8_quantize(x, "e5m2", 256)
    assert torch.equal(outs[0], ref_c.view(torch.uint8))
    assert_same(scales[0], ref_s)


# ---- refusals -----------------------------------------------------------------------------------
def test_native_refusals():
    x = [torch.randn(512), torch.randn(512)]
    c = [[256, 256], [256, 256]]
    outs, scales = codes_outputs(c, 128, "e4m3")
    with pytest.raises(ValueError, match="e4m3"):  # integer bits
        _C.all_to_all_simulate(x, [o.view(torch.uint8) for o in outs], c, bits=8, bucket_size=128, output_scales=scales)
    with pytest.raises(ValueError, match="round"):
        _C.all_to_all_simulate(x, outs, c, bits="e4m3", bucket_size=128, stochastic=True, output_scales=scales)
    with pytest.raises(ValueError, match="8192"):
        _C.all_to_all_simulate(x, outs, c, bits="e4m3", bucket_size=16384, output_scales=scales)
    with pytest.raises(RuntimeError):  # a float8 of the other format
        _C.all_to_all_simulate(x, [o.view(torch.float8_e5m2) for o in outs], c, bits="e4m3", bucket_size=128,
                               output_scales=scales)
    with pytest.raises(RuntimeError):  # scales of the wrong size
        _C.all_to_all_simulate(x, outs, c, bits="e4m3", bucket_size=128, output_scales=[s[:1] for s in scales])
    with pytest.raises(RuntimeError):  # scales of the wrong dtype
        _C.all_to_all_simulate(x, outs, c, bits="e4m3", bucket_size=128, output_scales=[s.double() for s in scales])
    with pytest.raises(ValueError, match="whole buckets"):  # counts that are not whole buckets
        c2 = [[200, 312], [312, 200]]
        o2, s2 = codes_outputs(c2, 8, "e4m3")
        _C.all_to_all_simulate(x, o2, c2, bits="e4m3", bucket_size=128, output_scales=[t[:4] for t in s2])
    # the generic reducer checks the same, and refuses codes that overlap the input
    red = _C.LocalReducerGroup(1, "SRA", 5000)
    y = torch.randn(1024)
    with pytest.raises((ValueError, RuntimeError), match="overlap"):
        red.all_to_all([y], [y.view(torch.uint8)[:1024]], [[1024]], bits="e4m3", bucket_size=128,
                       output_scales=[torch.zeros(8)])
    with pytest.raises((ValueError, RuntimeError), match="overlap"):
        red.all_to_all([y], [torch.zeros(1024, dtype=torch.uint8)], [[1024]], bits="e4m3", bucket_size=128,
                       output_scales=[y[:8]])


def _public(out, x, scales, **kw):
    kw.setdefault("bits", "e4m3")
    kw.setdefault("bucket_size", 128)
    cgx.all_to_all_single(out, x, output_scales=scales, **kw)


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
        dict(bucket_size=100),                                          # H % bucket != 0
        dict(bucket_size=16384),                                        # bucket > 8192
    ]
    for kw in cases:
        with pytest.raises(ValueError):
            _public(codes, x, scales, **kw)
    with pytest.raises(ValueError, match="output_scales"):  # host scales (the CUDA cases are in the GPU tier)
        _public(codes, x, scales)
    with pytest.raises(ValueError, match="float8"):
        _public(torch.empty(4, 512, dtype=torch.uint8), x, scales)
