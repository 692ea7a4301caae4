"""Stochastic FP8 rounding ("e4m3_sr" / "e5m2_sr", DESIGN §2.13h) without a GPU: the host encoder
against the independent oracle (``oracle.fp8_sr_quantize``, frexp arithmetic on the words of
``_C.philox_u16``) bit for bit over Gaussian, heavy-tailed, subnormal-range, on-grid, near-FMAX, zero,
tiny, NaN and Inf buckets; the rule's consequences (grid neighbours, on-grid values, the base format's
bytes on special buckets, unbiasedness over seeds, survival of small values); determinism and stream
separation; every simulator against the oracle; and the names and refusals of every front end."""
from __future__ import annotations

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
from _engine_cases import TIMEOUT_MS, assert_results, inputs_for, mixed_table

FMTS = ("e4m3_sr", "e5m2_sr")
BASE = {"e4m3_sr": "e4m3", "e5m2_sr": "e5m2"}
CODEC = {"e4m3_sr": 5, "e5m2_sr": 6}
FMAX = {"e4m3_sr": 448.0, "e5m2_sr": 57344.0}
EMIN_MB = {"e4m3_sr": (-6, 3), "e5m2_sr": (-14, 2)}
TDT = {"e4m3_sr": torch.float8_e4m3fn, "e5m2_sr": torch.float8_e5m2}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
KINDS = ("gauss", "heavy", "subnormal", "ongrid", "nearmax", "zero", "tiny", "nan", "inf")


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)
    monkeypatch.delenv("CGX_STOCHASTIC_ROUNDING", raising=False)


def _bucket_values(kind: str, n: int, fmt: str, g: torch.Generator) -> torch.Tensor:
    x = torch.randn(n, generator=g)
    if kind == "heavy":
        return x * torch.exp(torch.randn(n, generator=g) * 4)
    if kind == "subnormal":
        # most of the bucket 2^-10 .. 2^-20 of its maximum: the format's subnormals and below
        x = x * 2.0 ** -torch.randint(8, 22, (n,), generator=g).float()
        x[0] = 1.0
        return x
    if kind == "ongrid":
        # values whose x * inv is exactly on the grid: codes times the unit of a bucket with max FMAX
        codes = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).view(TDT[fmt]).float()
        codes = torch.where(torch.isfinite(codes), codes, torch.zeros_like(codes))
        codes[0] = FMAX[fmt]
        return codes
    if kind == "nearmax":
        return torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0) * (1 - torch.rand(n, generator=g) * 1e-3)
    if kind == "zero":
        return torch.where(torch.rand(n, generator=g) < 0.5, torch.tensor(-0.0), torch.tensor(0.0))
    if kind == "tiny":
        return x * 1e-44
    if kind == "nan":
        x[n // 2] = float("nan")
        return x
    if kind == "inf":
        x[n // 3] = float("-inf")
        return x
    return x


def _host_roundtrip(x: torch.Tensor, fmt: str, B: int, seed: int, seq: int, rank: int = 0) -> torch.Tensor:
    """the host encoder and decoder (the all-gather simulator at world 1: stream 1, indices from 0)"""
    out = torch.empty_like(x)
    _C.all_gather_simulate([x], [out], [(0, x.numel(), 8, B)], seed=seed, seq=seq, bits=fmt)
    return out


def _host_codes(x: torch.Tensor, fmt: str, B: int, seed: int, seq: int):
    codes = torch.empty(x.numel(), dtype=TDT[fmt])
    scales = torch.empty(x.numel() // B)
    _C.all_gather_simulate([x], [codes], [(0, x.numel(), 8, B)], seed=seed, seq=seq, bits=fmt, output_scales=[scales])
    return codes, scales


def _words(x: torch.Tensor, B: int, seed: int, seq: int, stream: int = 1, first: int = 0) -> np.ndarray:
    return O._sr_words(seed, seq, stream, first, x.numel(), O.effective_bucket(B))


def _assert_codes(got, ref, what):
    gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
    assert torch.equal(gn, rn), what
    assert torch.equal(got.view(torch.uint8)[~gn], ref.view(torch.uint8)[~rn]), what


# ---- the random words ------------------------------------------------------------------------------
def test_philox_words_are_the_integer_paths_offsets():
    """philox_u16 gives the bits integer stochastic rounding draws: a 1-bit max-min bucket of 0s and
    1s rounds x = 1/2 up exactly when h >= 2^15."""
    n, seed, seq = 4096, 77, 5
    x = torch.full((n,), 0.5)
    x[0], x[1] = 0.0, 1.0  # min 0, max 1: unit 1, x = 0.5 -> level floor(0.5 + h / 2^16)
    out = torch.empty_like(x)
    _C.all_gather_simulate([x], [out], [(0, n, 1, n)], stochastic=True, seed=seed, seq=seq)
    h = _C.philox_u16(seed, seq, 1, 0, n).numpy()
    assert np.array_equal(out.numpy()[2:], (h[2:] >= 32768).astype(np.float32))


# ---- the host encoder against the oracle -------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bucket,n", [(8, 64), (64, 1000), (100, 1037), (512, 4096), (1024, 5000), (8192, 8192),
                                      (8192, 20000)])
def test_host_encoder_is_the_rule(bucket, n, kind, fmt):
    g = torch.Generator().manual_seed(n + bucket)
    x = torch.cat([_bucket_values(kind, min(bucket, n - o), fmt, g) for o in range(0, n, bucket)])
    seed, seq = 1234567 + n, 3
    got = _host_roundtrip(x, fmt, bucket, seed, seq)
    want = O.fp8_sr_quantize_dequantize(x, fmt, bucket, _words(x, bucket, seed, seq))
    assert_same(got, want, f"{kind} B={bucket} n={n}")
    if n % bucket == 0:
        codes, scales = _host_codes(x, fmt, bucket, seed, seq)
        rc, rs = O.fp8_sr_quantize(x, fmt, bucket, _words(x, bucket, seed, seq))
        _assert_codes(codes, rc, f"{kind} codes")
        assert_same(scales, rs, f"{kind} scales")


@pytest.mark.parametrize("fmt", FMTS)
def test_every_code_is_a_grid_neighbour_and_on_grid_values_are_exact(fmt):
    g = torch.Generator().manual_seed(1)
    B, n = 512, 512 * 64
    x = torch.randn(n, generator=g) * torch.exp(torch.randn(n, generator=g) * 3)
    codes, units = O.fp8_sr_quantize(x, fmt, B, _words(x, B, 9, 0))
    rn_codes, rn_units = O.fp8_quantize(x, BASE[fmt], B)
    assert torch.equal(units, rn_units)
    y = (x.view(-1, B) / 1).numpy().astype(np.float32) * O._fp8_units(x.view(-1, B).numpy(), BASE[fmt])[1]
    y = y.reshape(-1)
    c = codes.float().numpy()
    # the two neighbours of y on the grid: round down and round up of |y|
    lo = O._fp8_sr_round(y, BASE[fmt], np.zeros(n, np.int64))
    hi = O._fp8_sr_round(y, BASE[fmt], np.full(n, 65535, np.int64))
    assert np.all((c == lo) | (c == hi))
    on_grid = lo == y
    assert on_grid.sum() > 0 and np.array_equal(c[on_grid], rn_codes.float().numpy()[on_grid])
    # the "ongrid" buckets: every value on the grid, every code the round-to-nearest one
    xg = _bucket_values("ongrid", 4096, fmt, g)
    got = _host_roundtrip(xg, fmt, 4096, 5, 6)
    assert_same(got, O.fp8_quantize_dequantize(xg, BASE[fmt], 4096), "on grid")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["zero", "tiny", "nan", "inf"])
def test_special_buckets_are_the_base_formats_bytes(kind, fmt):
    g = torch.Generator().manual_seed(3)
    x = _bucket_values(kind, 1024, fmt, g)
    if kind in ("nan", "inf"):
        x = torch.full((1024,), 2.0)
        x[7] = float("nan") if kind == "nan" else float("inf")
    for seed in (0, 1, 99):
        codes, scales = _host_codes(x, fmt, 1024, seed, 0)
        rc, rs = O.fp8_quantize(x, BASE[fmt], 1024)
        _assert_codes(codes, rc, kind)
        assert_same(scales, rs, kind)


@pytest.mark.parametrize("fmt", FMTS)
def test_unbiased_over_seeds(fmt):
    """Over N = 4096 seeds the mean decoded value of every element is within unit * (5 * (s/2) / sqrt(N)
    + s * 2^-16) of y * unit, s the grid spacing at |y|; round to nearest is further off on the same
    inputs."""
    N, B = 4096, 64
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, generator=g) * torch.exp(torch.randn(B, generator=g))
    x[0] = 8.0  # the bucket max: unit = 8 / FMAX
    unit, inv = O._fp8_units(x.view(1, -1).numpy(), BASE[fmt])
    y = (x.numpy() * inv.reshape(-1)).astype(np.float32).astype(np.float64)
    emin, mb = EMIN_MB[fmt]
    s = np.ldexp(1.0, np.maximum(np.frexp(np.abs(y))[1] - 1, emin) - mb)
    xs = x.repeat(N)
    words = np.concatenate([O._sr_words(seed, 0, 1, 0, B, B) for seed in range(N)])
    dec = O.fp8_sr_quantize_dequantize(xs, fmt, B, words).double().view(N, B)
    mean = dec.mean(0).numpy()
    u = float(unit.reshape(-1)[0])
    target = y * u
    tol = u * (5 * (s / 2) / np.sqrt(N) + s * 2.0 ** -16)
    assert np.all(np.abs(mean - target) <= tol)
    rn = O.fp8_quantize_dequantize(x, BASE[fmt], B).double().numpy()
    assert np.abs(rn - target).max() > np.abs(mean - target).max()
    # the host encoder draws the same: a handful of seeds through the simulator
    for seed in range(4):
        got = _host_roundtrip(x, fmt, B, seed, 0)
        assert torch.equal(got.double(), dec[seed].float().double())


@pytest.mark.parametrize("fmt", FMTS)
def test_small_values_survive_in_expectation(fmt):
    """Elements below half the smallest subnormal (round to nearest: 0) keep their mean over seeds;
    below 2^-16 of the smallest subnormal they become 0."""
    emin, mb = EMIN_MB[fmt]
    smallest = 2.0 ** (emin - mb)
    B, N = 16, 2048
    x = torch.zeros(B)
    x[0] = FMAX[fmt]  # unit 1
    x[1:8] = torch.tensor([0.3, 0.1, 0.45, -0.2, 0.05, 0.49, -0.4]) * smallest
    x[8] = smallest * 2.0 ** -17
    xs = x.repeat(N)
    words = np.concatenate([O._sr_words(seed, 2, 1, 0, B, B) for seed in range(N)])
    dec = O.fp8_sr_quantize_dequantize(xs, fmt, B, words).double().view(N, B)
    assert torch.all(O.fp8_quantize_dequantize(x, BASE[fmt], B)[1:9] == 0)
    mean = dec.mean(0)
    tol = 5 * smallest / 2 / np.sqrt(N) + smallest * 2.0 ** -16
    assert torch.all((mean[1:8] - x[1:8].double()).abs() <= tol)
    assert torch.all(dec[:, 8] == 0)


def test_determinism_and_streams():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(4096, generator=g)
    a = _host_roundtrip(x, "e5m2_sr", 512, 7, 1)
    assert torch.equal(a, _host_roundtrip(x, "e5m2_sr", 512, 7, 1))
    assert not torch.equal(a, _host_roundtrip(x, "e5m2_sr", 512, 8, 1))
    assert not torch.equal(a, _host_roundtrip(x, "e5m2_sr", 512, 7, 2))
    # another rank: the all-gather's shard 1 is drawn from stream 3
    xs = [x, x.clone()]
    outs = [torch.empty(8192) for _ in range(2)]
    _C.all_gather_simulate(xs, outs, [(0, 4096, 8, 512)], seed=7, seq=1, bits="e5m2_sr")
    assert torch.equal(outs[0][:4096], a) and not torch.equal(outs[0][4096:], a)


# ---- the simulators --------------------------------------------------------------------------------
@pytest.mark.parametrize("stochastic", [False, True])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,bucket", [(2, 7), (3, 128), (8, 512), (3, 1024), (2, 8192)])
def test_all_to_all_simulator(world, bucket, fmt, dtype, stochastic):
    c = A.counts(world, "uneven", A.base_elems(bucket), 7 * world + bucket)
    xs = A.inputs(c, dtype, world)
    outs = A.outputs(c, dtype)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=bucket, stochastic=stochastic, seed=41, seq=6)
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=bucket, seed=41, seq=6)
    for r in range(world):
        assert_same(outs[r], ref[r], f"rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
def test_all_to_all_simulator_across_nodes(fmt):
    world = 24
    c = A.counts(world, "uneven", 70, seed=world)
    xs = A.inputs(c, torch.bfloat16, seed=3)
    outs = A.outputs(c, torch.bfloat16)
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=64, seed=5, seq=1)
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=64, seed=5, seq=1)
    for r in range(world):
        assert_same(outs[r], ref[r], f"rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,bucket", [(2, 128), (3, 1024), (8, 512)])
def test_codes_simulators(world, bucket, fmt):
    c = [[v * 1024 for v in row] for row in A.counts(world, "uneven", 2, world)]
    xs = A.inputs(c, torch.bfloat16, bucket)
    outs = []
    scales = []
    for r in range(world):
        n = sum(c[q][r] for q in range(world))
        outs.append(torch.empty(n, dtype=TDT[fmt]))
        scales.append(torch.empty(n // bucket))
    _C.all_to_all_simulate(xs, outs, c, bits=fmt, bucket_size=bucket, seed=3, seq=2, output_scales=scales)
    rc, rs = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=bucket, seed=3, seq=2)
    for r in range(world):
        _assert_codes(outs[r], rc[r], f"rank {r} codes")
        assert_same(scales[r], rs[r], f"rank {r} scales")
    S = 2048
    sh = [torch.randn(S) * (q + 1) for q in range(world)]
    codes = [torch.empty(world * S, dtype=TDT[fmt]) for _ in range(world)]
    sc = [torch.empty(world * S // bucket) for _ in range(world)]
    _C.all_gather_simulate(sh, codes, [(0, S, 8, bucket)], seed=3, seq=2, bits=fmt, output_scales=sc)
    rc, rs = O.all_gather_codes_reference(sh, fmt, bucket, seed=3, seq=2)
    for r in range(world):
        _assert_codes(codes[r], rc, f"ag rank {r}")
        assert_same(sc[r], rs, f"ag rank {r}")


@pytest.mark.parametrize("stochastic", [False, True])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", (2, 3, 8))
def test_all_gather_and_one_shot_simulators(world, fmt, dtype, stochastic):
    S = 3 * 1024 + 37
    table = [(0, 37, 32, 512), (37, 2000, 8, 100), (2037, S - 2037, 8, 1024)]
    g = torch.Generator().manual_seed(world)
    own = [(torch.randn(S, generator=g) * (r + 1)).to(dtype) for r in range(world)]
    outs = [torch.empty(world * S, dtype=dtype) for _ in range(world)]
    _C.all_gather_simulate(own, outs, table, stochastic=stochastic, seed=9, seq=4, bits=fmt)
    assert_results(outs, [O.all_gather_reference(own, table, fmt, seed=9, seq=4)] * world, "ag")
    xs = [x.clone() for x in own]
    _C.oneshot_simulate(xs, table, average=True, stochastic=stochastic, seed=9, seq=4, bits=fmt)
    assert_results(xs, O.oneshot_reference(own, table, average=True, fmt=fmt, seed=9, seq=4), "oneshot")


@pytest.mark.parametrize("fmt", FMTS)
def test_stochastic_flag_has_no_effect(fmt):
    world, n = 3, 9000
    g = torch.Generator().manual_seed(4)
    xs = [torch.randn(n, generator=g).bfloat16() for _ in range(world)]
    table = [(0, n, 8, 512)]
    a = [x.clone() for x in xs]
    b = [x.clone() for x in xs]
    _C.sra_simulate(a, table, average=True, seed=1, seq=2, bits=fmt)
    _C.sra_simulate(b, table, average=True, stochastic=True, seed=1, seq=2, bits=fmt)
    assert_results(a, b, "sra")
    rs_in = [torch.randn(world * 4096, generator=g) for _ in range(world)]
    o1 = [torch.empty(4096) for _ in range(world)]
    o2 = [torch.empty(4096) for _ in range(world)]
    _C.reduce_scatter_simulate(rs_in, o1, [(0, 4096, 8, 512)], seed=1, seq=2, bits=fmt)
    _C.reduce_scatter_simulate(rs_in, o2, [(0, 4096, 8, 512)], stochastic=True, seed=1, seq=2, bits=fmt)
    assert_results(o1, o2, "rs")
    # and it differs from round to nearest and from another seed
    c = [x.clone() for x in xs]
    _C.sra_simulate(c, table, average=True, seed=2, seq=2, bits=fmt)
    d = [x.clone() for x in xs]
    _C.sra_simulate(d, table, average=True, bits=BASE[fmt])
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[0], d[0])


@pytest.mark.parametrize("fmt", FMTS)
def test_sra_and_reduce_scatter_use_the_phase_streams(fmt):
    """SRA phase A draws rank q's bits from stream 2q and phase B the owner's from 2c + 1; the
    reduce-scatter is phase A's sum: at world 2 each owner adds one peer's SR contribution."""
    world, S = 2, 2048
    g = torch.Generator().manual_seed(8)
    xs = [torch.randn(world * S, generator=g) for _ in range(world)]
    outs = [torch.empty(S) for _ in range(world)]
    _C.reduce_scatter_simulate(xs, outs, [(0, S, 8, 512)], seed=6, seq=1, bits=fmt)
    for c in range(world):
        q = 1 - c
        peer = O.fp8_sr_quantize_dequantize(xs[q][c * S:(c + 1) * S], fmt, 512,
                                            O._sr_words(6, 1, 2 * q, c * S, S, 512))
        want = (xs[c][c * S:(c + 1) * S].numpy() + peer.numpy()).astype(np.float32)
        assert_same(outs[c], torch.from_numpy(want), f"owner {c}")


# ---- the engine and the front ends -------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_engine_format_from_environment(fmt, monkeypatch):
    """CGX_COMPRESSION_FORMAT=<fmt> through LocalEngineGroup: the SR codec, deterministic for a seed,
    and different from the base format's result"""
    layers, total = mixed_table([(9000, 8, 512), (700, 8, 100)])
    cfg = dict(p2p=False, fusion_bytes=8192)
    runs = {}
    for name in (fmt, BASE[fmt]):
        for k in range(2):
            eg = _C.LocalEngineGroup(2, 2, cfg, 1, 1 << 16, TIMEOUT_MS)
            state = inputs_for(2, total, torch.float16, 1)
            monkeypatch.setenv("CGX_COMPRESSION_FORMAT", name)
            eg.allreduce_layers(state, layers, False)
            runs[(name, k)] = state
    assert_results(runs[(fmt, 0)], runs[(fmt, 1)], "same seed")
    assert not torch.equal(runs[(fmt, 0)][0], runs[(BASE[fmt], 0)][0])
    assert torch.equal(runs[(fmt, 0)][0], runs[(fmt, 0)][1])  # every rank ends with the same bytes


@pytest.mark.parametrize("fmt", FMTS)
def test_names_accepted_everywhere(fmt):
    for op in ("all_to_all", "allreduce", "reduce_scatter", "all_gather"):
        assert tuple(_C.a2a_bits(fmt, False, op)) == (8, CODEC[fmt])
        assert tuple(_C.a2a_bits(fmt, True, op)) == (8, CODEC[fmt])
    with cgx.compression(bits=fmt):
        assert os.environ["CGX_COMPRESSION_FORMAT"] == fmt
        assert os.environ["CGX_COMPRESSION_QUANTIZATION_BITS"] == "8"
    with cgx.compression(bits=fmt, stochastic=True):
        assert os.environ["CGX_COMPRESSION_FORMAT"] == fmt
    st = cgx.CGXState(None, compression_params={"bits": fmt, "bucket_size": 256})
    assert (st.quantization_bits, st.quantization_format) == (8, fmt)
    assert H._width_and_format(fmt) == (8, fmt)
    assert FS.CGXReduceScatter(fmt).bits == fmt
    assert FS.CGXReduceScatter(fmt, stochastic=True).bits == fmt


@pytest.mark.parametrize("fmt", FMTS)
def test_refusals(fmt, monkeypatch):
    # the FSDP2 all-gather rounds to nearest
    with pytest.raises(ValueError, match="all-gather"):
        FS.CGXAllGather(fmt)
    with pytest.raises(ValueError, match="all-gather"):
        FS.set_cgx_all_gather(torch.nn.Linear(4, 4), bits=fmt)
    # adaptive widths
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveCGXState(None, compression_params={"bits": fmt})
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveFSDPState(reduce_scatter_bits=fmt)
    with pytest.raises(ValueError, match="adaptive"):
        FS.CGXReduceScatter(fmt, adaptive=object())
    # the base names keep refusing stochastic rounding
    with pytest.raises(ValueError, match="round"):
        _C.a2a_bits(BASE[fmt], True, "all_to_all")
    # codes of the other base format
    other = torch.float8_e5m2 if fmt == "e4m3_sr" else torch.float8_e4m3fn
    x = torch.randn(4, 512)
    with pytest.raises(ValueError, match="float8"):
        cgx.all_to_all_single(torch.empty(4, 512, dtype=other), x, bits=fmt, bucket_size=128,
                              output_scales=torch.empty(4, 4))
    with pytest.raises(ValueError, match="float8"):
        cgx.all_gather_into_tensor(torch.empty(2048, dtype=other), x.reshape(-1), bits=fmt, bucket_size=128,
                                   output_scales=torch.empty(16))
    # integer-width layers in a table, in the reducers and the engine
    xs = [torch.randn(512) for _ in range(2)]
    for kind in ("SRA", "RING"):
        g = _C.LocalReducerGroup(2, kind, 5000)
        with pytest.raises(ValueError, match="bits 8 or 32"):
            g.allreduce(xs, [(0, 256, 8, 32), (256, 256, 4, 32)], bits=fmt)
        assert g.bytes_sent() == [0, 0]
    eg = _C.LocalEngineGroup(2, 2, dict(p2p=False, inner_reduction="ALLTOALL"), 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises((ValueError, RuntimeError)):
        eg.allreduce_layers(xs, [(0, 512, 8, 32)], False, bits=fmt)
    assert all(eg.stats(r)["calls"] == 0 for r in range(2))
    # oracles without a random stream refuse the SR formats instead of rounding to nearest
    with pytest.raises(ValueError, match="stochastically"):
        O.sra_reference(xs, [(0, 512, 8, 32)], fmt=fmt)
    with pytest.raises(ValueError):
        O.fp8_quantize(xs[0], fmt, 32)
