"""FP8 wire formats of the compressed allreduce without a GPU: the SRA and one-shot simulators against
the independent reference (numpy fp32 sums over ``oracle.fp8_quantize_dequantize``) for both formats,
every dtype, several bucket sizes and worlds; mixed tables with raw layers, averaging, explicit
prescales and the edge inputs; the host generic SRA and Ring reducers and the compressed broadcast;
the engine's stages (intra-node, cross-node, the leaders' compressed broadcast) against
``oracle.engine_reference``; the argument checks, which raise before anything is sent; and the DDP
hook state."""
from __future__ import annotations

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import hooks as H

from _edge_inputs import edge_inputs
from _engine_cases import (C, TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, mixed_table)

FMTS = ("e4m3", "e5m2")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
# raw entries between FP8 ones, buckets that do not divide the layers
MIXED = [(0, 37, 32, 512), (37, 3000, 8, 100), (3037, 301, 32, 512), (3338, 1501, 8, 7), (4839, 700, 8, 1024)]
N_MIXED = 5539


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)


def _inputs(world, n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def _sra_sim(xs, layers, fmt, **kw):
    out = [x.clone() for x in xs]
    C.sra_simulate(out, layers, bits=fmt, **kw)
    return out


def _oneshot_sim(xs, layers, fmt, **kw):
    out = [x.clone() for x in xs]
    C.oneshot_simulate(out, layers, bits=fmt, **kw)
    return out


def _check(xs, layers, fmt, what, **kw):
    assert_results(_sra_sim(xs, layers, fmt, **kw), O.sra_reference(xs, layers, fmt=fmt, **kw), f"sra {what}")
    assert_results(_oneshot_sim(xs, layers, fmt, **kw), O.oneshot_reference(xs, layers, fmt=fmt, **kw),
                   f"oneshot {what}")


# ---- simulators against the reference ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("bucket", [8, 512, 1024, 300])
def test_simulators_equal_reference(bucket, world, fmt, dtype):
    n = 9000
    table = [(0, n, 8, bucket)]
    xs = _inputs(world, n, dtype, 13 * world + bucket)
    _check(xs, table, fmt, f"{fmt} W={world} B={bucket}")
    _check(xs, table, fmt, f"{fmt} W={world} B={bucket} avg", average=True)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [2, 5])
def test_mixed_tables_with_raw_layers(world, fmt, dtype):
    xs = _inputs(world, N_MIXED + 50, dtype, world)  # 50 elements outside every layer are kept
    _check(xs, MIXED, fmt, "mixed")
    _check(xs, MIXED, fmt, "mixed avg", average=True)
    _check(xs, MIXED, fmt, "mixed prescale", prescale=0.3)
    kw = dict(lanes=4, min_lane_elems=512)  # more chunks than ranks' worth of lanes: the SRA's owners move
    assert_results(_sra_sim(xs, MIXED, fmt, **kw), O.sra_reference(xs, MIXED, fmt=fmt, **kw), "sra mixed lanes")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("where", ["owner", "peer"])
def test_edge_inputs(where, fmt, dtype):
    world, bucket, n = 3, 64, 64 * 90
    table = [(0, n, 8, bucket)]
    owners = O.block_owners(table, n, world, 1, dtype, False, 2048)
    xs, planted = edge_inputs(dtype, n, bucket, 5, world=world, bits=8, owners=owners, where=where)
    assert planted
    _check(xs, table, fmt, f"edge {where}")


def test_nonfinite_bucket_decodes_to_nan_everywhere():
    n, B = 256, 64
    for fmt in FMTS:
        xs = [torch.ones(n), torch.ones(n)]
        xs[1][3] = float("inf")    # a peer's value for rank 0's chunk, bucket 0
        xs[0][70] = float("nan")   # the owner's own value, bucket 1
        for out in (_sra_sim(xs, [(0, n, 8, B)], fmt), _oneshot_sim(xs, [(0, n, 8, B)], fmt)):
            for o in out:
                assert torch.isnan(o[:2 * B]).all() and torch.isfinite(o[2 * B:]).all()
            assert torch.equal(out[0].view(torch.int32), out[1].view(torch.int32))


def test_zero_buckets_keep_signed_zeros():
    # an FP8 code keeps the sign of a zero: the SRA's owner sums -0 + -0 = -0 and encodes it; the
    # one-shot sum starts from +0, so +0 + -0 = +0
    n = 64
    for fmt in FMTS:
        xs = [torch.full((n,), -0.0), torch.full((n,), -0.0)]
        sra, one = _sra_sim(xs, [(0, n, 8, 64)], fmt), _oneshot_sim(xs, [(0, n, 8, 64)], fmt)
        assert all(torch.equal(o.view(torch.int32), xs[0].view(torch.int32)) for o in sra)
        assert all(torch.equal(o.view(torch.int32), torch.zeros(n).view(torch.int32)) for o in one)
        _check(xs, [(0, n, 8, 64)], fmt, f"signed zeros {fmt}")


def test_error_is_relative_per_element():
    # one outlier in the bucket: max-min's step swamps the small values, FP8 keeps them
    x = torch.linspace(1.0, 2.0, 512)
    x[0] = 1e3
    xs = [x, torch.zeros(512)]
    for fmt, bound in (("e4m3", 2 ** -4), ("e5m2", 2 ** -3)):
        got = _sra_sim(xs, [(0, 512, 8, 512)], fmt)[0]
        assert ((got - x).abs() <= 2 * bound * x.abs()).all()
    mm = _sra_sim(xs, [(0, 512, 8, 512)], None)[0]
    assert ((mm[1:] - x[1:]).abs() > 0.25 * x[1:]).any()


# ---- the generic reducers on host memory ------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_host_generic_reducers(world, fmt, dtype):
    xs = _inputs(world, N_MIXED, dtype, 3 + world)
    kw = dict(average=True)
    for kind, ref in (("SRA", O.sra_reference), ("RING", O.ring_reference)):
        out = [x.clone() for x in xs]
        C.LocalReducerGroup(world, kind, 5000).allreduce(out, MIXED, bits=fmt, **kw)
        if kind == "SRA":
            want = ref(xs, MIXED, lanes=1, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS, fmt=fmt, **kw)
        else:
            want = ref(xs, MIXED, fmt=fmt, **kw)
        assert_results(out, want, f"generic {kind}")
    for root in {0, world - 1}:
        out = [x.clone() for x in xs]
        C.LocalReducerGroup(world, "SRA", 5000).broadcast_compressed(out, MIXED, root, bits=fmt)
        assert_results(out, O.broadcast_compressed_reference(xs, MIXED, root=root, fmt=fmt), f"bcast root {root}")


def test_generic_sra_equals_the_simulator_of_its_plan():
    # lanes = 1, rank chunks: the generic SRA is the fused kernel's arithmetic
    xs = _inputs(4, N_MIXED, torch.bfloat16, 9)
    for fmt in FMTS:
        out = [x.clone() for x in xs]
        C.LocalReducerGroup(4, "SRA", 5000).allreduce(out, MIXED, bits=fmt, prescale=0.7)
        assert_results(out, _sra_sim(xs, MIXED, fmt, prescale=0.7, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS),
                       f"generic sra {fmt}")


# ---- the engine: intra-node, cross-node and the compressed broadcast --------------------------------
TABLE8 = [(37, 32, 512), (9000, 8, 512), (301, 32, 512), (2001, 8, 64), (700, 8, 100), (1200, 8, 8), (513, 8, 1)]
ENGINE = [
    dict(world=2, local=2, inner="SRA", cross="RING", bcast=True, icomp=True),
    dict(world=3, local=3, inner="RING", cross="RING", bcast=True, icomp=True),
    dict(world=4, local=2, inner="SRA", cross="RING", bcast=True, icomp=True),
    dict(world=6, local=3, inner="RING", cross="SRA", bcast=True, icomp=True),
    dict(world=4, local=1, inner="SRA", cross="SRA", bcast=True, icomp=True),
    dict(world=6, local=2, inner="SRA", cross="RING", bcast=False, icomp=False),
    dict(world=8, local=4, inner="SRA", cross="SRA", bcast=True, icomp=False),
]


def engine_id(h):
    return (f"w{h['world']}l{h['local']}-{h['inner']}-{h['cross']}-{'bcast' if h['bcast'] else 'nobcast'}-"
            f"{'icomp' if h['icomp'] else 'iraw'}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("h", ENGINE, ids=engine_id)
def test_engine_stages(h, fmt):
    cfg = dict(inner_reduction=h["inner"], cross_reduction=h["cross"], intra_broadcast=h["bcast"],
               intra_compress=h["icomp"], p2p=False, fusion_bytes=8192)
    layers, total = mixed_table(TABLE8)
    world, local = h["world"], h["local"]
    dtype = DTYPES[world % 3]
    g = C.LocalEngineGroup(world, local, cfg, 1, 1 << 16, TIMEOUT_MS)
    state = inputs_for(world, total, dtype, world * 7 + local)
    for k in (1, 2):
        want, stages = O.engine_reference(state, layers, local_size=local, config=cfg, lanes=1, average=k == 2,
                                          call_seq=k, cuda=False, fmt=fmt)
        g.allreduce_layers(state, layers, k == 2, bits=fmt)
        assert_results(state, want, f"call {k}")
        assert_log(g, stages, world)


def test_engine_reads_the_format_from_the_environment(monkeypatch):
    layers, total = mixed_table(TABLE8)
    cfg = dict(p2p=False, fusion_bytes=8192)
    g = C.LocalEngineGroup(3, 3, cfg, 1, 1 << 16, TIMEOUT_MS)
    state = inputs_for(3, total, torch.float16, 1)
    want, _ = O.engine_reference(state, layers, local_size=3, config=cfg, lanes=1, cuda=False, fmt="e5m2")
    monkeypatch.setenv("CGX_COMPRESSION_FORMAT", "e5m2")
    g.allreduce_layers(state, layers, False)
    assert_results(state, want, "CGX_COMPRESSION_FORMAT=e5m2")
    # "maxmin" (or unset) is the max-min path
    monkeypatch.setenv("CGX_COMPRESSION_FORMAT", "maxmin")
    want, _ = O.engine_reference(state, layers, local_size=3, config=cfg, lanes=1, call_seq=2, cuda=False)
    g.allreduce_layers(state, layers, False)
    assert_results(state, want, "CGX_COMPRESSION_FORMAT=maxmin")


# ---- argument checks ---------------------------------------------------------------------------------
def test_value_errors_before_anything_runs():
    xs = _inputs(2, 64, torch.float32, 0)
    before = [x.clone() for x in xs]
    bad_table = [(0, 32, 8, 32), (32, 32, 4, 32)]
    with pytest.raises(ValueError, match="bits 8 or 32"):
        C.sra_simulate(xs, bad_table, bits="e4m3")
    with pytest.raises(ValueError, match="bits 8 or 32"):
        C.oneshot_simulate(xs, bad_table, bits="e5m2")
    with pytest.raises(ValueError, match="round"):
        C.sra_simulate(xs, [(0, 64, 8, 32)], stochastic=True, bits="e5m2")
    for bad in ("E4M3", "fp8", ""):
        with pytest.raises(ValueError, match="cgx allreduce: .*e4m3"):
            C.oneshot_simulate(xs, [(0, 64, 8, 32)], bits=bad)
    for kind in ("SRA", "RING"):
        g = C.LocalReducerGroup(2, kind, 5000)
        with pytest.raises(ValueError, match="bits 8 or 32"):
            g.allreduce(xs, bad_table, bits="e4m3")
        with pytest.raises(ValueError, match="round"):
            g.allreduce(xs, [(0, 64, 8, 32)], stochastic=True, bits="e4m3")
        with pytest.raises(ValueError, match="bits 8 or 32"):
            g.broadcast_compressed(xs, bad_table, 0, bits="e5m2")
        assert g.bytes_sent() == [0, 0]
    g = C.LocalReducerGroup(2, "ALLTOALL", 5000)
    with pytest.raises(ValueError, match="all-to-all reduction"):
        g.allreduce(xs, [(0, 64, 8, 32)], bits="e4m3")
    assert g.bytes_sent() == [0, 0]
    for o, b in zip(xs, before):
        assert torch.equal(o, b)
    with pytest.raises(ValueError):
        O.sra_reference(xs, bad_table, fmt="e4m3")
    with pytest.raises(ValueError):
        O.oneshot_reference(xs, [(0, 64, 8, 32)], fmt="e3m4")


@pytest.mark.parametrize("case", ["width", "stochastic", "alltoall", "name"])
def test_engine_rejects_before_sending(case, monkeypatch):
    layers = [(0, 64, 8, 32), (64, 64, 4 if case == "width" else 8, 32)]
    cfg = dict(p2p=False, inner_reduction="ALLTOALL" if case == "alltoall" else "SRA")
    g = C.LocalEngineGroup(2, 2, cfg, 1, 1 << 16, TIMEOUT_MS)
    xs = _inputs(2, 128, torch.float32, 1)
    before = [x.clone() for x in xs]
    if case == "stochastic":
        monkeypatch.setenv("CGX_STOCHASTIC_ROUNDING", "1")
    want = {"width": "bits 8 or 32", "stochastic": "round", "alltoall": "all-to-all reduction",
            "name": "CGX_COMPRESSION_FORMAT"}[case]
    if case == "name":
        monkeypatch.setenv("CGX_COMPRESSION_FORMAT", "fp8")
        with pytest.raises((ValueError, RuntimeError), match=want):
            g.allreduce_layers(xs, layers, False)
    else:
        with pytest.raises((ValueError, RuntimeError), match=want):
            g.allreduce_layers(xs, layers, False, bits="e4m3")
    assert all(g.stats(r)["calls"] == 0 and g.stats(r)["wire_bytes"] == 0 for r in range(2))
    for o, b in zip(xs, before):
        assert torch.equal(o, b)


def test_public_api_rejects_before_sending():
    # no process group exists: each call must fail on its arguments before looking for one
    t = torch.ones(64)
    with pytest.raises(ValueError, match="e4m3"):
        cgx.all_reduce(t, bits="fp8")
    with pytest.raises(ValueError, match="round"):
        cgx.all_reduce(t, bits="e5m2", stochastic=True)
    with pytest.raises(ValueError, match="e4m3"):
        with cgx.compression(bits="int8"):
            pass


def test_compression_sets_and_restores_the_format(monkeypatch):
    import os

    monkeypatch.delenv("CGX_COMPRESSION_QUANTIZATION_BITS", raising=False)
    with cgx.compression(bits="e5m2"):
        assert os.environ["CGX_COMPRESSION_FORMAT"] == "e5m2"
        assert os.environ["CGX_COMPRESSION_QUANTIZATION_BITS"] == "8"
        with cgx.compression(bits=4):  # an integer width inside selects max-min again
            assert os.environ["CGX_COMPRESSION_FORMAT"] == "maxmin"
        assert os.environ["CGX_COMPRESSION_FORMAT"] == "e5m2"
        with cgx.compression(bucket_size=64):  # no width given: the format stays
            assert os.environ["CGX_COMPRESSION_FORMAT"] == "e5m2"
    assert "CGX_COMPRESSION_FORMAT" not in os.environ and "CGX_COMPRESSION_QUANTIZATION_BITS" not in os.environ


# ---- the DDP hook state ------------------------------------------------------------------------------
def test_cgx_state_format_and_state_dict_round_trip():
    st = cgx.CGXState(None, compression_params={"bits": "e5m2", "bucket_size": 256})
    assert (st.quantization_bits, st.quantization_format, st.quantization_bucket_size) == (8, "e5m2", 256)
    sd = st.state_dict()
    assert sd["quantization_bits"] == "e5m2"
    other = cgx.CGXState(None, compression_params={"bits": 4})
    assert other.quantization_format is None
    other.load_state_dict(sd)
    assert (other.quantization_bits, other.quantization_format) == (8, "e5m2")
    st.load_state_dict(dict(sd, quantization_bits=2))
    assert (st.quantization_bits, st.quantization_format) == (2, None)
    assert st.state_dict()["quantization_bits"] == 2
    with pytest.raises(ValueError, match="e4m3"):
        cgx.CGXState(None, compression_params={"bits": "e3m4"})
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveCGXState(None, compression_params={"bits": "e4m3"})
    assert H._width_and_format("e4m3") == (8, "e4m3") and H._width_and_format(6) == (6, None)
