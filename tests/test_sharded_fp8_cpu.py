"""FP8 wire formats of the compressed reduce-scatter and all-gather without a GPU: the CPU simulators
against the independent reference (numpy fp32 sums over ``oracle.fp8_quantize_dequantize``) for both
formats, every dtype, several bucket sizes and worlds; multi-layer tables with raw entries, averaging
and the edge inputs; the generic reducers on host memory; the two-stage composition of the engine
against the single-stage reference where it must equal it; and the argument checks, which raise
before anything is sent."""
from __future__ import annotations

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import fsdp as FS

from _bitwise import assert_same
from _edge_inputs import edge_inputs
from _engine_cases import TIMEOUT_MS, assert_results, clean_environment  # noqa: F401

FMTS = ("e4m3", "e5m2")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
# raw entries between FP8 ones, buckets that do not divide the layers
MIXED = [(0, 37, 32, 512), (37, 3000, 8, 100), (3037, 301, 32, 512), (3338, 1501, 8, 7), (4839, 700, 8, 1024)]
S_MIXED = 5539


def _full(world, S, dtype, seed, scale_by_rank=True):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(world * S, generator=g) * ((r + 1) if scale_by_rank else 1)).to(dtype)
            for r in range(world)]


def _own(full):
    W = len(full)
    S = full[0].numel() // W
    return [full[r][r * S:(r + 1) * S].clone() for r in range(W)]


def _rs_sim(full, table, fmt, **kw):
    W = len(full)
    outs = [torch.empty(full[0].numel() // W, dtype=full[0].dtype) for _ in range(W)]
    _C.reduce_scatter_simulate(full, outs, table, bits=fmt, **kw)
    return outs


def _ag_sim(shards, table, fmt):
    W = len(shards)
    outs = [torch.empty(W * shards[0].numel(), dtype=shards[0].dtype) for _ in range(W)]
    _C.all_gather_simulate(shards, outs, table, bits=fmt)
    return outs


def _check_rs(full, table, fmt, what, **kw):
    got = _rs_sim(full, table, fmt, **kw)
    want = O.reduce_scatter_reference(full, table, fmt=fmt, **kw)
    assert_results(got, want, what)


def _check_ag(shards, table, fmt, what):
    got = _ag_sim(shards, table, fmt)
    want = O.all_gather_reference(shards, table, fmt)
    assert_results(got, [want] * len(shards), what)


# ---- simulators against the reference ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("bucket", [8, 512, 1024, 300])
def test_simulators_equal_reference(bucket, world, fmt, dtype):
    S = 2600
    table = [(0, S, 8, bucket)]
    full = _full(world, S, dtype, 11 * world + bucket)
    _check_rs(full, table, fmt, f"rs {fmt} W={world} B={bucket}")
    _check_rs(full, table, fmt, f"rs {fmt} W={world} B={bucket} avg", average=True)
    _check_ag(_own(full), table, fmt, f"ag {fmt} W={world} B={bucket}")


def test_world1_all_gather_is_the_round_trip():
    x = torch.randn(3000, dtype=torch.bfloat16)
    for fmt in FMTS:
        got = _ag_sim([x], [(0, 3000, 8, 512)], fmt)[0]
        assert_same(got, O.fp8_quantize_dequantize(x, fmt, 512), fmt)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [2, 5])
def test_mixed_tables_with_raw_entries(world, fmt, dtype):
    full = _full(world, S_MIXED, dtype, world)
    _check_rs(full, MIXED, fmt, "rs mixed")
    _check_rs(full, MIXED, fmt, "rs mixed avg", average=True)
    _check_rs(full, MIXED, fmt, "rs mixed prescale", prescale=0.3)
    _check_ag(_own(full), MIXED, fmt, "ag mixed")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("where", ["owner", "peer"])
def test_edge_inputs(where, fmt, dtype):
    world, bucket, S = 3, 64, 64 * 60
    table = [(0, S, 8, bucket)]
    # planted buckets of shard 1 (its owner is rank 1; "peer" plants them on rank 2)
    xs, _ = edge_inputs(dtype, S, bucket, 7, world=world, bits=8, owners=[1] * S, where=where)
    full = [torch.cat([torch.randn(S).to(dtype) if c != 1 else xs[r] for c in range(world)]) for r in range(world)]
    _check_rs(full, table, fmt, f"rs edge {where}")
    _check_ag([x.clone() for x in xs], table, fmt, f"ag edge {where}")


def test_peer_nonfinite_makes_the_bucket_nan_and_own_ones_propagate_per_element():
    S, B = 64, 32
    full = [torch.ones(2 * S), torch.ones(2 * S)]
    full[1][3] = float("inf")     # rank 1's value in shard 0, bucket 0: a peer's bucket for rank 0
    full[0][S + 40] = float("nan")  # rank 0's value in shard 1, bucket 1: a peer's bucket for rank 1
    full[0][5] = float("inf")     # rank 0's own value in its shard
    out = _rs_sim(full, [(0, S, 8, B)], "e4m3")
    assert torch.isnan(out[0][:B]).all() and torch.isfinite(out[0][B:]).all()
    assert torch.isnan(out[1][B:]).all() and torch.isfinite(out[1][:B]).all()
    full[1][3] = 1.0
    out = _rs_sim(full, [(0, S, 8, B)], "e4m3")
    assert torch.isinf(out[0][5]) and torch.isfinite(out[0][torch.arange(S) != 5]).all()


def test_error_is_relative_per_element():
    # one outlier in the bucket: max-min's step swamps the small values, FP8 keeps them
    x = torch.linspace(1.0, 2.0, 512)
    x[0] = 1e3
    shards = [x, torch.zeros(512)]
    for fmt, bound in (("e4m3", 2 ** -4), ("e5m2", 2 ** -3)):
        got = _ag_sim(shards, [(0, 512, 8, 512)], fmt)[0][:512]
        assert ((got - x).abs() <= bound * x.abs()).all()
    mm = _ag_sim(shards, [(0, 512, 8, 512)], None)[0][:512]
    assert ((mm[1:] - x[1:]).abs() > 0.25 * x[1:]).any()


# ---- the generic reducers on host memory ------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", [1, 2, 4])
def test_host_generic_reducer(world, fmt, dtype):
    full = _full(world, S_MIXED, dtype, 3 + world)
    g = _C.LocalReducerGroup(world, "SRA", 5000)
    outs = [torch.empty(S_MIXED, dtype=dtype) for _ in range(world)]
    g.reduce_scatter(full, outs, MIXED, average=True, bits=fmt)
    assert_results(outs, _rs_sim(full, MIXED, fmt, average=True), "generic rs")
    outs = [torch.empty(world * S_MIXED, dtype=dtype) for _ in range(world)]
    g.all_gather(_own(full), outs, MIXED, bits=fmt)
    assert_results(outs, _ag_sim(_own(full), MIXED, fmt), "generic ag")


# ---- two stages (several nodes) ---------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,local", [(4, 1), (6, 1), (4, 2), (6, 3), (8, 4), (8, 2), (4, 4)])
def test_two_stage_engine(world, local, fmt):
    dtype = torch.bfloat16
    g = _C.LocalEngineGroup(world, local, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    full = _full(world, S_MIXED, dtype, world + local)
    # the all-gather decodes every shard from one FP8 round trip, whatever the topology
    outs = [torch.empty(world * S_MIXED, dtype=dtype) for _ in range(world)]
    g.all_gather(_own(full), outs, MIXED, bits=fmt)
    assert_results(outs, [O.all_gather_reference(_own(full), MIXED, fmt)] * world, "two-stage ag")
    outs = [torch.empty(S_MIXED, dtype=dtype) for _ in range(world)]
    g.reduce_scatter(full, outs, True, MIXED, bits=fmt)
    if local == 1 or local == world:  # one rank per node, or one node: a single stage
        assert_results(outs, O.reduce_scatter_reference(full, MIXED, average=True, fmt=fmt), "two-stage rs")
    else:
        # a remote value is quantized at most twice: close to the single stage, not equal to it
        want = O.reduce_scatter_reference(full, MIXED, average=True, fmt=fmt)
        for r in range(world):
            err = (outs[r].float() - want[r].float()).norm() / want[r].float().norm()
            assert torch.isfinite(outs[r].float()).all() and err < 0.15, f"rank {r}: relative L2 error {err}"


# ---- argument checks ---------------------------------------------------------------------------------
def test_value_errors_before_anything_runs():
    full, outs = _full(2, 64, torch.float32, 0), [torch.empty(64), torch.empty(64)]
    shards, gathered = _own(full), [torch.empty(128), torch.empty(128)]
    bad_table = [(0, 32, 8, 32), (32, 32, 4, 32)]
    with pytest.raises(ValueError, match="bits 8 or 32"):
        _C.reduce_scatter_simulate(full, outs, bad_table, bits="e4m3")
    with pytest.raises(ValueError, match="bits 8 or 32"):
        _C.all_gather_simulate(shards, gathered, bad_table, bits="e5m2")
    with pytest.raises(ValueError, match="round"):
        _C.reduce_scatter_simulate(full, outs, [(0, 64, 8, 32)], stochastic=True, bits="e5m2")
    for bad in ("E4M3", "fp8", ""):
        with pytest.raises(ValueError, match="e4m3"):
            _C.all_gather_simulate(shards, gathered, [(0, 64, 8, 32)], bits=bad)
    g = _C.LocalReducerGroup(2, "SRA", 5000)
    with pytest.raises(ValueError, match="reduce_scatter"):
        g.reduce_scatter(full, outs, bad_table, bits="e4m3")
    with pytest.raises(ValueError, match="round"):
        g.all_gather(shards, gathered, [(0, 64, 8, 32)], stochastic=True, bits="e4m3")
    with pytest.raises(ValueError):
        O.reduce_scatter_reference(full, bad_table, fmt="e4m3")
    with pytest.raises(ValueError):
        O.all_gather_reference(shards, [(0, 64, 8, 32)], fmt="e3m4")
    # the parser names the op and keeps the words of the all-to-all's messages
    with pytest.raises(ValueError, match="cgx all_gather: .*e4m3"):
        _C.a2a_bits("int8", False, "all_gather")


def test_public_api_rejects_before_sending():
    # no process group exists: each call must fail on its arguments before looking for one
    out, inp = torch.empty(64), torch.empty(128)
    with pytest.raises(ValueError, match="bits 8 or 32"):
        cgx.reduce_scatter_tensor(out, inp, bits="e5m2", layers=[(0, 64, 4, 64)])
    with pytest.raises(ValueError, match="round"):
        cgx.reduce_scatter_tensor(out, inp, bits="e5m2", stochastic=True)
    with pytest.raises(ValueError, match="e4m3"):
        cgx.all_gather_into_tensor(inp, out, bits="fp8")
    with pytest.raises(ValueError, match="bits 8 or 32"):
        cgx.all_gather_into_tensor(inp, out, bits="e4m3", layers=[(0, 64, 2, 64)])


def test_fsdp_comms_and_adaptive_state():
    params = [((16, 8), 128), ((16,), 16), ((4, 4, 3), 48)]
    assert FS.fsdp_shard_table(params, "e4m3", 64) == [(0, 128, 8, 64), (128, 16, 32, 64), (144, 48, 8, 64)]
    assert FS.fsdp_shard_table(params, 4, 64) == [(0, 128, 4, 64), (128, 16, 32, 64), (144, 48, 4, 64)]
    assert FS.CGXReduceScatter("e5m2").bits == "e5m2" and FS.CGXAllGather(8).bits == 8
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveFSDPState(reduce_scatter_bits="e5m2")
    with pytest.raises(ValueError, match="adaptive"):
        cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits="e4m3")
    with pytest.raises(ValueError, match="adaptive"):
        FS.CGXAllGather("e4m3", adaptive=object())
