"""The compressed reduce-scatter and all-gather over several nodes, on host memory.

The hierarchical references of torch_cgx_b200/ops/oracle.py reduce to the flat ones where they
must; the generic reducers' Reducer::reduce_scatter / ::all_gather (C.LocalReducerGroup, W 1-16,
all dtypes, bits 1-8 and raw, bucket sizes 1 to 10000, averaging, skip_incomplete, mixed tables,
hostile inputs, stochastic rounding) equal the references and the CPU simulators bit for bit and
send the bytes of the plan; the engine's two-stage composition (C.LocalEngineGroup without heaps)
equals ``oracle.sharded_engine_reference`` in values and stage logs at every (W, L) of
``TOPOLOGIES``, with and without intra-node compression; and each wrong semantics of
``SHARDED_PERTURBATIONS`` fails a named case. All parameters are fixed lists."""
import pytest
import torch

from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same, mismatch
from _engine_cases import (C, TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, set_stochastic)
from _reducer_cases import config_id, configs
from _sharded_cases import (TOPOLOGIES, gather_with_skip, own_shards, sharded_bytes_sent, sharded_inputs,
                            shard_table)

DTYPES = [torch.float32, torch.float16, torch.bfloat16]
CONFIGS = configs()
MIXED = [(0, 37, 32, 512), (37, 3000, 4, 100), (3037, 301, 32, 512), (3338, 1501, 3, 7), (4839, 700, 8, 1024)]
S_MIXED = 5539


# ---- the references ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("world", [1, 2, 4, 6])
def test_hier_reduce_scatter_with_one_rank_per_node_is_flat(world, dtype):
    full = inputs_for(world, world * S_MIXED, dtype, world)
    for average in (False, True):
        want = O.reduce_scatter_reference(full, MIXED, average=average)
        for local in ({1, world}):  # one rank per node, and one node
            got = O.reduce_scatter_hier_reference(full, MIXED, local_size=local, average=average)
            assert_results(got, want, f"L={local} avg={average}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("world,local", TOPOLOGIES + [(2, 2), (3, 1), (8, 8)])
def test_hier_all_gather_is_flat(world, local, dtype):
    shards = inputs_for(world, S_MIXED, dtype, world + local)
    want = O.all_gather_reference(shards, MIXED)
    got = O.all_gather_hier_reference(shards, MIXED, local_size=local)
    assert_results(got, [want] * world, f"W={world} L={local}")


def test_hier_reduce_scatter_differs_from_flat_across_nodes_of_several_ranks():
    # a remote contribution is quantized once more on its way: the two-stage result is not the flat one
    full = inputs_for(4, 4 * S_MIXED, torch.float32, 3)
    flat = O.reduce_scatter_reference(full, MIXED)
    hier = O.reduce_scatter_hier_reference(full, MIXED, local_size=2)
    assert any(mismatch(a, b) for a, b in zip(hier, flat))


# ---- the generic reducers ----------------------------------------------------------------------------
@pytest.mark.parametrize("c", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_host_reduce_scatter(c):
    W, dtype, skip = c["world"], c["dtype"], c["skip_incomplete"]
    layers, S = shard_table(c)
    full = sharded_inputs(c, S)
    g = C.LocalReducerGroup(W, "SRA", TIMEOUT_MS)
    outs = [torch.full((S,), -7.25, dtype=dtype) for _ in range(W)]
    g.reduce_scatter(full, outs, layers, c["average"], skip)
    want = O.reduce_scatter_reference(full, layers, average=c["average"], skip_incomplete=skip)
    assert_results(outs, want, "vs reference")
    sim = [torch.empty(S, dtype=dtype) for _ in range(W)]
    C.reduce_scatter_simulate(full, sim, layers, 1, c["average"], skip)
    assert_results(outs, sim, "vs reduce_scatter_simulate")
    assert g.bytes_sent() == sharded_bytes_sent("reduce_scatter", layers, S, W, dtype, skip)


@pytest.mark.parametrize("c", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_host_all_gather(c):
    W, dtype, skip = c["world"], c["dtype"], c["skip_incomplete"]
    layers, S = shard_table(c)
    shards = own_shards(sharded_inputs(c, S))
    g = C.LocalReducerGroup(W, "SRA", TIMEOUT_MS)
    outs = [torch.full((W * S,), -7.25, dtype=dtype) for _ in range(W)]
    g.all_gather(shards, outs, layers, skip)
    assert_results(outs, [gather_with_skip(shards, layers, skip)] * W, "vs reference")
    if not skip:
        sim = [torch.empty(W * S, dtype=dtype) for _ in range(W)]
        C.all_gather_simulate(shards, sim, layers)
        assert_results(outs, sim, "vs all_gather_simulate")
    assert g.bytes_sent() == sharded_bytes_sent("all_gather", layers, S, W, dtype, skip)


@pytest.mark.parametrize("world,dtype", [(2, torch.float32), (3, torch.bfloat16), (5, torch.float16),
                                         (8, torch.float32), (16, torch.bfloat16)])
def test_host_stochastic_matches_the_simulators(world, dtype):
    S = S_MIXED
    full = inputs_for(world, world * S, dtype, 40 + world)
    g = C.LocalReducerGroup(world, "RING", TIMEOUT_MS)  # the sharded methods do not depend on the reducer kind
    outs = [torch.empty(S, dtype=dtype) for _ in range(world)]
    g.reduce_scatter(full, outs, MIXED, True, False, True, 9, 77, prescale=0.375)
    sim = [torch.empty(S, dtype=dtype) for _ in range(world)]
    C.reduce_scatter_simulate(full, sim, MIXED, 1, False, False, True, 9, 77, prescale=0.375)
    assert_results(outs, sim, "reduce-scatter")
    det = O.reduce_scatter_reference(full, MIXED, prescale=0.375)
    assert any(mismatch(a, b) for a, b in zip(outs, det)), "stochastic rounding had no effect"
    shards = own_shards(full)
    outs = [torch.empty(world * S, dtype=dtype) for _ in range(world)]
    g.all_gather(shards, outs, MIXED, False, True, 9, 78)
    sim = [torch.empty(world * S, dtype=dtype) for _ in range(world)]
    C.all_gather_simulate(shards, sim, MIXED, True, 9, 78)
    assert_results(outs, sim, "all-gather")


def test_host_in_place_all_gather():
    W, dtype = 3, torch.float16
    shards = inputs_for(W, S_MIXED, dtype, 5)
    outs = [torch.zeros(W * S_MIXED, dtype=dtype) for _ in range(W)]
    for r in range(W):
        outs[r][r * S_MIXED:(r + 1) * S_MIXED] = shards[r]
    g = C.LocalReducerGroup(W, "SRA", TIMEOUT_MS)
    g.all_gather([o[r * S_MIXED:(r + 1) * S_MIXED] for r, o in enumerate(outs)], outs, MIXED)
    assert_results(outs, [O.all_gather_reference(shards, MIXED)] * W, "in place")


# ---- the engine's two stages, on host memory ---------------------------------------------------------
def engine_case(op, world, local, cfg, dtype, *, average=False, table=MIXED, stochastic=False, seed=0, calls=1,
                monkeypatch=None):
    """`calls` sharded calls through a LocalEngineGroup without heaps, each checked against
    sharded_engine_reference (values and every rank's stage log)."""
    cfg = dict(cfg, p2p=False)
    S = sum(l[1] for l in table)
    if monkeypatch is not None:
        set_stochastic(monkeypatch, stochastic, seed)
    g = C.LocalEngineGroup(world, local, cfg, 1, 1 << 16, TIMEOUT_MS)
    rs = op == "reduce_scatter"
    for k in range(1, calls + 1):
        full = inputs_for(world, world * S, dtype, world * 7 + local + k)
        ins = full if rs else own_shards(full)
        outs = [torch.full((S if rs else world * S,), -7.25, dtype=dtype) for _ in range(world)]
        if rs:
            g.reduce_scatter(ins, outs, average, table)
        else:
            g.all_gather(ins, outs, table)
        want, stages = O.sharded_engine_reference(op, ins, table, local_size=local, config=cfg, lanes=1,
                                                  average=average, call_seq=k, cuda=False, stochastic=stochastic,
                                                  seed=seed)
        assert_results(outs, want, f"{op} call {k}")
        assert_log(g, stages, world)
    return g


@pytest.mark.parametrize("icomp", [True, False], ids=["icomp", "iraw"])
@pytest.mark.parametrize("world,local", TOPOLOGIES)
def test_engine_reduce_scatter(world, local, icomp, monkeypatch):
    dtype = DTYPES[(world + local) % 3]
    engine_case("reduce_scatter", world, local, dict(intra_compress=icomp), dtype, average=world % 4 == 0, calls=2,
                monkeypatch=monkeypatch)


@pytest.mark.parametrize("icomp", [True, False], ids=["icomp", "iraw"])
@pytest.mark.parametrize("world,local", TOPOLOGIES)
def test_engine_all_gather(world, local, icomp, monkeypatch):
    dtype = DTYPES[(world + local + 1) % 3]
    g = engine_case("all_gather", world, local, dict(intra_compress=icomp), dtype, calls=2, monkeypatch=monkeypatch)
    assert g.stats(0)["calls"] == 2


@pytest.mark.parametrize("world,local", [(4, 2), (6, 3), (4, 1), (8, 2)])
def test_engine_stochastic(world, local, monkeypatch):
    for op in ("reduce_scatter", "all_gather"):
        engine_case(op, world, local, dict(inner_reduction="RING", cross_reduction="ALLTOALL"), torch.float32,
                    average=True, stochastic=True, seed=world + local, calls=2, monkeypatch=monkeypatch)


def test_engine_default_table_and_skip_incomplete(monkeypatch):
    # no table: one layer of S with the environment's width and bucket; skip_incomplete for the reduce-scatter
    monkeypatch.setenv("CGX_COMPRESSION_QUANTIZATION_BITS", "3")
    monkeypatch.setenv("CGX_COMPRESSION_BUCKET_SIZE", "100")
    monkeypatch.setenv("CGX_COMPRESSION_SKIP_INCOMPLETE_BUCKETS", "1")
    W, L, S = 6, 2, 1234
    g = C.LocalEngineGroup(W, L, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    full = inputs_for(W, W * S, torch.bfloat16, 2)
    outs = [torch.empty(S, dtype=torch.bfloat16) for _ in range(W)]
    g.reduce_scatter(full, outs, True)
    want, stages = O.sharded_engine_reference("reduce_scatter", full, [(0, S, 3, 100)], local_size=L,
                                              config=dict(p2p=False), lanes=1, average=True, cuda=False,
                                              skip_incomplete=True)
    assert_results(outs, want, "reduce-scatter")
    assert_log(g, stages, W)
    outs = [torch.empty(W * S, dtype=torch.bfloat16) for _ in range(W)]
    g.all_gather(own_shards(full), outs)
    assert_results(outs, [O.all_gather_reference(own_shards(full), [(0, S, 3, 100)])] * W, "all-gather")


def test_engine_counters_follow_the_allreduce():
    # node-local stages count their elements, wire bytes and raw bytes; the cross-node stage is not counted
    W, L = 6, 3
    g = C.LocalEngineGroup(W, L, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    full = inputs_for(W, W * S_MIXED, torch.float32, 1)
    g.reduce_scatter(full, [torch.empty(S_MIXED) for _ in range(W)], False, MIXED)
    sent = sharded_bytes_sent("reduce_scatter", MIXED, S_MIXED, L, torch.float32, False)
    for r in range(W):
        st = g.stats(r)
        assert st["calls"] == 1 and st["kernel_launches"] == 0
        assert st["elements"] == (W // L) * L * S_MIXED
        assert st["wire_bytes"] == (W // L) * sent[r % L]
        assert st["raw_bytes"] == (W // L) * S_MIXED * (L - 1) * 4


# ---- the references tell wrong semantics apart -------------------------------------------------------
@pytest.mark.parametrize("perturb,op,world,local", [
    ("prescale_local", "reduce_scatter", 4, 2),
    ("quantized_own_partial", "reduce_scatter", 6, 3),
    ("transposed_ranks", "reduce_scatter", 6, 2),
    ("requantized_gather", "all_gather", 4, 2),
    ("transposed_ranks", "all_gather", 8, 4),
])
def test_reference_detects_wrong_semantics(perturb, op, world, local):
    assert perturb in O.SHARDED_PERTURBATIONS
    cfg = dict(p2p=False)
    g = C.LocalEngineGroup(world, local, cfg, 1, 1 << 16, TIMEOUT_MS)
    full = inputs_for(world, world * S_MIXED, torch.float32, 12)
    if op == "reduce_scatter":
        outs = [torch.empty(S_MIXED) for _ in range(world)]
        g.reduce_scatter(full, outs, True, MIXED)
        good = O.reduce_scatter_hier_reference(full, MIXED, local_size=local, average=True)
        bad = O.reduce_scatter_hier_reference(full, MIXED, local_size=local, average=True, perturb=perturb)
    else:
        shards = own_shards(full)
        outs = [torch.empty(world * S_MIXED) for _ in range(world)]
        g.all_gather(shards, outs, MIXED)
        good = O.all_gather_hier_reference(shards, MIXED, local_size=local)
        bad = O.all_gather_hier_reference(shards, MIXED, local_size=local, perturb=perturb)
    assert_results(outs, good, "unperturbed reference")
    assert any(mismatch(o, b) for o, b in zip(outs, bad)), f"{perturb} was not detected"


# ---- the harness -------------------------------------------------------------------------------------
def test_harness_rejects_bad_arguments():
    g = C.LocalEngineGroup(4, 2, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    full = inputs_for(4, 4 * 100, torch.float32, 1)
    with pytest.raises(Exception, match="W x S"):
        g.reduce_scatter(full, [torch.empty(99) for _ in range(4)], False, [(0, 99, 4, 8)])
    with pytest.raises(Exception, match="tile"):
        g.reduce_scatter(full, [torch.empty(100) for _ in range(4)], False, [(0, 90, 4, 8)])
    with pytest.raises(Exception, match="overlaps"):
        g.all_gather([t[50:150] for t in full], full, [(0, 100, 4, 8)])
    # the group stays usable after a rejected call
    outs = [torch.empty(100) for _ in range(4)]
    g.reduce_scatter(full, outs, False, [(0, 100, 4, 8)])
    assert_results(outs, O.reduce_scatter_hier_reference(full, [(0, 100, 4, 8)], local_size=2), "after a rejection")
    r = C.LocalReducerGroup(2, "SRA", TIMEOUT_MS)
    with pytest.raises(Exception, match="inputs of W \\* S"):
        r.reduce_scatter([torch.empty(10)] * 2, [torch.empty(4)] * 2, [(0, 4, 4, 8)])
