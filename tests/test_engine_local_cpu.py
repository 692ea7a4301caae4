"""The allreduce engine (engine/engine.cc) on host memory with W virtual ranks in one process
(C.LocalEngineGroup): fusion groups, the generic intra-node reducers, the two-level hierarchy with
every cross-node reducer and both broadcasts, averaging, stochastic rounding. Each call's values must
equal ``oracle.engine_reference`` bit for bit (NaN-aware) and each rank's stage log must equal the
stage sequence the reference derives from the configuration. All parameters are fixed lists."""
import pytest
import torch

from torch_cgx_b200.ops import oracle as O

from _bitwise import mismatch
from _engine_cases import (C, TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, mixed_table, set_stochastic)

DTYPES = [torch.float32, torch.float16, torch.bfloat16]
# raw head (the next layer starts at an odd offset), a layer larger than the fusion buffer (sliced),
# a raw layer, small compressed layers that share groups
TABLE = [(37, 32, 512), (9000, 4, 512), (301, 32, 512), (2001, 5, 64), (700, 2, 100), (1200, 8, 8), (513, 3, 1)]
FUSION = 8192


def run_case(world, local, cfg, dtype, *, average, stochastic=False, seed=0, calls=1, table=TABLE, monkeypatch=None):
    cfg = dict(cfg, p2p=False, fusion_bytes=cfg.get("fusion_bytes", FUSION))
    layers, total = mixed_table(table)
    g = C.LocalEngineGroup(world, local, cfg, 1, 1 << 16, TIMEOUT_MS)
    if monkeypatch is not None:
        set_stochastic(monkeypatch, stochastic, seed)
    ins = inputs_for(world, total, dtype, world * 7 + local)
    state = [t.clone() for t in ins]
    for k in range(1, calls + 1):
        want, stages = O.engine_reference(state, layers, local_size=local, config=cfg, lanes=1, average=average,
                                          call_seq=k, cuda=False, stochastic=stochastic, seed=seed)
        g.allreduce_layers(state, layers, average)
        assert_results(state, want, f"call {k}")
        assert_log(g, stages, world)
    return g, ins, layers


SINGLE = [(2, "SRA"), (3, "RING"), (5, "ALLTOALL"), (4, "SRA"), (8, "RING")]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("world,inner", SINGLE)
def test_single_node_generic(world, inner, dtype, monkeypatch):
    g, _, _ = run_case(world, world, dict(inner_reduction=inner), dtype, average=world % 2 == 0, calls=2,
                       monkeypatch=monkeypatch)
    groups = C.split_for_fusion(mixed_table(TABLE)[0], torch.empty(0, dtype=dtype).element_size(), FUSION)
    assert len(groups) > 3 and any(len(gr) > 1 for gr in groups), "no fusion to test"
    assert g.stats(0)["calls"] == 2


# (W, L) x every hierarchy switch: each value of each appears, stochastic and deterministic alike
HIER = [
    dict(world=4, local=2, inner="SRA", cross="RING", bcast=True, icomp=True, stochastic=False),
    dict(world=6, local=3, inner="RING", cross="SRA", bcast=True, icomp=False, stochastic=False),
    dict(world=8, local=4, inner="ALLTOALL", cross="ALLTOALL", bcast=False, icomp=True, stochastic=False),
    dict(world=4, local=1, inner="SRA", cross="SRA", bcast=True, icomp=True, stochastic=False),
    dict(world=6, local=2, inner="SRA", cross="RING", bcast=False, icomp=False, stochastic=False),
    dict(world=4, local=2, inner="RING", cross="ALLTOALL", bcast=True, icomp=True, stochastic=True),
    dict(world=6, local=3, inner="SRA", cross="RING", bcast=False, icomp=True, stochastic=True),
    dict(world=8, local=4, inner="SRA", cross="SRA", bcast=True, icomp=False, stochastic=True),
    dict(world=4, local=1, inner="RING", cross="RING", bcast=False, icomp=False, stochastic=True),
    dict(world=6, local=2, inner="ALLTOALL", cross="SRA", bcast=True, icomp=True, stochastic=True),
]


def hier_id(h):
    return (f"w{h['world']}l{h['local']}-{h['inner']}-{h['cross']}-{'bcast' if h['bcast'] else 'nobcast'}-"
            f"{'icomp' if h['icomp'] else 'iraw'}-{'sr' if h['stochastic'] else 'det'}")


@pytest.mark.parametrize("h", HIER, ids=hier_id)
def test_hierarchy(h, monkeypatch):
    cfg = dict(inner_reduction=h["inner"], cross_reduction=h["cross"], intra_broadcast=h["bcast"],
               intra_compress=h["icomp"])
    dtype = DTYPES[h["world"] % 3]
    run_case(h["world"], h["local"], cfg, dtype, average=h["world"] % 4 == 0, stochastic=h["stochastic"],
             seed=h["world"] * 3, calls=2, monkeypatch=monkeypatch)


def test_dummy_compression_sums_exactly(monkeypatch):
    # integers: every partial sum is exact in fp32, so a raw allreduce gives the exact sum everywhere
    cfg = dict(dummy_compression=True, p2p=False, fusion_bytes=FUSION, cross_reduction="SRA")
    layers, total = mixed_table(TABLE)
    W = 4
    g = C.LocalEngineGroup(W, 2, cfg, 1, 1 << 16, TIMEOUT_MS)
    gen = torch.Generator().manual_seed(3)
    ins = [torch.randint(-1000, 1000, (total,), generator=gen).float() for _ in range(W)]
    out = [t.clone() for t in ins]
    g.allreduce_layers(out, layers, False)
    exact = sum(ins)
    for r in range(W):
        assert torch.equal(out[r], exact), f"rank {r}"
    assert all(s["kind"] != "bcast_compressed" for s in g.log(0))


def test_registered_layers_on_host(monkeypatch):
    # allreduce() resolves the layer table from the registry, as the process group does
    sizes = [(37, 32, 512), (5000, 3, 256), (333, 6, 7)]
    for i, (n, bits, bucket) in enumerate(sizes):
        C.register_layer(2, i, n, bits, bucket)
    layers, total = mixed_table(sizes)
    assert C.extract_layers(total, 2)[0] == layers
    cfg = dict(p2p=False, fusion_bytes=4096, inner_reduction="RING")
    g = C.LocalEngineGroup(3, 3, cfg, 1, 1 << 16, TIMEOUT_MS)
    ins = inputs_for(3, total, torch.float32, 1)
    out = [t.clone() for t in ins]
    g.allreduce(out, True, 2)
    want, stages = O.engine_reference(ins, layers, local_size=3, config=cfg, lanes=1, average=True, cuda=False)
    assert_results(out, want, "registered bucket")
    assert_log(g, stages, 3)


# ---- the reference tells wrong semantics apart -------------------------------------------------------
@pytest.mark.parametrize("perturb,h", [
    ("prescale_local", dict(world=4, local=2, cfg=dict(inner_reduction="SRA"), stochastic=False)),
    ("raw_broadcast", dict(world=4, local=2, cfg=dict(inner_reduction="RING"), stochastic=False)),
    ("cross_seq_unmarked", dict(world=4, local=2, cfg=dict(cross_reduction="SRA"), stochastic=True)),
])
def test_reference_detects_wrong_semantics(perturb, h, monkeypatch):
    cfg = dict(h["cfg"], p2p=False, fusion_bytes=FUSION)
    layers, total = mixed_table(TABLE)
    set_stochastic(monkeypatch, h["stochastic"], 5)
    g = C.LocalEngineGroup(h["world"], h["local"], cfg, 1, 1 << 16, TIMEOUT_MS)
    ins = inputs_for(h["world"], total, torch.float32, 9)
    out = [t.clone() for t in ins]
    g.allreduce_layers(out, layers, True)
    kw = dict(local_size=h["local"], config=cfg, lanes=1, average=True, cuda=False, stochastic=h["stochastic"],
              seed=5)
    good, _ = O.engine_reference(ins, layers, **kw)
    assert_results(out, good, "unperturbed reference")
    bad, _ = O.engine_reference(ins, layers, perturb=perturb, **kw)
    assert any(mismatch(o, b) for o, b in zip(out, bad)), f"{perturb} was not detected"


# ---- the harness itself -----------------------------------------------------------------------------
def test_group_rejects_bad_arguments():
    with pytest.raises(Exception, match="at most 8 ranks per node"):
        C.LocalEngineGroup(16, 16, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises(Exception, match="does not divide"):
        C.LocalEngineGroup(6, 4, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises(Exception, match="unknown config key"):
        C.LocalEngineGroup(2, 2, dict(p2p=False, fusion_mb=1), 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises(Exception, match="SRA, RING or ALLTOALL"):
        C.LocalEngineGroup(2, 2, dict(p2p=False, cross_reduction="TREE"), 1, 1 << 16, TIMEOUT_MS)
    g = C.LocalEngineGroup(2, 1, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises(Exception, match="one tensor per virtual rank"):
        g.allreduce_layers([torch.zeros(10)], [(0, 10, 4, 8)], False)
    # the group stays usable after a rejected call
    ins = inputs_for(2, 100, torch.float32, 4)
    out = [t.clone() for t in ins]
    g.allreduce_layers(out, [(0, 100, 4, 8)], False)
    want, _ = O.engine_reference(ins, [(0, 100, 4, 8)], local_size=1, config=dict(p2p=False), lanes=1, cuda=False)
    assert_results(out, want, "after a rejected call")
