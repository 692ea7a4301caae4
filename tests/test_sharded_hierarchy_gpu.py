"""The compressed reduce-scatter and all-gather over several nodes, on ONE GPU.

The generic reducers' Reducer::reduce_scatter / ::all_gather through the device backend equal the
host path bit for bit (every case of the host tier, stochastic rounding included). W
AllreduceEngines in one process (C.LocalEngineGroup) run the two-stage composition on device
memory: without heaps (generic reducers in both stages) at every (W, L) of ``TOPOLOGIES``, and with
heaps (fused rs_kernel / ag_kernel launches inside each node, several windows per launch group, next
to the device-memory cross-node stage) at (4, 2), (6, 3), (8, 2) and (8, 4). Values equal
``oracle.sharded_engine_reference`` bit for bit and every rank's stage log equals the reference's.
On one node the NCCL-transport path (generic intra-node reducer) gives the fused kernels' bytes.
With several GPUs (``-m multigpu``, ``CGX_LOCAL_SIZE`` nodes): the public API against the
hierarchical references, and an FSDP2 MLP with both compressed comms tracks NCCL. All parameters are
fixed lists."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _engine_cases import (C, TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, set_stochastic)
from _reducer_cases import config_id, configs
from _sharded_cases import TOPOLOGIES, own_shards, sharded_inputs, shard_table

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
CONFIGS = configs()
MIXED = [(0, 37, 32, 512), (37, 3000, 4, 100), (3037, 301, 32, 512), (3338, 1501, 3, 7), (4839, 700, 8, 1024)]
S_MIXED = 5539
LANES = 2
SLOT = 4096  # several windows per fused stage


# ---- the generic reducers through the device backend ---------------------------------------------------
def reducer_run(op, c, device, stochastic):
    W, dtype, skip = c["world"], c["dtype"], c["skip_incomplete"]
    layers, S = shard_table(c)
    full = sharded_inputs(c, S)
    g = C.LocalReducerGroup(W, "SRA", TIMEOUT_MS)
    if op == "reduce_scatter":
        ins = [t.to(device) for t in full]
        outs = [torch.full((S,), -7.25, dtype=dtype, device=device) for _ in range(W)]
        g.reduce_scatter(ins, outs, layers, c["average"], skip, stochastic, 5, 9)
    else:
        ins = [t.to(device) for t in own_shards(full)]
        outs = [torch.full((W * S,), -7.25, dtype=dtype, device=device) for _ in range(W)]
        g.all_gather(ins, outs, layers, skip, stochastic, 5, 9)
    return [o.cpu() for o in outs], g.bytes_sent()


@pytest.mark.parametrize("op", ["reduce_scatter", "all_gather"])
@pytest.mark.parametrize("c", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_device_reducers_match_host(c, op):
    stochastic = c["seed"] % 2 == 1
    dev, dev_sent = reducer_run(op, c, "cuda", stochastic)
    host, host_sent = reducer_run(op, c, "cpu", stochastic)
    assert_results(dev, host, f"{op} device vs host")
    assert dev_sent == host_sent


# ---- the engine ------------------------------------------------------------------------------------------
def engine_case(op, g, world, local, cfg, dtype, *, average=False, stochastic=False, seed=0, calls=2, monkeypatch):
    set_stochastic(monkeypatch, stochastic, seed)
    rs = op == "reduce_scatter"
    S = S_MIXED
    for k in range(1, calls + 1):
        full = inputs_for(world, world * S, dtype, world * 11 + local + k)
        ins = full if rs else own_shards(full)
        outs = [torch.full((S if rs else world * S,), -7.25, dtype=dtype, device="cuda") for _ in range(world)]
        dev_in = [t.cuda() for t in ins]
        if rs:
            g.reduce_scatter(dev_in, outs, average, MIXED)
        else:
            g.all_gather(dev_in, outs, MIXED)
        torch.cuda.synchronize()
        want, stages = O.sharded_engine_reference(op, ins, MIXED, local_size=local, config=cfg, lanes=LANES,
                                                  slot_bytes=g.slot_bytes(), average=average, call_seq=k,
                                                  stochastic=stochastic, seed=seed)
        assert_results(outs, want, f"{op} call {k}")
        assert_log(g, stages, world)
        for s in stages[0]:
            assert s["kind"] not in ("rs", "ag") or s["numel"] > 0
    return g


@pytest.mark.parametrize("op", ["reduce_scatter", "all_gather"])
@pytest.mark.parametrize("world,local", TOPOLOGIES)
def test_engine_without_heaps(world, local, op, monkeypatch):
    cfg = dict(p2p=False, intra_compress=world % 4 != 0)
    g = C.LocalEngineGroup(world, local, cfg, LANES, 1 << 16, TIMEOUT_MS)
    engine_case(op, g, world, local, cfg, DTYPES[(world + local) % 3], average=local % 2 == 0,
                stochastic=world == 6, seed=world, monkeypatch=monkeypatch)


HEAPS = [
    dict(world=4, local=2, icomp=True, stochastic=False),
    dict(world=6, local=3, icomp=False, stochastic=True),
    dict(world=8, local=2, icomp=True, stochastic=True),
    dict(world=8, local=4, icomp=False, stochastic=False),
]


@pytest.mark.parametrize("op", ["reduce_scatter", "all_gather"])
@pytest.mark.parametrize("h", HEAPS, ids=[f"w{h['world']}l{h['local']}-{'icomp' if h['icomp'] else 'iraw'}-"
                                          f"{'sr' if h['stochastic'] else 'det'}" for h in HEAPS])
def test_engine_with_heaps(h, op, monkeypatch):
    # fused launches inside each node next to the generic cross-node stage: the group quiesces every
    # rank before each sharded stage (LocalEngineGroup's observer)
    W, L = h["world"], h["local"]
    cfg = dict(intra_compress=h["icomp"], min_lane_elems=1024)
    g = C.LocalEngineGroup(W, L, cfg, LANES, SLOT, TIMEOUT_MS)
    dtype = DTYPES[W % 3]
    engine_case(op, g, W, L, cfg, dtype, average=True, stochastic=h["stochastic"], seed=W + L,
                monkeypatch=monkeypatch)
    kinds = [s["kind"] for s in g.log(0)]
    fused = "rs" if op == "reduce_scatter" else "ag"
    assert kinds.count(fused) > W // L, "no node-local stage was cut into several windows"
    st = g.stats(0)
    assert st["kernel_launches"] == 2 * kinds.count(fused)  # two calls, the same launches


@pytest.mark.parametrize("stochastic", [False, True], ids=["det", "sr"])
@pytest.mark.parametrize("world,dtype", [(2, torch.float32), (3, torch.bfloat16), (5, torch.float16)])
def test_single_node_generic_matches_fused(world, dtype, stochastic, monkeypatch):
    # CGX_INNER_COMMUNICATOR_TYPE=NCCL on one node: the generic intra-node reducer, same bytes as the kernels
    set_stochastic(monkeypatch, stochastic, 3)
    fused = C.LocalEngineGroup(world, world, dict(min_lane_elems=1024), LANES, SLOT, TIMEOUT_MS)
    generic = C.LocalEngineGroup(world, world, dict(p2p=False), LANES, SLOT, TIMEOUT_MS)
    full = [t.cuda() for t in inputs_for(world, world * S_MIXED, dtype, world)]
    got = {}
    for name, g in (("fused", fused), ("generic", generic)):
        rs = [torch.empty(S_MIXED, dtype=dtype, device="cuda") for _ in range(world)]
        g.reduce_scatter(full, rs, True, MIXED)
        ag = [torch.empty(world * S_MIXED, dtype=dtype, device="cuda") for _ in range(world)]
        g.all_gather(rs, ag, MIXED)
        torch.cuda.synchronize()
        got[name] = [t.cpu() for t in rs + ag]
    assert_results(got["generic"], got["fused"], "generic vs fused")
    assert {s["kind"] for s in generic.log(0)} == {"generic_ag"}
    assert {s["kind"] for s in fused.log(0)} == {"ag"}
    if not stochastic:
        want = O.reduce_scatter_reference([t.cpu() for t in full], MIXED, average=True)
        assert_results(got["fused"][:world], want, "reduce-scatter vs reference")


# ---- several GPUs, CGX_LOCAL_SIZE nodes ------------------------------------------------------------------
def _pg_hier(rank, world):
    local = int(os.environ["CGX_LOCAL_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        assert cgx.get_backend().local_size() == local
        for dtype in DTYPES:
            for bits, bucket, average in ((2, 512, False), (4, 100, True), (8, 1024, False)):
                S = 70_001
                full = inputs_for(world, world * S, dtype, world + bits)
                out = torch.empty(S, dtype=dtype, device="cuda")
                cgx.reduce_scatter_tensor(out, full[rank].cuda(), bits=bits, bucket_size=bucket, average=average)
                ref = O.reduce_scatter_hier_reference(full, [(0, S, bits, bucket)], local_size=local, average=average)
                assert_same(out.cpu(), ref[rank], f"reduce-scatter {dtype} bits {bits}")
                shards = own_shards(full)
                gathered = torch.empty(world * S, dtype=dtype, device="cuda")
                cgx.all_gather_into_tensor(gathered, shards[rank].cuda(), bits=bits, bucket_size=bucket)
                assert_same(gathered.cpu(), O.all_gather_reference(shards, [(0, S, bits, bucket)]),
                            f"all-gather {dtype} bits {bits}")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world,local", [(4, 2), (8, 4)])
def test_public_api_across_nodes(world, local):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_hier, world, env={"CGX_LOCAL_SIZE": str(local)}, timeout=600)


def _fsdp_mlp_both(rank, world, steps):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        losses = {}
        for kind in ("nccl", "cgx"):
            torch.manual_seed(0)
            model = torch.nn.Sequential(*[torch.nn.Sequential(torch.nn.Linear(512, 512), torch.nn.GELU())
                                          for _ in range(4)], torch.nn.Linear(512, 10)).cuda()
            for m in model[:4]:
                fully_shard(m)
            fully_shard(model)
            if kind == "cgx":
                cgx.set_cgx_reduce_scatter(model, bits=8)
                cgx.set_cgx_all_gather(model, bits=8)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            g = torch.Generator(device="cuda").manual_seed(rank)
            before = cgx.get_backend().stats()[0]
            out = []
            for _ in range(steps):
                x = torch.randn(64, 512, device="cuda", generator=g)
                y = (x[:, :10] > 0).float().argmax(1)
                loss = torch.nn.functional.cross_entropy(model(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad()
                out.append(loss.item())
            calls = cgx.get_backend().stats()[0] - before
            assert (calls > 0) == (kind == "cgx"), f"{kind}: {calls} compressed calls"
            losses[kind] = np.array(out)
        # 8-bit gradients and weights: the loss curve stays within 2% of the uncompressed one
        assert np.all(np.abs(losses["cgx"] - losses["nccl"]) <= 0.02 * losses["nccl"]), losses
        assert losses["cgx"][-1] < losses["cgx"][0]
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world,local", [(4, 2), (8, 4)])
def test_fsdp2_mlp_across_nodes_tracks_nccl(world, local):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_fsdp_mlp_both, world, args=(20,), env={"CGX_LOCAL_SIZE": str(local)}, timeout=600)
