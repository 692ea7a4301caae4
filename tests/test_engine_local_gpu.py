"""The allreduce engine (engine/engine.cc) at world > 1 on ONE GPU: W real AllreduceEngines with
connect_local heaps and loopback generic reducers in one process (C.LocalEngineGroup). Every call's
values equal ``oracle.engine_reference`` bit for bit (NaN-aware) and every rank's stage log equals
the stage sequence the reference derives from the configuration: fusion groups past the 16-group
sequence wrap, sliced layers, one-shot and three-phase groups in one call, groups halved to fit the
heap slot, the registered-bucket fast path (replayed launches, RNG sequence numbers, plan reuse and
invalidation, the overlap lane cap), the two-level hierarchy on the device-memory generic reducers,
dummy compression, the byte counters and the sharded collectives. Each rank's tensor is a view at
element offset 1, 3 or 5 of a sentinel-filled buffer whose guard bands must stay intact. All
parameters are fixed lists."""
import pytest
import torch

from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same, mismatch
from _edge_inputs import edge_inputs
from _engine_cases import (C, TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, mixed_table, set_stochastic)
from _reducer_cases import expected_bytes_sent

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
GUARD = 64
SENTINEL = -7.25  # exact in every dtype
LANES = 2
FUSION = 16 << 10    # more than 16 groups per call
ONESHOT = 6 << 10    # groups up to 6 KiB take the one-shot kernel
SLOT = 4096          # raw groups of 16 KiB do not fit one chunk at W <= 3: they are halved
SINGLE_CFG = dict(fusion_bytes=FUSION, oneshot_max_bytes=ONESHOT, min_lane_elems=1024)


def single_cfg(dtype):
    """SINGLE_CFG with the byte limits scaled to the element size: the same groups in every dtype."""
    es = torch.empty(0, dtype=dtype).element_size()
    return dict(SINGLE_CFG, fusion_bytes=FUSION * es // 4, oneshot_max_bytes=ONESHOT * es // 4)


def guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device="cuda")
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def assert_guards(buf, offset, n, what):
    b = buf.cpu()
    assert_same(b[:offset], torch.full((offset,), SENTINEL, dtype=b.dtype), f"{what}: elements before the view")
    assert_same(b[offset + n:], torch.full((GUARD,), SENTINEL, dtype=b.dtype), f"{what}: elements after the view")


def run_guarded(fn, ins, offset):
    """fn(views) on CUDA views of `ins` at `offset` in guarded buffers; returns the results on the CPU."""
    bufs = [guarded(t, offset) for t in ins]
    views = [v for _, v in bufs]
    fn(views)
    torch.cuda.synchronize()
    for r, (buf, _) in enumerate(bufs):
        assert_guards(buf, offset, ins[0].numel(), f"rank {r}")
    return [v.cpu() for v in views]


def single_table(bits, bucket):
    """A raw head (odd offsets after it), a compressed layer larger than the fusion buffer (sliced),
    many small mixed layers that share groups, raw layers of whole groups."""
    sizes = [(37, 32, 512), (20_000, bits, bucket), (301, 32, 512), (2001, 5, 64)]
    sizes += [(1500 + 37 * i, (bits + i) % 8 + 1, (64, 512, 7, 1000)[i % 4]) for i in range(24)]
    sizes += [(4096, 32, 512), (6000, 32, 512), (777, 2, 8)]
    return mixed_table(sizes)


def kinds(stages):
    return [s["kind"] for s in stages]


# ---- single node -------------------------------------------------------------------------------------
SINGLE = [(2, torch.float32, 4, 512, False), (3, torch.float16, 1, 100, True), (4, torch.bfloat16, 8, 1024, False),
          (5, torch.float32, 3, 7, True), (8, torch.float16, 6, 256, False), (2, torch.bfloat16, 2, 8, True),
          (3, torch.float32, 7, 1, False), (4, torch.float16, 5, 64, True)]


@pytest.mark.parametrize("world,dtype,bits,bucket,average", SINGLE,
                         ids=[f"w{w}-{str(d)[6:]}-q{b}-b{k}-{'avg' if a else 'sum'}" for w, d, b, k, a in SINGLE])
def test_single_node(world, dtype, bits, bucket, average):
    layers, total = single_table(bits, bucket)
    cfg = single_cfg(dtype)
    g = C.LocalEngineGroup(world, world, cfg, LANES, SLOT, TIMEOUT_MS)
    ins = inputs_for(world, total, dtype, world * 10 + bits)
    # hostile values in the sliced layer: non-finite on an owner or a peer, spans that overflow, tiny...
    xs, _ = edge_inputs(dtype, 20_000, O.effective_bucket(bucket), bits, world=world, bits=bits,
                        where="peer" if average else "owner")
    for r in range(world):
        ins[r][37:20_037] = xs[r]
    want, stages = O.engine_reference(ins, layers, local_size=world, config=cfg, lanes=LANES,
                                      slot_bytes=g.slot_bytes(), average=average)
    got = run_guarded(lambda v: g.allreduce_layers(v, layers, average), ins, (1, 3, 5)[world % 3])
    assert_results(got, want, "engine vs reference")
    assert_log(g, stages, world)
    k = kinds(stages[0])
    groups = C.split_for_fusion(layers, torch.empty(0, dtype=dtype).element_size(), cfg["fusion_bytes"])
    assert len(groups) > 16, "the group index does not wrap"
    assert "oneshot" in k and "sra" in k, "one call should mix one-shot and three-phase groups"
    if dtype == torch.float32 and world <= 3:
        assert len(k) > len(groups), "no group was halved"


def test_stats_match_the_plans():
    W, dtype = 3, torch.float32
    layers, total = single_table(4, 512)
    g = C.LocalEngineGroup(W, W, SINGLE_CFG, LANES, SLOT, TIMEOUT_MS)
    ins = inputs_for(W, total, dtype, 2)
    _, stages = O.engine_reference(ins, layers, local_size=W, config=SINGLE_CFG, lanes=LANES,
                                   slot_bytes=g.slot_bytes())
    run_guarded(lambda v: g.allreduce_layers(v, layers, False), ins, 1)
    for r in range(W):
        wire = raw = elems = 0
        for s in stages[r]:
            one = s["kind"] == "oneshot"
            p = C.build_plan(s["layers"], world=1 if one else W, lanes=LANES, dtype=0,
                             min_lane_elems=SINGLE_CFG["min_lane_elems"])
            elems += p["numel"]
            if one:
                wire += p["total_wire"] * (W - 1)
                raw += p["numel"] * 4 * (W - 1)
            else:
                mine, my_elems = p["chunk_wire_bytes"][r], p["chunk_elems"][r]
                wire += p["total_wire"] - mine + mine * (W - 1)
                raw += ((p["numel"] - my_elems) + my_elems * (W - 1)) * 4
        st = g.stats(r)
        assert (st["calls"], st["kernel_launches"], st["elements"]) == (1, len(stages[r]), elems)
        assert (st["wire_bytes"], st["raw_bytes"]) == (wire, raw), f"rank {r}"


def test_generic_intra_stats():
    # inner_reduction=RING bypasses the fused kernel: the generic reducer's bytes on the device
    W, cfg = 3, dict(SINGLE_CFG, inner_reduction="RING", fusion_bytes=1 << 20)
    layers, total = mixed_table([(37, 32, 512), (9000, 4, 512), (1333, 3, 100)])
    g = C.LocalEngineGroup(W, W, cfg, LANES, SLOT, TIMEOUT_MS)
    ins = inputs_for(W, total, torch.bfloat16, 3)
    want, stages = O.engine_reference(ins, layers, local_size=W, config=cfg, lanes=LANES, slot_bytes=g.slot_bytes(),
                                      average=True)
    got = run_guarded(lambda v: g.allreduce_layers(v, layers, True), ins, 3)
    assert_results(got, want, "generic intra")
    assert_log(g, stages, W)
    sent = expected_bytes_sent("RING", layers, W, torch.bfloat16, False)
    for r in range(W):
        st = g.stats(r)
        assert st["wire_bytes"] == sent[r] and st["kernel_launches"] == 0
        assert st["raw_bytes"] == 2 * total * 2 * (W - 1) // W


# ---- registered buckets: the fast path -----------------------------------------------------------------
def register(bucket_idx, sizes):
    for i, (n, bits, bucket) in enumerate(sizes):
        C.register_layer(bucket_idx, i, n, bits, bucket)
    layers, total = mixed_table(sizes)
    assert C.extract_layers(total, bucket_idx)[0] == layers
    return layers, total


def plans(g, W):
    return [g.num_plans(r) for r in range(W)]


BUCKET_SIZES = [(37, 32, 512), (9000, 4, 512), (3000, 32, 512), (5000, 3, 100), (800, 8, 8)]


@pytest.mark.parametrize("stochastic", [False, True], ids=["det", "sr"])
@pytest.mark.parametrize("world,dtype", [(2, torch.float32), (3, torch.bfloat16), (4, torch.float16)])
def test_registered_bucket_replays_the_slow_path(world, dtype, stochastic, monkeypatch):
    # small slot and fusion buffer: groups are halved, so the replayed launches carry both the group
    # and the piece index in their RNG sequence
    set_stochastic(monkeypatch, stochastic, 77)
    cfg = dict(SINGLE_CFG, fusion_bytes=12 << 10, oneshot_max_bytes=2 << 10)
    layers, total = register(3, BUCKET_SIZES)
    g = C.LocalEngineGroup(world, world, cfg, LANES, 2560, TIMEOUT_MS)
    ins = inputs_for(world, total, dtype, world)
    state = [t.clone() for t in ins]
    first = None
    for call in (1, 2, 3):
        want, stages = O.engine_reference(state, layers, local_size=world, config=cfg, lanes=LANES,
                                          slot_bytes=g.slot_bytes(), average=True, call_seq=call,
                                          stochastic=stochastic, seed=77)
        before = plans(g, world)
        state = run_guarded(lambda v: g.allreduce(v, True, 3), state, call)
        assert_results(state, want, f"call {call}")
        assert_log(g, stages, world, fast=call > 1)
        if call == 1:
            first = [[dict(s, seq=None, layers=None) for s in g.log(r)] for r in range(world)]
            if world == 2:
                assert any(s["kind"] == "sra" and s["seq"] & 7 for s in stages[0]), "no group was halved"
        else:
            assert plans(g, world) == before, f"call {call} built a plan"
            assert [[dict(s, seq=None, layers=None) for s in g.log(r)] for r in range(world)] == first


def test_registered_bucket_invalidation(monkeypatch):
    W, dtype = 3, torch.float32
    cfg = dict(SINGLE_CFG, fusion_bytes=1 << 20)
    layers, total = register(1, BUCKET_SIZES)
    g = C.LocalEngineGroup(W, W, cfg, LANES, 1 << 16, TIMEOUT_MS)
    seq = [0]

    def call(ins, bucket, layers, *, overlapped=False, fresh):
        seq[0] += 1
        want, stages = O.engine_reference(ins, layers, local_size=W, config=cfg, lanes=LANES,
                                          slot_bytes=g.slot_bytes(), call_seq=seq[0], overlapped=overlapped)
        before = plans(g, W)
        got = run_guarded(lambda v: g.allreduce(v, False, bucket, overlapped), ins, 5)
        assert_results(got, want, f"call {seq[0]}")
        grew = [a > b for a, b in zip(plans(g, W), before)]
        assert all(grew) if fresh else not any(grew), f"call {seq[0]}: fresh plan {grew}, expected {fresh}"
        return stages

    ins = inputs_for(W, total, dtype, 1)
    call(ins, 1, layers, fresh=True)
    call(ins, 1, layers, fresh=False)
    # a registered width changes
    C.set_quantization_bits(1, 1, 6)
    layers6 = C.extract_layers(total, 1)[0]
    assert layers6 != layers
    call(ins, 1, layers6, fresh=True)
    call(ins, 1, layers6, fresh=False)
    # the dtype changes
    call([t.bfloat16() for t in ins], 1, layers6, fresh=True)
    # the size changes: no registered layout of that size, the environment's width for the whole buffer
    monkeypatch.setenv("CGX_COMPRESSION_QUANTIZATION_BITS", "4")
    short = [t[:total - 5].clone() for t in ins]
    call(short, 1, [(0, total - 5, 4, 512)], fresh=True)
    call(short, 1, [(0, total - 5, 4, 512)], fresh=False)
    # the environment's width changes
    monkeypatch.setenv("CGX_COMPRESSION_QUANTIZATION_BITS", "2")
    call(short, 1, [(0, total - 5, 2, 512)], fresh=True)
    # overlapped: at most overlap_lanes CTAs
    g2 = C.LocalEngineGroup(W, W, dict(cfg, overlap_lanes=1, oneshot_max_bytes=0), LANES, 1 << 16, TIMEOUT_MS)
    for overlapped in (False, True):
        want, stages = O.engine_reference(ins, layers6, local_size=W, config=dict(cfg, overlap_lanes=1,
                                          oneshot_max_bytes=0), lanes=LANES, slot_bytes=g2.slot_bytes(),
                                          call_seq=1 + overlapped, overlapped=overlapped)
        got = run_guarded(lambda v: g2.allreduce(v, False, 1, overlapped), ins, 1)
        assert_results(got, want, f"overlapped={overlapped}")
        assert_log(g2, stages, W)
        lanes = {s["lanes"] for s in stages[0]}
        assert lanes == {1} if overlapped else max(lanes) == LANES


# ---- two-level hierarchy -------------------------------------------------------------------------------
HIER = [
    dict(world=4, local=2, inner="SRA", cross="RING", bcast=True, icomp=True, stochastic=False),
    dict(world=6, local=3, inner="RING", cross="SRA", bcast=True, icomp=False, stochastic=True),
    dict(world=8, local=4, inner="SRA", cross="ALLTOALL", bcast=False, icomp=True, stochastic=False),
    dict(world=4, local=1, inner="SRA", cross="SRA", bcast=True, icomp=True, stochastic=True),
    dict(world=6, local=2, inner="SRA", cross="RING", bcast=False, icomp=False, stochastic=True),
    dict(world=8, local=4, inner="RING", cross="RING", bcast=True, icomp=True, stochastic=True),
    dict(world=4, local=2, inner="SRA", cross="ALLTOALL", bcast=True, icomp=False, stochastic=False),
    dict(world=6, local=3, inner="SRA", cross="SRA", bcast=True, icomp=True, stochastic=True),
]


def hier_id(h):
    return (f"w{h['world']}l{h['local']}-{h['inner']}-{h['cross']}-{'bcast' if h['bcast'] else 'nobcast'}-"
            f"{'icomp' if h['icomp'] else 'iraw'}-{'sr' if h['stochastic'] else 'det'}")


@pytest.mark.parametrize("h", HIER, ids=hier_id)
def test_hierarchy(h, monkeypatch):
    set_stochastic(monkeypatch, h["stochastic"], 31)
    cfg = dict(fusion_bytes=8 << 10, oneshot_max_bytes=3 << 10, min_lane_elems=1024, inner_reduction=h["inner"],
               cross_reduction=h["cross"], intra_broadcast=h["bcast"], intra_compress=h["icomp"])
    layers, total = mixed_table([(37, 32, 512), (9000, 4, 512), (301, 32, 512), (2001, 5, 64), (700, 2, 100),
                                 (1200, 8, 8)])
    W, L = h["world"], h["local"]
    dtype = DTYPES[W % 3]
    # several nodes share this one GPU and CUDA context: no heaps there, since a cudaFree in one
    # node's generic stage can wait for another node's fused kernel while that one waits for a peer
    # the same driver call holds up. The device-memory generic reducers run every stage instead.
    cfg["p2p"] = False
    g = C.LocalEngineGroup(W, L, cfg, LANES, 1 << 16, TIMEOUT_MS)
    state = inputs_for(W, total, dtype, W + L)
    for call in (1, 2):
        want, stages = O.engine_reference(state, layers, local_size=L, config=cfg, lanes=LANES,
                                          slot_bytes=g.slot_bytes(), average=call == 2, call_seq=call,
                                          stochastic=h["stochastic"], seed=31)
        state = run_guarded(lambda v: g.allreduce_layers(v, layers, call == 2), state, call * 2 - 1)
        assert_results(state, want, f"call {call}")
        assert_log(g, stages, W)


def test_dummy_compression_sums_exactly():
    W = 4
    cfg = dict(SINGLE_CFG, dummy_compression=True)
    layers, total = single_table(3, 64)
    g = C.LocalEngineGroup(W, W, cfg, LANES, SLOT, TIMEOUT_MS)
    gen = torch.Generator().manual_seed(3)
    ins = [torch.randint(-1000, 1000, (total,), generator=gen).float() for _ in range(W)]
    got = run_guarded(lambda v: g.allreduce_layers(v, layers, False), ins, 3)
    exact = sum(ins)
    for r in range(W):
        assert torch.equal(got[r], exact), f"rank {r}"


# ---- sharded collectives -------------------------------------------------------------------------------
@pytest.mark.parametrize("world,dtype", [(2, torch.float32), (3, torch.bfloat16), (5, torch.float16)])
def test_reduce_scatter_and_all_gather(world, dtype, monkeypatch):
    monkeypatch.setenv("CGX_COMPRESSION_QUANTIZATION_BITS", "4")
    monkeypatch.setenv("CGX_COMPRESSION_BUCKET_SIZE", "100")
    S = 7001
    g = C.LocalEngineGroup(world, world, dict(SINGLE_CFG), LANES, 1 << 16, TIMEOUT_MS)
    full = inputs_for(world, world * S, dtype, world)
    outs = [torch.zeros(S, dtype=dtype, device="cuda") for _ in range(world)]
    g.reduce_scatter([t.cuda() for t in full], outs, True)
    want = O.reduce_scatter_reference(full, [(0, S, 4, 100)], average=True)
    assert_results(outs, want, "reduce-scatter")
    shards = [t[:S].clone() for t in full]
    gathered = [torch.zeros(world * S, dtype=dtype, device="cuda") for _ in range(world)]
    g.all_gather([t.cuda() for t in shards], gathered)
    ref = O.all_gather_reference(shards, [(0, S, 4, 100)])
    assert_results(gathered, [ref] * world, "all-gather")
    assert g.stats(0)["calls"] == 2


# ---- the reference tells wrong semantics apart -------------------------------------------------------
def test_reference_detects_shifted_oneshot_threshold():
    W, dtype = 3, torch.float32
    layers, total = single_table(4, 512)
    g = C.LocalEngineGroup(W, W, SINGLE_CFG, LANES, SLOT, TIMEOUT_MS)
    ins = inputs_for(W, total, dtype, 8)
    got = run_guarded(lambda v: g.allreduce_layers(v, layers, True), ins, 1)
    kw = dict(local_size=W, config=SINGLE_CFG, lanes=LANES, slot_bytes=g.slot_bytes(), average=True)
    good, _ = O.engine_reference(ins, layers, **kw)
    assert_results(got, good, "unperturbed reference")
    bad, _ = O.engine_reference(ins, layers, perturb="oneshot_shifted", **kw)
    assert any(mismatch(a, b) for a, b in zip(got, bad)), "the shifted one-shot threshold was not detected"


# ---- the harness -----------------------------------------------------------------------------------------
def test_group_refuses_non_resident_heaps():
    resident = min(C.max_resident_ctas(d) for d in (0, 1, 2))
    with pytest.raises(Exception, match="cannot all be resident"):
        C.LocalEngineGroup(4, 4, {}, resident // 8 + 1, 1 << 16, TIMEOUT_MS)
    with pytest.raises(Exception, match="cannot all be resident"):
        C.LocalEngineGroup(8, 4, {}, resident // 16 + 1, 1 << 16, TIMEOUT_MS)
