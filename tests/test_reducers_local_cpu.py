"""The generic reducers (reduce/reducers.cc) on host memory, with W virtual ranks in one process
(C.LocalReducerGroup: one host thread per rank, loopback transport), against the independent
references of torch_cgx_b200/ops/oracle.py, bit for bit and NaN-aware: SRA, Ring, the debug
all-to-all and the compressed broadcast, W 1-16, all dtypes, bits 1-8 and raw, bucket sizes 1 to
10000 (clamped), averaging, skip_incomplete, mixed tables at odd offsets, hostile inputs, chunks
that are empty. Perturbed references (wrong semantics) are told apart from the reducers, and the
bytes each rank sends match the plan. All parameters are fixed lists."""
import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same, mismatch
from _reducer_cases import (OPS, config_id, configs, expected_bytes_sent, group_for, make_case, reference,
                            run_op)

C = cgx._C
CONFIGS = configs()


def run_host(op, ins, layers, **kw):
    g = group_for(op, len(ins), record=True)
    out = [t.clone() for t in ins]
    run_op(g, op, out, layers, **kw)
    return out, g


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("c", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_host_reducers_match_reference(c, op):
    ins, layers = make_case(c)
    kw = dict(skip_incomplete=c["skip_incomplete"])
    if not op.startswith("BCAST"):
        kw["average"] = c["average"]
    got, g = run_host(op, ins, layers, **kw)
    ref = reference(op, ins, layers, **kw)
    for r in range(c["world"]):
        assert_same(got[r], ref[r], f"{op} rank {r} vs reference")
    if op == "SRA":
        sim = [t.clone() for t in ins]
        C.sra_simulate(sim, layers, 1, c["average"], c["skip_incomplete"], False, 0, 0, O.GENERIC_MIN_LANE_ELEMS)
        for r in range(c["world"]):
            assert_same(got[r], sim[r], f"SRA rank {r} vs sra_simulate")
    if op != "ALLTOALL":  # inside the layers every rank ends with the same values
        inside = torch.zeros(ins[0].numel(), dtype=torch.bool)
        for off, m, _, _ in O.layer_segments(layers, c["skip_incomplete"]):
            inside[off:off + m] = True
        for r in range(c["world"]):
            assert_same(got[r][inside], got[0][inside], f"{op}: rank {r} differs from rank 0")
    want = expected_bytes_sent(op, layers, c["world"], c["dtype"], c["skip_incomplete"])
    assert g.bytes_sent() == want, f"{op}: bytes sent {g.bytes_sent()} != plan {want}"
    per_src = [0] * c["world"]
    for _, src, _, data in g.messages():
        per_src[src] += data.numel()
    assert per_src == want, f"{op}: recorded messages {per_src} != plan {want}"


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("world,n", [(8, 33), (16, 5), (16, 70), (5, 1), (3, 2)])
def test_host_reducers_with_empty_chunks(world, n, op):
    # fewer blocks than ranks: some ranks own nothing and send empty chunks
    dtype = torch.float16 if n % 2 else torch.float32
    layers = [(0, n, 4, 8)] if n > 2 else [(0, n, 2, 1)]
    g = torch.Generator().manual_seed(world * n)
    ins = [(torch.randn(n, generator=g) * (r + 1)).to(dtype) for r in range(world)]
    plan = C.build_plan(layers, world=world, lanes=1, dtype=0 if dtype == torch.float32 else 1)
    assert any(b == 0 for b in plan["chunk_wire_bytes"]), "every rank owns a chunk"
    got, _ = run_host(op, ins, layers)
    ref = reference(op, ins, layers)
    for r in range(world):
        assert_same(got[r], ref[r], f"{op} rank {r}")


def test_host_stochastic_is_deterministic_and_bounded():
    # no bit-exact reference with stochastic rounding: two runs agree, and the result stays near the sum
    W, layers = 4, [(0, 6000, 3, 100)]
    g = torch.Generator().manual_seed(5)
    ins = [torch.randn(6000, generator=g) for _ in range(W)]
    exact = sum(t.double() for t in ins)
    for op in ("SRA", "RING"):
        a, _ = run_host(op, ins, layers, stochastic=True, seed=9, seq=1)
        b, _ = run_host(op, ins, layers, stochastic=True, seed=9, seq=1)
        d, _ = run_host(op, ins, layers, stochastic=True, seed=10, seq=1)
        assert_same(a[0], b[0], f"{op}: stochastic run repeated")
        assert mismatch(a[0], d[0]), f"{op}: the seed changes nothing"
        span = max(float(t.max() - t.min()) for t in ins) * W
        assert (a[0].double() - exact).abs().max() < span / 7 * W


# ---- the references tell wrong semantics apart ----------------------------------------------------
def _ring_variant(ins, layers, *, quantize_own=False, chunk_bucket_grid=False, raw_hop=None):
    """A copy of ring_reference with one semantic change switched on (none: identical)."""
    W, dtype, n = len(ins), ins[0].dtype, ins[0].numel()
    segs = O.layer_segments(layers, False)
    chunk = O.block_owners(layers, n, W, 1, dtype, False, O.GENERIC_MIN_LANE_ELEMS)
    starts = {c: int(np.flatnonzero(chunk == c)[0]) for c in range(W) if (chunk == c).any()}

    def Q(v):
        out = v.copy()
        for off, m, bits, bucket in segs:
            if bits >= 32 or not chunk_bucket_grid:
                out[off:off + m] = O._contribution(v[off:off + m], bits, bucket, dtype)
                continue
            # buckets counted from the start of the chunk that holds the layer's first element
            shift = (off - starts[int(chunk[off])]) % bucket
            w = np.concatenate([np.repeat(v[off:off + 1], shift), v[off:off + m]])
            out[off:off + m] = O._qdq_buckets(w, bits, bucket)[0][shift:]
        return out

    acc = [t.float().numpy().copy() for t in ins]
    if quantize_own:
        acc = [Q(a) for a in acc]
    for s in range(W - 1):
        sent = [a.copy() if s == raw_hop else Q(a) for a in acc]
        for r in range(W):
            sel = chunk == (r - s) % W
            acc[(r + 1) % W][sel] = acc[(r + 1) % W][sel] + sent[r][sel]
    out = ins[0].float().numpy().copy()
    for c in range(W):
        sel = chunk == c
        out[sel] = Q(acc[(c - 1) % W])[sel]
    return torch.from_numpy(out).to(dtype)


def _alltoall_variant(ins, layers, *, reverse_peers=False):
    W, dtype = len(ins), ins[0].dtype
    segs = O.layer_segments(layers, False)
    xs = [t.float().numpy() for t in ins]
    qs = [O._quantized(x, segs, dtype) for x in xs]
    acc = xs[0].copy()
    for q in (reversed(range(1, W)) if reverse_peers else range(1, W)):
        acc = acc + qs[q]
    return torch.from_numpy(acc).to(dtype)


@pytest.mark.parametrize("perturbation", ["none", "quantize_own", "chunk_bucket_grid", "raw_hop", "reverse_peers"])
def test_reference_detects_wrong_semantics(perturbation):
    # the 4-bit layer starts at an odd offset inside rank 0's chunk; four ranks so that hops and peer order matter
    layers = [(0, 37, 32, 512), (37, 9000, 4, 512), (9037, 1333, 3, 100)]
    W = 4
    g = torch.Generator().manual_seed(1)
    ins = [torch.randn(10_370, generator=g) * (r + 1) for r in range(W)]
    if perturbation in ("none", "reverse_peers"):
        got, _ = run_host("ALLTOALL", ins, layers)
        v = _alltoall_variant(ins, layers, reverse_peers=perturbation == "reverse_peers")
        if perturbation == "none":
            assert_same(v, got[0])
        else:
            assert mismatch(v, got[0]), "reverse_peers was not detected"
    if perturbation != "reverse_peers":
        got, _ = run_host("RING", ins, layers)
        kw = {"raw_hop": 1} if perturbation == "raw_hop" else {} if perturbation == "none" else {perturbation: True}
        v = _ring_variant(ins, layers, **kw)
        if perturbation == "none":
            assert_same(v, got[0])
            assert_same(v, O.ring_reference(ins, layers)[0])
        else:
            assert mismatch(v, got[0]), f"{perturbation} was not detected"


# ---- the harness itself -----------------------------------------------------------------------------
def test_group_rejects_bad_arguments():
    with pytest.raises(Exception, match="kind"):
        C.LocalReducerGroup(2, "TREE", 1000)
    with pytest.raises(Exception, match="world"):
        C.LocalReducerGroup(17, "SRA", 1000)
    g = C.LocalReducerGroup(3, "RING", 1000)
    with pytest.raises(Exception, match="one tensor per virtual rank"):
        g.allreduce([torch.zeros(10)] * 2, [(0, 10, 4, 8)])
    with pytest.raises(Exception, match="one dtype, size"):
        g.allreduce([torch.zeros(10), torch.zeros(10), torch.zeros(11)], [(0, 10, 4, 8)])
    # the group stays usable after a rejected call
    ins = [torch.randn(100) for _ in range(3)]
    out = [t.clone() for t in ins]
    g.allreduce(out, [(0, 100, 4, 8)])
    assert_same(out[1], O.ring_reference(ins, [(0, 100, 4, 8)])[1])
