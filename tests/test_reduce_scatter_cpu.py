"""The CPU simulator of the compressed reduce-scatter (C.reduce_scatter_simulate, the arithmetic of
rs_kernel) against the independent NumPy reference (ops/oracle.py reduce_scatter_reference), bit for
bit and NaN-aware, plus the plan and window properties the kernel relies on."""
import numpy as np
import pytest
import torch
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same, mismatch
from _edge_inputs import CASES, FINITE, edge_inputs

C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
LANES, MIN_LANE = 3, 64

layer = st.tuples(st.integers(1, 2000), st.sampled_from([1, 2, 3, 4, 5, 6, 7, 8, 32]),
                  st.sampled_from([1, 3, 7, 8, 16, 32, 64, 100, 256, 512, 1000, 1024, 10_000]))
case = st.fixed_dictionaries({
    "specs": st.lists(layer, min_size=1, max_size=4),
    "world": st.integers(1, 16),
    "dtype": st.sampled_from(DTYPES),
    "average": st.booleans(),
    "skip_incomplete": st.booleans(),
    "source": st.sampled_from(["randn", "edge_owner", "edge_peer"]),
    "seed": st.integers(0, 2 ** 20),
})


def shard_table(specs):
    out, off = [], 0
    for n, bits, bucket in specs:
        out.append((off, n, bits, bucket))
        off += n
    return out, off


def rs_inputs(W, S, dtype, seed, source="randn", shard_layers=None, cases=CASES):
    """W inputs of W * S elements. Edge inputs: every shard gets its own hostile layer; a non-finite
    value sits on the shard's receiver ("edge_owner") or on the next rank ("edge_peer")."""
    if source == "randn":
        g = torch.Generator().manual_seed(seed)
        return [(torch.randn(W * S, generator=g) * (r + 1)).to(dtype) for r in range(W)]
    bucket = next((b for _, _, bits, b in shard_layers if bits < 32), 64)
    bits = next((bits for _, _, bits, _ in shard_layers if bits < 32), 4)
    ins = [torch.empty(W * S, dtype=dtype) for _ in range(W)]
    for c in range(W):
        xs, _ = edge_inputs(dtype, S, O.effective_bucket(bucket), seed + c, world=W, bits=bits, owners=[c] * S,
                            where="owner" if source == "edge_owner" else "peer", cases=cases)
        for r in range(W):
            ins[r][c * S:(c + 1) * S] = xs[r]
    return ins


def simulate(ins, shard_layers, *, average, skip_incomplete, stochastic=False, seed=0, seq=0):
    W = len(ins)
    outs = [torch.full((ins[0].numel() // W,), -7.25, dtype=ins[0].dtype) for _ in range(W)]
    C.reduce_scatter_simulate(ins, outs, shard_layers, LANES, average, skip_incomplete, stochastic, seed, seq,
                              MIN_LANE)
    return outs


@settings(max_examples=80, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case)
def test_simulator_matches_reference(c):
    shard_layers, S = shard_table(c["specs"])
    ins = rs_inputs(c["world"], S, c["dtype"], c["seed"], c["source"], shard_layers)
    kw = dict(average=c["average"], skip_incomplete=c["skip_incomplete"])
    sim = simulate(ins, shard_layers, **kw)
    ref = O.reduce_scatter_reference(ins, shard_layers, **kw)
    for r in range(c["world"]):
        assert_same(sim[r], ref[r], f"rank {r}")


def _grid():
    i = 0
    for world in range(1, 17):
        for dtype in DTYPES:
            bits = 1 + (i * 3) % 8
            bucket = (1, 7, 64, 100, 512, 1024, 8192)[i % 7]
            yield pytest.param(world, dtype, bits, bucket, i % 2 == 1, i % 3 == 0, i,
                               id=f"w{world}-{str(dtype)[6:]}-q{bits}-b{bucket}")
            i += 1


@pytest.mark.parametrize("world,dtype,bits,bucket,average,skip_incomplete,i", list(_grid()))
def test_simulator_matches_reference_on_edge_inputs(world, dtype, bits, bucket, average, skip_incomplete, i):
    # a raw head, the hostile layer (partial last bucket) and a raw tail, in every shard
    nq = min(max(40 * bucket, 3000), 3 * 8192) + bucket // 2
    shard_layers = [(0, 37, 32, 512), (37, nq, bits, bucket), (37 + nq, 301, 32, 512)]
    S = 37 + nq + 301
    ins = rs_inputs(world, S, dtype, 100 + i, "edge_owner" if i % 2 else "edge_peer", shard_layers)
    sim = simulate(ins, shard_layers, average=average, skip_incomplete=skip_incomplete)
    ref = O.reduce_scatter_reference(ins, shard_layers, average=average, skip_incomplete=skip_incomplete)
    for r in range(world):
        assert_same(sim[r], ref[r], f"rank {r}")


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case, st.booleans())
def test_results_within_one_round_bound(c, stochastic):
    shard_layers, S = shard_table(c["specs"])
    source = "randn" if c["source"] == "randn" else "edge_owner"
    ins = rs_inputs(c["world"], S, c["dtype"], c["seed"], source, shard_layers, cases=FINITE)
    kw = dict(average=c["average"], skip_incomplete=c["skip_incomplete"])
    if stochastic:
        out = simulate(ins, shard_layers, stochastic=True, seed=7, seq=3, **kw)
    else:
        out = O.reduce_scatter_reference(ins, shard_layers, **kw)
    for r, (exact, bound) in enumerate(O.reduce_scatter_exact_and_bound(ins, shard_layers, stochastic=stochastic,
                                                                         **kw)):
        got = out[r].double().numpy()
        ok = np.isfinite(exact) & np.isfinite(bound) & np.isfinite(got)
        bad = ok & ~(np.abs(got - exact) <= bound)
        assert not bad.any(), f"rank {r}: {int(bad.sum())} elements outside the one-round bound"


def test_stochastic_rounding_differs_from_deterministic_and_is_seeded():
    shard_layers = [(0, 4096, 2, 512)]
    ins = rs_inputs(4, 4096, torch.float32, 3)
    det = simulate(ins, shard_layers, average=True, skip_incomplete=False)
    a = simulate(ins, shard_layers, average=True, skip_incomplete=False, stochastic=True, seed=7, seq=1)
    b = simulate(ins, shard_layers, average=True, skip_incomplete=False, stochastic=True, seed=7, seq=1)
    assert_same(a[2], b[2])
    assert mismatch(a[2], det[2]), "stochastic rounding did not change the result"


def test_fp32_equals_the_allreduce_phase_b_sum():
    # rank r's reduce-scatter output is the unrequantized accumulator of the allreduce over the same
    # W shards: quantizing it once more gives the allreduce result on shard r
    W, S = 4, 3000
    shard_layers = [(0, 1000, 32, 512), (1000, 2000, 4, 128)]
    layers = [(c * S + o, n, b, k) for c in range(W) for (o, n, b, k) in shard_layers]
    ins = rs_inputs(W, S, torch.float32, 11)
    rs = simulate(ins, shard_layers, average=False, skip_incomplete=False)
    ar = O.sra_reference(ins, layers, lanes=1, min_lane_elems=S)  # one lane: chunk c == shard c
    for r in range(W):
        assert_same(O.quantize_dequantize_layers(rs[r], shard_layers), ar[0][r * S:(r + 1) * S], f"shard {r}")


# ---- the reference tells wrong semantics apart ----------------------------------------------
def _rs_variant(ins, shard_layers, r, *, quantize_own=False, reverse_peers=False, buffer_bucket_grid=False):
    W = len(ins)
    S = ins[0].numel() // W
    xs = [t.float().numpy()[r * S:(r + 1) * S] for t in ins]
    out = np.zeros(S, np.float32)

    def contrib(v, bits, bucket):
        if bits >= 32:
            return O.round_to_dtype(v, ins[0].dtype)
        shift = (r * S) % bucket if buffer_bucket_grid else 0  # buckets counted from the input start
        v = np.concatenate([np.repeat(v[:1], shift), v])
        return O._qdq_buckets(v, bits, bucket)[0][shift:]

    for off, m, bits, bucket in O.layer_segments(shard_layers, False):
        sl = slice(off, off + m)
        acc = contrib(xs[r][sl], bits, bucket) if quantize_own else xs[r][sl].copy()
        for q in (reversed(range(W)) if reverse_peers else range(W)):
            if q != r:
                acc = acc + contrib(xs[q][sl], bits, bucket)
        out[sl] = acc
    return torch.from_numpy(out).to(ins[0].dtype)


@pytest.mark.parametrize("perturbation", ["none", "quantize_own", "reverse_peers", "buffer_bucket_grid"])
def test_reference_detects_wrong_semantics(perturbation):
    W, S = 4, 7333
    shard_layers = [(0, 1000, 32, 512), (1000, 6000, 4, 512), (7000, 333, 3, 100)]
    ins = rs_inputs(W, S, torch.float32, 1)
    sim = simulate(ins, shard_layers, average=False, skip_incomplete=False)
    kw = {} if perturbation == "none" else {perturbation: True}
    for r in (1, 2):
        got = _rs_variant(ins, shard_layers, r, **kw)
        if perturbation == "none":
            assert_same(got, O.reduce_scatter_reference(ins, shard_layers)[r])
            assert_same(got, sim[r])
        else:
            assert mismatch(got, sim[r]), f"{perturbation} was not detected on rank {r}"


# ---- plan and window properties ------------------------------------------------------------
@settings(max_examples=60, deadline=None, derandomize=True)
@given(st.lists(layer, min_size=1, max_size=4), st.integers(1, 16), st.integers(1, 64),
       st.sampled_from([64, 256, 2048]), st.sampled_from(DTYPES), st.booleans())
def test_replicated_table_gives_chunk_c_equal_copy_c(specs, world, lanes, min_lane, dtype, skip_incomplete):
    shard_layers, S = shard_table(specs)
    layers = [(c * S + o, n, b, k) for c in range(world) for (o, n, b, k) in shard_layers]
    plan = C.build_plan(layers, world=world, lanes=lanes, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete,
                        min_lane_elems=min_lane)
    G, lf, blocks = plan["lanes"], plan["lane_first"], plan["blocks"]
    assert plan["chunk_elems"] == [S] * world
    for c in range(world):
        b0, b1 = lf[c * G], lf[(c + 1) * G]
        offs = blocks[b0:b1, 0]
        assert int(offs.min()) == c * S and int((blocks[b0:b1, 0] + blocks[b0:b1, 1]).max()) == (c + 1) * S
        assert int(blocks[b0:b1, 1].sum()) == S, f"chunk {c} is not copy {c}"


@settings(max_examples=60, deadline=None, derandomize=True)
@given(st.lists(layer, min_size=1, max_size=4), st.integers(1, 16), st.sampled_from(DTYPES), st.booleans(),
       st.sampled_from([4096, 16384, 65536, 1 << 20]))
def test_windows_cover_the_shard_on_bucket_boundaries_and_fit_the_slot(specs, world, dtype, skip_incomplete, slot):
    shard_layers, S = shard_table(specs)
    wins = C.reduce_scatter_windows(shard_layers, world, 4, DT_CODE[dtype], skip_incomplete, MIN_LANE, slot)
    pieces = [l for w in wins for l in w]
    # in order, without gaps or overlaps, every piece inside one layer with that layer's config
    end = 0
    for off, n, bits, bucket in pieces:
        assert off == end
        end += n
        src = next(l for l in shard_layers if l[0] <= off < l[0] + l[1])
        assert (bits, bucket) == (src[2], src[3]) and off + n <= src[0] + src[1]
        if bits < 32:  # cut at a bucket start of the layer (and of the clamped bucket)
            assert (off - src[0]) % bucket == 0 and (off - src[0]) % O.effective_bucket(bucket) == 0
    assert end == S
    for w in wins:
        layers = [(c * S + o, n, b, k) for c in range(world) for (o, n, b, k) in w]
        plan = C.build_plan(layers, world=world, lanes=4, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete,
                            min_lane_elems=MIN_LANE)
        assert plan["max_chunk_wire"] <= slot


def test_windows_do_not_change_the_result():
    # the simulator over each window (its plan only) reproduces the one-window result bit for bit
    W, dtype = 3, torch.float16
    shard_layers = [(0, 5000, 3, 100), (5000, 10_000, 2, 10_000), (15_000, 999, 32, 512), (15_999, 9000, 8, 512)]
    S = 24_999
    ins = rs_inputs(W, S, dtype, 5)
    whole = simulate(ins, shard_layers, average=True, skip_incomplete=True)
    wins = C.reduce_scatter_windows(shard_layers, W, 4, DT_CODE[dtype], True, MIN_LANE, 4096)
    assert len(wins) > 3
    for r in range(W):
        got = torch.full((S,), -7.25, dtype=dtype)
        for w in wins:
            lo, hi = w[0][0], w[-1][0] + w[-1][1]
            rel = [(o - lo, n, b, k) for o, n, b, k in w]
            part = [torch.cat([t[c * S + lo:c * S + hi] for c in range(W)]) for t in ins]
            got[lo:hi] = simulate(part, rel, average=True, skip_incomplete=True)[r]
        assert_same(got, whole[r], f"rank {r}")


def test_bad_shard_tables_are_rejected():
    with pytest.raises(ValueError, match="tile"):
        C.reduce_scatter_windows([(0, 100, 4, 64), (120, 10, 4, 64)], 2, 4, 0, False, MIN_LANE, 1 << 20)
    with pytest.raises(ValueError, match="tile"):
        C.reduce_scatter_windows([(5, 100, 4, 64)], 2, 4, 0, False, MIN_LANE, 1 << 20)
