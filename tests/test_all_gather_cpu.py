"""The CPU simulator of the compressed all-gather (C.all_gather_simulate, the arithmetic of ag_kernel)
against the independent NumPy reference (ops/oracle.py all_gather_reference), bit for bit and
NaN-aware; the fp32 identity allreduce == all_gather(reduce_scatter); and the FSDP2 shard table."""
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
LANES, MIN_LANE = 3, 64

layer = st.tuples(st.integers(1, 2000), st.sampled_from([1, 2, 3, 4, 5, 6, 7, 8, 32]),
                  st.sampled_from([1, 3, 7, 8, 16, 32, 64, 100, 256, 512, 1000, 1024, 10_000]))
case = st.fixed_dictionaries({
    "specs": st.lists(layer, min_size=1, max_size=4),
    "world": st.integers(1, 16),
    "dtype": st.sampled_from(DTYPES),
    "source": st.sampled_from(["randn", "edge_owner", "edge_peer"]),
    "seed": st.integers(0, 2 ** 20),
})


def shard_table(specs):
    out, off = [], 0
    for n, bits, bucket in specs:
        out.append((off, n, bits, bucket))
        off += n
    return out, off


def ag_inputs(W, S, dtype, seed, source="randn", shard_layers=None, cases=CASES):
    """W shards of S elements. Edge inputs: hostile buckets in every shard, a non-finite value on
    rank seed % W ("edge_owner") or on the ranks other than it ("edge_peer")."""
    if source == "randn":
        g = torch.Generator().manual_seed(seed)
        return [(torch.randn(S, generator=g) * (r + 1)).to(dtype) for r in range(W)]
    bucket = next((b for _, _, bits, b in shard_layers if bits < 32), 64)
    bits = next((bits for _, _, bits, _ in shard_layers if bits < 32), 4)
    xs, _ = edge_inputs(dtype, S, O.effective_bucket(bucket), seed, world=W, bits=bits, owners=[seed % W] * S,
                        where="owner" if source == "edge_owner" else "peer", cases=cases)
    return list(xs)


def simulate(ins, shard_layers, *, stochastic=False, seed=0, seq=0):
    W = len(ins)
    outs = [torch.full((W * ins[0].numel(),), -7.25, dtype=ins[0].dtype) for _ in range(W)]
    C.all_gather_simulate(ins, outs, shard_layers, stochastic, seed, seq)
    return outs


def check_all_ranks(sim, ref):
    for r, s in enumerate(sim):
        assert_same(s, ref, f"rank {r}")


@settings(max_examples=80, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case)
def test_simulator_matches_reference(c):
    shard_layers, S = shard_table(c["specs"])
    ins = ag_inputs(c["world"], S, c["dtype"], c["seed"], c["source"], shard_layers)
    check_all_ranks(simulate(ins, shard_layers), O.all_gather_reference(ins, shard_layers))


def _grid():
    i = 0
    for world in range(1, 17):
        for dtype in DTYPES:
            for bits in (1 + (i * 3) % 8, 1 + (i * 3 + 4) % 8):
                bucket = (1, 7, 64, 100, 512, 1024, 8192, 10_000)[i % 8]
                yield pytest.param(world, dtype, bits, bucket, i, id=f"w{world}-{str(dtype)[6:]}-q{bits}-b{bucket}")
                i += 1


@pytest.mark.parametrize("world,dtype,bits,bucket,i", list(_grid()))
def test_simulator_matches_reference_on_edge_inputs(world, dtype, bits, bucket, i):
    # a raw head, the hostile layer (partial last bucket) and a raw tail, in every shard
    nq = min(max(40 * bucket, 3000), 3 * 8192) + bucket // 2
    shard_layers = [(0, 37, 32, 512), (37, nq, bits, bucket), (37 + nq, 301, 32, 512)]
    S = 37 + nq + 301
    ins = ag_inputs(world, S, dtype, 100 + i, "edge_owner" if i % 2 else "edge_peer", shard_layers)
    check_all_ranks(simulate(ins, shard_layers), O.all_gather_reference(ins, shard_layers))


def test_world1_is_the_round_trip_and_buckets_above_8192_are_clamped():
    x = torch.randn(3 * 8192 + 5) * 3
    x[100] = 40.0  # an outlier in the first 8192 elements only
    out = simulate([x], [(0, x.numel(), 3, 20_000)])[0]
    assert_same(out, O.quantize_dequantize_layers(x, [(0, x.numel(), 3, 20_000)]))
    assert_same(out, O.quantize_dequantize_layers(x, [(0, x.numel(), 3, 8192)]))
    assert mismatch(out, O.quantize_dequantize(x, 3, x.numel())[0])  # one unclamped bucket


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case)
def test_stochastic_results_within_one_round_bound(c):
    shard_layers, S = shard_table(c["specs"])
    source = "randn" if c["source"] == "randn" else "edge_owner"
    ins = ag_inputs(c["world"], S, c["dtype"], c["seed"], source, shard_layers, cases=FINITE)
    out = simulate(ins, shard_layers, stochastic=True, seed=7, seq=3)[0]
    for q, x in enumerate(ins):
        exact, bound = O.exact_sum_and_bound([x], shard_layers, stochastic=True, oneshot=True)
        # a bucket whose unit is below 1e-10 decodes to its min: the bound takes its span as
        # unit * levels, which misses the rounding of a subnormal unit (at most levels * 2^-150)
        bound = bound + 255 * 2.0 ** -150
        got = out[q * S:(q + 1) * S].double().numpy()
        ok = np.isfinite(exact) & np.isfinite(bound) & np.isfinite(got)
        bad = ok & ~(np.abs(got - exact) <= bound)
        assert not bad.any(), f"shard {q}: {int(bad.sum())} elements outside the one-round bound"


def test_stochastic_rounding_differs_from_deterministic_and_is_seeded():
    shard_layers = [(0, 4096, 2, 512)]
    ins = ag_inputs(4, 4096, torch.float32, 3)
    det = simulate(ins, shard_layers)
    a = simulate(ins, shard_layers, stochastic=True, seed=7, seq=1)
    b = simulate(ins, shard_layers, stochastic=True, seed=7, seq=1)
    c = simulate(ins, shard_layers, stochastic=True, seed=7, seq=2)
    assert_same(a[2], b[2])
    assert_same(a[0], a[3])
    assert mismatch(a[2], det[2]), "stochastic rounding did not change the result"
    assert mismatch(a[2], c[2]), "the sequence number did not change the random stream"


# ---- the reference tells wrong semantics apart ----------------------------------------------
def _ag_variant(ins, shard_layers, r, *, owner_exact=False, buffer_bucket_grid=False):
    """Rank r's output under a wrong semantics: its own shard kept unquantized, or buckets counted
    from the start of the gathered buffer instead of each shard's start."""
    W, S = len(ins), ins[0].numel()
    parts = []
    for q, x in enumerate(ins):
        if owner_exact and q == r:
            parts.append(x.clone())
            continue
        v = x.float().numpy()
        out = np.zeros(S, np.float32)
        for off, m, bits, bucket in O.layer_segments(shard_layers, False):
            seg = v[off:off + m]
            if bits >= 32:
                out[off:off + m] = O.round_to_dtype(seg, x.dtype)
                continue
            shift = (q * S) % bucket if buffer_bucket_grid else 0
            out[off:off + m] = O._qdq_buckets(np.concatenate([np.repeat(seg[:1], shift), seg]), bits, bucket)[0][shift:]
        parts.append(torch.from_numpy(out).to(x.dtype))
    return torch.cat(parts)


@pytest.mark.parametrize("perturbation", ["none", "owner_exact", "buffer_bucket_grid"])
def test_reference_detects_wrong_semantics(perturbation):
    W, S = 4, 7333
    shard_layers = [(0, 1000, 32, 512), (1000, 6000, 4, 512), (7000, 333, 3, 100)]
    ins = ag_inputs(W, S, torch.float32, 1)
    sim = simulate(ins, shard_layers)
    kw = {} if perturbation == "none" else {perturbation: True}
    for r in (1, 2):
        got = _ag_variant(ins, shard_layers, r, **kw)
        if perturbation == "none":
            assert_same(got, O.all_gather_reference(ins, shard_layers))
            assert_same(got, sim[r])
        else:
            assert mismatch(got, sim[r]), f"{perturbation} was not detected on rank {r}"


# ---- allreduce == all_gather(reduce_scatter) for fp32 ----------------------------------------
@pytest.mark.parametrize("average", [False, True])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 7])
def test_fp32_allreduce_is_all_gather_of_reduce_scatter(W, average):
    # the reduce-scatter output is the allreduce's phase-B accumulator of chunk r; the SRA's
    # publish requantizes exactly that accumulator with the same buckets, as the all-gather does
    S = 9133
    shard_layers = [(0, 700, 32, 512), (700, 4000, 4, 256), (4700, 4000, 2, 512), (8700, 433, 6, 100)]
    layers = [(c * S + o, n, b, k) for c in range(W) for (o, n, b, k) in shard_layers]
    g = torch.Generator().manual_seed(W)
    ins = [torch.randn(W * S, generator=g) * (r + 1) for r in range(W)]
    rs = [torch.empty(S) for _ in range(W)]
    C.reduce_scatter_simulate(ins, rs, shard_layers, LANES, average, False, False, 0, 0, MIN_LANE)
    ag = simulate(rs, shard_layers)
    ar = [t.clone() for t in ins]
    C.sra_simulate(ar, layers, LANES, average, False, False, 0, 0, MIN_LANE)
    for r in range(W):
        assert_same(ag[r], ar[r], f"rank {r}")


# ---- FSDP2 shard table -----------------------------------------------------------------------
def test_fsdp_shard_table_is_per_parameter_with_raw_vectors():
    # an MLP block with a LayerNorm, sharded over W = 4: FSDP pads dim 0 to a multiple of W
    params = [((512, 256), 128 * 256), ((512,), 128), ((256,), 64), ((256,), 64), ((10, 512), 3 * 512),
              ((10,), 3)]
    assert cgx.fsdp_shard_table(params, bits=8, bucket_size=256) == [
        (0, 32768, 8, 256), (32768, 128, 32, 256), (32896, 64, 32, 256), (32960, 64, 32, 256),
        (33024, 1536, 8, 256), (34560, 3, 32, 256)]
    # empty shards (a parameter smaller than the world) contribute nothing; scalars are raw
    assert cgx.fsdp_shard_table([((3, 3), 0), ((), 1), ((4, 4, 4), 16)], bits=4) == [
        (0, 1, 32, 512), (1, 16, 4, 512)]
    assert cgx.fsdp_shard_table([]) == []


def test_fsdp_shard_table_tiles_the_shard_for_the_windows():
    params = [((1000, 37), 250 * 37), ((1000,), 250), ((7, 3, 3, 3), 2 * 27)]
    table = cgx.fsdp_shard_table(params, bits=4, bucket_size=512)
    S = sum(n for _, n in params)
    wins = C.reduce_scatter_windows(table, 4, 4, 0, False, MIN_LANE, 4096)
    assert sum(l[1] for w in wins for l in w) == S
