"""The CPU simulators of the fused SRA and one-shot kernels against the independent
reference of the whole operation (torch_cgx_b200/ops/oracle.py), bit for bit and
NaN-aware, on random layer tables, every world size the harness accepts, all dtypes and
hostile inputs. Also: the reference stays within its own exact-sum bound, and perturbed
copies of the reference (wrong semantics) are told apart from the simulator."""
import numpy as np
import pytest
import torch
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.ops import fake_quantize, quantize

from _bitwise import assert_same, mismatch
from _edge_inputs import CASES, FINITE, edge_inputs

C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
LANES, MIN_LANE = 3, 64

layer = st.tuples(st.integers(1, 3000), st.sampled_from([1, 2, 3, 4, 5, 6, 7, 8, 32]),
                  st.sampled_from([1, 3, 7, 8, 16, 32, 64, 100, 256, 512, 1000, 1024]))
case = st.fixed_dictionaries({
    "specs": st.lists(layer, min_size=1, max_size=5),
    "first_off": st.sampled_from([0, 1, 5]),
    "world": st.integers(1, 16),
    "dtype": st.sampled_from(DTYPES),
    "average": st.booleans(),
    "skip_incomplete": st.booleans(),
    "source": st.sampled_from(["randn", "edge_owner", "edge_peer"]),
    "seed": st.integers(0, 2 ** 20),
})


def make_layers(specs, first_off=0):
    out, off = [], first_off
    for n, bits, bucket in specs:
        out.append((off, n, bits, bucket))
        off += n
    return out, off


def make_inputs(c, layers, total, *, finite_only=False):
    W, dtype = c["world"], c["dtype"]
    if c["source"] == "randn":
        g = torch.Generator().manual_seed(c["seed"])
        return [(torch.randn(total, generator=g) * (r + 1)).to(dtype) for r in range(W)]
    owners = O.block_owners(layers, total, W, LANES, dtype, c["skip_incomplete"], MIN_LANE)
    owners[owners < 0] = 0
    bucket = next((b for _, _, bits, b in layers if bits < 32), 64)
    bits = next((bits for _, _, bits, _ in layers if bits < 32), 4)
    ins, _ = edge_inputs(dtype, total, bucket, c["seed"], world=W, bits=bits, owners=owners,
                         where="owner" if c["source"] == "edge_owner" else "peer",
                         cases=FINITE if finite_only else CASES)
    return ins


@settings(max_examples=70, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case)
def test_simulators_match_reference(c):
    layers, total = make_layers(c["specs"], c["first_off"])
    ins = make_inputs(c, layers, total)
    kw = dict(average=c["average"], skip_incomplete=c["skip_incomplete"])
    sim = [t.clone() for t in ins]
    C.sra_simulate(sim, layers, LANES, c["average"], c["skip_incomplete"], False, 0, 0, MIN_LANE)
    ref = O.sra_reference(ins, layers, lanes=LANES, min_lane_elems=MIN_LANE, **kw)
    one = [t.clone() for t in ins]
    C.oneshot_simulate(one, layers, LANES, c["average"], c["skip_incomplete"], False, 0, 0, MIN_LANE)
    oref = O.oneshot_reference(ins, layers, **kw)
    for r in range(c["world"]):
        assert_same(sim[r], ref[r], f"sra_simulate rank {r}")
        assert_same(one[r], oref[r], f"oneshot_simulate rank {r}")


def _check_bound(out, exact, bound):
    got = out.double().numpy()
    ok = np.isfinite(exact) & np.isfinite(bound) & np.isfinite(got)
    err = np.abs(got - exact)
    bad = ok & ~(err <= bound)
    assert not bad.any(), f"{int(bad.sum())} elements outside the bound, first {int(np.argmax(bad))}: " \
                          f"err {err[bad][0]:.3e} > bound {bound[bad][0]:.3e}"


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(case, st.booleans())
def test_results_within_exact_sum_bound(c, stochastic):
    c = dict(c, source="randn" if c["source"] == "randn" else "edge_owner")
    layers, total = make_layers(c["specs"], c["first_off"])
    ins = make_inputs(c, layers, total, finite_only=True)
    kw = dict(lanes=LANES, min_lane_elems=MIN_LANE, average=c["average"], skip_incomplete=c["skip_incomplete"])
    exact, bound = O.exact_sum_and_bound(ins, layers, stochastic=stochastic, **kw)
    if stochastic:
        out = [t.clone() for t in ins]
        C.sra_simulate(out, layers, LANES, c["average"], c["skip_incomplete"], True, 7, 3, MIN_LANE)
    else:
        out = O.sra_reference(ins, layers, **kw)
    _check_bound(out[0], exact, bound)
    oexact, obound = O.exact_sum_and_bound(ins, layers, stochastic=stochastic, oneshot=True, **kw)
    oout = [t.clone() for t in ins]
    C.oneshot_simulate(oout, layers, LANES, c["average"], c["skip_incomplete"], stochastic, 7, 3, MIN_LANE)
    _check_bound(oout[0], oexact, obound)


# ---- the reference tells wrong semantics apart ----------------------------------------------
def _sra_variant(ins, layers, *, average=False, quantize_own=False, buffer_bucket_grid=False, reverse_peers=False):
    """A copy of sra_reference with one semantic change switched on (none: identical)."""
    W, dtype = len(ins), ins[0].dtype
    n = ins[0].numel()
    ps = np.float32(1.0) / np.float32(W) if average else np.float32(1.0)
    xs = [t.float().numpy() * ps for t in ins]
    owner = O.block_owners(layers, n, W, LANES, dtype, False, MIN_LANE)
    out = ins[0].float().numpy().copy()

    def contrib(v, off, bits, bucket):
        if bits >= 32:
            return O.round_to_dtype(v, dtype)
        shift = off % bucket if buffer_bucket_grid else 0
        v = np.concatenate([np.repeat(v[:1], shift), v])  # v[0] does not change its bucket's min/max
        return O._qdq_buckets(v, bits, bucket)[0][shift:]

    for off, m, bits, bucket in O.layer_segments(layers, False):
        sl = slice(off, off + m)
        own = owner[sl]
        acc = np.choose(own, [x[sl] for x in xs]).astype(np.float32)
        if quantize_own:
            acc = np.choose(own, [contrib(x[sl], off, bits, bucket) for x in xs]).astype(np.float32)
        for q in (reversed(range(W)) if reverse_peers else range(W)):
            acc = np.where(own != q, acc + contrib(xs[q][sl], off, bits, bucket), acc)
        out[sl] = contrib(acc, off, bits, bucket)
    return torch.from_numpy(out).to(dtype)


@pytest.mark.parametrize("perturbation", ["none", "quantize_own", "buffer_bucket_grid", "reverse_peers"])
def test_reference_detects_wrong_semantics(perturbation):
    # a layer whose start is not a multiple of its bucket; four ranks so that the peer order matters
    layers = [(0, 1000, 32, 512), (1000, 6000, 4, 512), (7000, 333, 3, 100)]
    W = 4
    g = torch.Generator().manual_seed(1)
    ins = [torch.randn(7333, generator=g) * (r + 1) for r in range(W)]
    sim = [t.clone() for t in ins]
    C.sra_simulate(sim, layers, LANES, True, False, False, 0, 0, MIN_LANE)
    kw = {} if perturbation == "none" else {perturbation: True}
    got = _sra_variant(ins, layers, average=True, **kw)
    if perturbation == "none":
        assert_same(got, O.sra_reference(ins, layers, lanes=LANES, min_lane_elems=MIN_LANE, average=True)[0])
        assert_same(got, sim[0])
    else:
        assert mismatch(got, sim[0]), f"{perturbation} was not detected"


# ---- pinned behaviour ---------------------------------------------------------------------------
def test_buckets_above_8192_are_clamped():
    # one block holds at most 8192 elements, so larger buckets quantize as 8192-element buckets
    assert C.MAX_BLOCK_ELEMS == O.MAX_BUCKET == 8192
    g = torch.Generator().manual_seed(0)
    x = torch.randn(30_000, generator=g)
    x[20_000] = 50.0  # an outlier that a true 20000-element bucket would spread over more elements
    for bucket in (8193, 10_000, 20_000):
        assert torch.equal(quantize(x, 4, bucket), quantize(x, 4, 8192))
        plan = C.build_plan([(0, x.numel(), 4, bucket)], world=1, lanes=1)
        assert set(plan["blocks"][:, 3].tolist()) == {8192}
    y = fake_quantize(x, 4, 20_000)
    assert_same(y, O.quantize_dequantize_like(x, 4, 8192))
    assert not torch.equal(y, O.quantize_dequantize_like(x, 4, 20_000))
    assert O.effective_bucket(20_000) == 8192
    # skip_incomplete counts the complete buckets with the requested size, before the clamp
    assert O.layer_segments([(0, 30_000, 4, 20_000)], True) == [(0, 20_000, 4, 8192), (20_000, 10_000, 32, 0)]
    ins = [x.clone(), x.flip(0).clone()]
    sim = [t.clone() for t in ins]
    C.sra_simulate(sim, [(0, 30_000, 4, 20_000)], 1, False, True, False, 0, 0, 2048)
    assert_same(sim[0], O.sra_reference(ins, [(0, 30_000, 4, 20_000)], skip_incomplete=True)[0])


@pytest.mark.parametrize("dtype", DTYPES)
def test_poisoned_bucket_meta_is_the_canonical_nan(dtype):
    # the GPU's min.NaN / max.NaN and fp32 arithmetic return 0x7FFFFFFF; the CPU bytes must match
    B = 64
    x = torch.randn(6 * B).to(dtype)
    x[3] = float("nan")
    x[B:2 * B] = float("inf")            # inf - inf
    x[2 * B + 5] = float("-inf")         # min = -inf, unit = inf
    x[3 * B:4 * B] = float("nan")
    meta = quantize(x, 4, B)[0, :6 * 8].view(torch.int32).view(6, 2)
    canon = 0x7FFFFFFF
    assert meta[0].tolist() == [canon, canon]
    assert meta[1].tolist() == [canon, int(np.float32(np.inf).view(np.int32))]
    assert meta[2, 0].item() == int(np.float32(np.inf).view(np.int32))
    assert meta[3].tolist() == [canon, canon]
    assert np.isfinite(meta[4:].numpy().view(np.float32)).all()
    # raw records carry the prescaled value: a NaN there is canonical as well
    w = C.quantize(x, [(0, x.numel(), 32, 512)], 1, 1, False, 0.5, False, 0, 0, 0, 0, 2048)
    nan_bits = {torch.float32: canon, torch.float16: 0x7FFF, torch.bfloat16: 0x7FFF}[dtype]
    raw = w[0, :x.numel() * x.element_size()].view(torch.int32 if dtype == torch.float32 else torch.int16)
    assert int(raw[3]) & (0xFFFFFFFF if dtype == torch.float32 else 0xFFFF) == nan_bits


@pytest.mark.parametrize("dtype", DTYPES)
def test_quantize_dequantize_follows_ieee_on_non_finite(dtype):
    x = torch.randn(64).to(dtype)
    x[10] = float("inf")
    dec, q = O.quantize_dequantize(x, 4, 64)
    # unit = inf, 1/unit = 0: finite elements get t = 0.5 -> level 0 -> inf * 0 + min = NaN;
    # the inf element gets t = inf * 0 = NaN -> top level -> inf * 15 + min = +inf
    assert dec[10].item() == float("inf") and q[10].item() == 15
    assert torch.isnan(torch.cat([dec[:10], dec[11:]])).all()
    assert_same(fake_quantize(x, 4, 64), dec.to(dtype))


def test_fma32_rounds_once():
    # a*b + c lies just below the midpoint 1 + 3*2^-24 of two fp32 values, closer than half an
    # fp64 ulp: rounding through fp64 lands on the midpoint and then rounds up (to even)
    a = torch.tensor([2.0 ** -24 * (1 + 2.0 ** -15)], dtype=torch.float32)
    b = torch.tensor([1 - 2.0 ** -15], dtype=torch.float32)
    c = torch.tensor([1 + 2.0 ** -23], dtype=torch.float32)
    assert (a.double() * b.double() + c.double()).float().item() == 1 + 2.0 ** -22  # double rounding
    assert O._fma32(a, b, c).item() == 1 + 2.0 ** -23


@pytest.mark.parametrize("dtype", DTYPES)
def test_edge_generator_plants_what_it_says(dtype):
    ins, planted = edge_inputs(dtype, 64 * 64, 64, 3, world=3, bits=4)
    cases = {p.case for p in planted}
    assert {"nan", "pinf", "ninf", "both_inf", "all_pinf", "all_nan", "pzero", "nzero", "tiny"} <= cases
    assert {f"outlier@{p}" for p in (0, 7, 8, 15, 16, 63)} <= cases
    for p in planted:
        seg = [t[p.lo:p.hi].float() for t in ins]
        if p.nonfinite:
            assert not torch.isfinite(seg[p.rank]).all()
            assert all(torch.isfinite(s).all() for r, s in enumerate(seg) if r != p.rank)
        else:
            assert all(torch.isfinite(s).all() for s in seg), p.case
        if p.case in ("eps_below", "eps_above"):
            v = seg[0].numpy()
            unit = (v.max() - v.min()) * (np.float32(1) / np.float32(15))
            assert (unit < np.float32(1e-10)) == (p.case == "eps_below")
        if p.case == "nzero":
            assert all(torch.signbit(s).all() for s in seg)
