"""Adaptive per-layer widths without a GPU: the CPU quantization-error estimator against the
quantize -> dequantize round trip, the bit allocator against brute force, and AdaptiveCGXState in a
two-rank DDP run on CPU tensors (CGX_COMPRESS_CPU=1)."""
import itertools
import math

import numpy as np
import pytest
import torch
import torch.distributed as dist

from _dist_utils import spawn
from _edge_inputs import edge_inputs

CANDS = (1, 2, 3, 4, 5, 6, 7, 8)


def _ref(t, layers, cands, prescale=1.0, skip=False):
    """fp64 sum of (round trip - x')^2 per layer, from the CPU quantize / dequantize ops."""
    from torch_cgx_b200.ops import fake_quantize

    xf = t.float() * prescale  # the fp32 values the encoder sees
    out = np.zeros((len(layers), len(cands)))
    for l, (off, n, _, b) in enumerate(layers):
        x = xf[off:off + n].contiguous()
        for k, bits in enumerate(cands):
            rt = fake_quantize(x, bits, min(b, 8192), skip_incomplete=skip)
            out[l, k] = ((rt.double() - x.double()) ** 2).sum().item()
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("skip", [False, True], ids=["tail", "skip_incomplete"])
def test_estimator_matches_round_trip(dtype, skip):
    from torch_cgx_b200.ops import quantization_error

    g = torch.Generator().manual_seed(1)
    layers, off = [], 3  # offsets not multiples of 8
    for b in (8, 13, 64, 100, 512, 1000, 8192, 20000):  # 20000 is clamped to 8192
        for n in (5, 777, 9001):
            layers.append((off, n, 4, b))
            off += n + 3
    t = (torch.randn(off, generator=g) * 3).to(dtype)
    got = quantization_error(t, layers, CANDS, prescale=0.375, skip_incomplete=skip).numpy()
    np.testing.assert_allclose(got, _ref(t, layers, CANDS, 0.375, skip), rtol=1e-5, atol=0)


def test_estimator_constant_buckets_and_shape():
    from torch_cgx_b200.ops import quantization_error

    t = torch.full((1000,), 0.3)
    t[500:] = -2.0
    e = quantization_error(t, [(0, 500, 4, 100), (500, 500, 4, 64), (0, 0, 4, 8)], (2, 4))
    assert e.dtype == torch.float64 and e.shape == (3, 2)
    assert torch.equal(e, torch.zeros(3, 2))


def test_estimator_non_finite_rows():
    from torch_cgx_b200.ops import quantization_error

    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        (x,), planted = edge_inputs(dtype, 64 * 256, 256, seed=2)
        row = quantization_error(x, [(p.lo, p.hi - p.lo, 4, 256) for p in planted], CANDS)
        for p, r in zip(planted, row):
            if p.nonfinite:
                assert not torch.isfinite(r).any(), p
            elif p.case not in ("span_overflow", "wide_range"):
                # span_overflow: max - min overflows and the wire decodes NaN as well; wide_range: a
                # finite error whose square can overflow fp32
                assert torch.isfinite(r).all(), p


def test_estimator_stochastic_closed_form_and_sampling():
    from torch_cgx_b200.ops import fake_quantize, quantization_error

    g = torch.Generator().manual_seed(4)
    x = torch.randn(4096, generator=g)
    B, bits = 512, 3
    got = quantization_error(x, [(0, 4096, bits, B)], (bits,), stochastic=True)[0, 0].item()
    # closed form in fp64
    xb = x.double().view(-1, B)
    mn, mx = x.view(-1, B).min(1).values, x.view(-1, B).max(1).values
    unit = ((mx - mn) * np.float32(1 / 7)).double()
    f = (xb - mn.double()[:, None]) / unit[:, None]
    f = f - f.floor()
    closed = ((unit ** 2)[:, None] * f * (1 - f)).sum().item()
    assert got == pytest.approx(closed, rel=1e-4)
    # 64 seeded stochastic round trips: the sample mean of the squared error has a standard error
    # of sd / 8; 6 standard errors plus 1e-3 relative for the closed form's fp32 inputs
    samples = [((fake_quantize(x, bits, B, stochastic=True, seed=s).double() - x.double()) ** 2).sum().item()
               for s in range(64)]
    mean, sd = float(np.mean(samples)), float(np.std(samples, ddof=1))
    assert abs(mean - got) <= 6 * sd / 8 + 1e-3 * got, (mean, got, sd)


def test_estimator_rejects_bad_input():
    from torch_cgx_b200 import _C

    t = torch.randn(100)
    for bad in (lambda: _C.quantization_error(t[::2], [(0, 10, 4, 8)], [4]),
                lambda: _C.quantization_error(t.double(), [(0, 10, 4, 8)], [4]),
                lambda: _C.quantization_error(t, [(95, 10, 4, 8)], [4]),
                lambda: _C.quantization_error(t, [(-1, 10, 4, 8)], [4]),
                lambda: _C.quantization_error(t, [(0, 10, 4, 0)], [4]),
                lambda: _C.quantization_error(t, [(0, 10, 4, 8)], [9]),
                lambda: _C.quantization_error(t, [(0, 10, 4, 8)], [0]),
                lambda: _C.quantization_error(t, [(0, 10, 4, 8)], [])):
        with pytest.raises(RuntimeError):
            bad()


# ---- allocator --------------------------------------------------------------------------------
def _cost(numels, buckets, cands):
    from torch_cgx_b200.ops import wire_bytes

    return np.array([[wire_bytes(n, c, b) for c in cands] for n, b in zip(numels, buckets)])


def test_allocator_equals_brute_force():
    from torch_cgx_b200.ops import allocate_bits

    rng = np.random.default_rng(0)
    for _ in range(60):
        L, K = rng.integers(1, 5), rng.integers(1, 5)
        cands = sorted(rng.choice(np.arange(1, 9), K, replace=False).tolist())
        numels = rng.integers(8, 3000, L).tolist()
        buckets = rng.choice([8, 64, 512], L).tolist()
        cost = _cost(numels, buckets, cands)
        err = rng.random((L, K)) * 10.0 ** rng.integers(-3, 3, (L, 1))
        target = cands[rng.integers(K)]
        budget = int(cost[:, cands.index(target)].sum() * rng.uniform(0.8, 1.3))
        got = allocate_bits(err, numels, buckets, cands, budget, resolution=budget, target_bits=target)
        best = None
        for pick in itertools.product(range(K), repeat=L):
            if sum(cost[l, k] for l, k in enumerate(pick)) <= budget:
                e = sum(err[l, k] for l, k in enumerate(pick))
                best = e if best is None else min(best, e)
        idx = [cands.index(b) for b in got]
        got_e = sum(err[l, k] for l, k in enumerate(idx))
        if best is None:  # nothing fits: the uniform target assignment comes back
            assert got == [target] * L
        else:
            assert sum(cost[l, k] for l, k in enumerate(idx)) <= budget
            assert got_e == pytest.approx(best, rel=1e-12)


def test_allocator_large_instances_within_budget_and_better_than_uniform():
    from torch_cgx_b200.ops import allocate_bits

    rng = np.random.default_rng(1)
    cands = (2, 3, 4, 5, 6, 7, 8)
    for _ in range(10):
        L = 150
        numels = rng.integers(1000, 2_000_000, L).tolist()
        buckets = [512] * L
        cost = _cost(numels, buckets, cands)
        scale = 10.0 ** rng.uniform(-6, 0, (L, 1))
        err = scale * np.array(numels)[:, None] * 4.0 ** -np.array(cands)[None, :]
        budget = int(cost[:, 2].sum())
        got = allocate_bits(err, numels, buckets, cands, budget)
        idx = [cands.index(b) for b in got]
        assert sum(cost[l, k] for l, k in enumerate(idx)) <= budget
        assert sum(err[l, k] for l, k in enumerate(idx)) <= err[:, 2].sum()
        assert len(set(got)) > 1


def test_allocator_ties_single_candidate_and_non_finite_rows():
    from torch_cgx_b200.ops import allocate_bits

    numels, buckets = [4096, 4096, 4096], [512] * 3
    zeros = np.zeros((3, 3))
    budget = int(_cost(numels, buckets, (2, 4, 8))[:, 1].sum())
    a = allocate_bits(zeros, numels, buckets, (2, 4, 8), budget)
    assert a == [2, 2, 2]  # equal error: fewest bytes
    assert allocate_bits(zeros, numels, buckets, (2, 4, 8), budget) == a
    assert allocate_bits(np.ones((3, 1)), numels, buckets, (5,), budget) == [5, 5, 5]
    err = np.array([[9.0, 3.0, 1.0], [np.nan, 1.0, 1.0], [np.inf, 0.0, 0.0]])
    got = allocate_bits(err, numels, buckets, (2, 4, 8), budget, current=[4, 6, 3])
    assert got[1:] == [6, 3]
    got = allocate_bits(err, numels, buckets, (2, 4, 8), budget)
    assert got[1:] == [4, 4]


def test_allocator_cost_is_the_plans_record_size():
    """The allocator's cost of a layer is the meta + payload of the plan's blocks for it; the plan
    adds only the 16-byte alignment of each block record's two sections."""
    from torch_cgx_b200 import _C
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes

    for n, bits, b in itertools.product((1, 9, 5000, 70001, 300000), (1, 2, 3, 4, 5, 8), (8, 13, 512, 1024, 20000)):
        plan = _C.build_plan([(0, n, bits, b)], 1, 1, 0, False, 1 << 30)
        blocks = plan["blocks"].tolist()
        records = sum(-(-bn // bb) * 8 + (bn // bb * -(-bb // 8) + -(-(bn % bb) // 8)) * bb_bits
                      for (_, bn, bb_bits, bb, _) in blocks)
        assert layer_wire_bytes(n, bits, b) == records
        assert records <= plan["total_wire"] < records + 32 * len(blocks)


# ---- two-rank DDP on CPU tensors ----------------------------------------------------------------
class _Net(torch.nn.Module):
    """Layers whose gradients differ in scale by orders of magnitude."""

    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(64, 256)
        self.b = torch.nn.Linear(256, 64)
        self.c = torch.nn.Linear(64, 10)

    def forward(self, x):
        h = torch.relu(self.a(x)) * 0.001
        h = torch.relu(self.b(h)) * 100.0
        return self.c(h)


def _train(rank, world, state, steps=8, register_native=False):
    import torch_cgx_b200 as cgx
    from torch.nn.parallel import DistributedDataParallel as DDP

    cgx.reset_layers()
    torch.manual_seed(0)
    ddp = DDP(_Net())
    if register_native:
        assert cgx.register_cgx_hook(ddp, state) is None
    else:
        ddp.register_comm_hook(state, cgx.cgx_hook)
    opt = torch.optim.SGD(ddp.parameters(), lr=0.002)
    widths = []
    for step in range(steps):
        g = torch.Generator().manual_seed(100 + step * world + rank)  # different data per rank
        x, y = torch.randn(16, 64, generator=g), torch.randint(0, 10, (16,), generator=g)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ddp(x), y).backward()
        opt.step()
        widths.append([tuple(r) for r in cgx._C.registered_bucket(0)] if cgx._C.num_registered_buckets() else [])
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    return flat, widths


def _adaptive_world2(rank, world):
    import torch_cgx_b200 as cgx
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes

    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        params = {"bits": 4, "bucket_size": 64}
        st = cgx.AdaptiveCGXState(None, 16, params, period=3)
        flat, widths = _train(rank, world, st)
        # registered at step 2 (uniform), decisions apply at steps 3 and 6
        assert st.assignment and len(set(st.assignment.values())) > 1, st.assignment
        changed = [s for s in range(1, len(widths)) if widths[s] != widths[s - 1]]
        assert set(changed) <= {2, 3, 6}, changed
        table = cgx._C.registered_bucket(0)
        for (b, l), bits in st.assignment.items():
            assert b == 0 and table[l][1] == bits
        used = sum(layer_wire_bytes(n, table[l][1], 64) for (_, l, _, n) in st.adapted_layers)
        assert used <= sum(layer_wire_bytes(n, 4, 64) for (_, _, _, n) in st.adapted_layers)
        both = [torch.zeros(len(table), 3, dtype=torch.int64) for _ in range(world)]
        dist.all_gather(both, torch.tensor(table, dtype=torch.int64))
        assert torch.equal(both[0], both[1])
        gathered = [torch.zeros_like(flat) for _ in range(world)]
        dist.all_gather(gathered, flat)
        assert torch.equal(gathered[0], gathered[1])  # replicas bit-identical

        # one candidate: the plain CGXState trajectory, bit for bit
        one, _ = _train(rank, world, cgx.AdaptiveCGXState(None, 16, params, candidate_bits=(4,), period=2))
        plain, _ = _train(rank, world, cgx.CGXState(None, 16, params))
        assert torch.equal(one, plain)

        # checkpoint: a fresh state loaded from state_dict re-applies the assignment at registration
        sd = st.state_dict()
        st2 = cgx.AdaptiveCGXState(None, 16, params, period=1000)
        st2.load_state_dict(sd)
        _, w2 = _train(rank, world, st2, steps=3)
        assert st2.assignment == sd["assignment"]
        assert {l: b for (_, l), b in sd["assignment"].items()}.items() <= {l: r[1] for l, r in enumerate(w2[2])}.items()

        # register_cgx_hook installs the Python hook for the adaptive state
        a, _ = _train(rank, world, cgx.AdaptiveCGXState(None, 16, params, period=3), register_native=True)
        assert torch.equal(a, flat)
    finally:
        dist.destroy_process_group()


def test_adaptive_state_world2_cpu():
    spawn(_adaptive_world2, 2, env={"CGX_COMPRESS_CPU": "1"})


def test_adaptive_state_rejects_bad_arguments():
    import torch_cgx_b200 as cgx

    with pytest.raises(ValueError):
        cgx.AdaptiveCGXState(object(), candidate_bits=(4, 9))
    with pytest.raises(ValueError):
        cgx.AdaptiveCGXState(object(), period=0)
    assert math.isfinite(cgx.ops.quantization_error(torch.ones(8), [(0, 8, 4, 8)])[0, 0].item())
