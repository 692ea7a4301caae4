"""Adaptive widths in C++ without a GPU: the C++ bit allocator against its NumPy reference on
thousands of seeded instances, and the adaptive native DDP hook against the Python hook in a
two-rank run on CPU tensors (CGX_COMPRESS_CPU=1)."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from _dist_utils import spawn
from test_adaptive_bits_cpu import _Net


# ---- allocator ----------------------------------------------------------------------------------
def _instance(rng, L, K, resolution):
    """One allocator input with the awkward cases mixed in: ties, non-finite rows, clamped buckets."""
    from torch_cgx_b200.ops.oracle import _layer_wire_bytes

    cands = rng.choice(np.arange(1, 9), K, replace=bool(rng.random() < 0.2)).tolist()
    if rng.random() < 0.5:
        cands = sorted(cands)
    numels = rng.integers(0, 50_000, L) if rng.random() < 0.8 else rng.integers(0, 20, L)
    numels = numels.tolist()
    buckets = rng.choice([1, 3, 8, 13, 64, 512, 1024, 8192, 8193, 20000, 100_000], L).tolist()
    kind = rng.integers(0, 5)
    if kind == 0:    # continuous
        err = rng.random((L, K)) * 10.0 ** rng.integers(-6, 6, (L, 1))
    elif kind == 1:  # integer valued: many equal sums
        err = rng.integers(0, 4, (L, K)).astype(np.float64)
    elif kind == 2:  # all equal
        err = np.full((L, K), float(rng.integers(0, 3)))
    elif kind == 3:  # duplicated rows
        base = rng.random((max(1, L // 3), K))
        err = base[rng.integers(0, len(base), L)] if L else np.zeros((0, K))
    else:            # error falling with width, like real tables
        c = np.array(cands, dtype=np.float64)
        err = (np.array(numels, dtype=np.float64)[:, None] + 1) * 4.0 ** -c[None, :] * rng.uniform(0.1, 10, (L, 1))
    err = err.reshape(L, K)
    if L and rng.random() < 0.3:  # non-finite rows
        for l in rng.choice(L, rng.integers(1, min(L, 4) + 1), replace=False):
            err[l, rng.integers(K)] = rng.choice([np.nan, np.inf, -np.inf])
    current = None
    if rng.random() < 0.5:
        current = rng.choice([1, 2, 3, 4, 5, 6, 7, 8, 32], L).tolist()
    target = None
    r = rng.random()
    if r < 0.5:
        target = int(rng.choice(cands))
    elif r < 0.6:
        target = int(rng.integers(1, 9))  # possibly not a candidate
    ref_bits = target if target is not None else int(rng.choice(cands))
    uniform = sum(_layer_wire_bytes(n, ref_bits, b) for n, b in zip(numels, buckets))
    budget = int(uniform * rng.choice([0.0, 0.3, 0.9, 1.0, 1.0, 1.05, 1.5, 3.0])) + int(rng.choice([-1, 0, 0, 1]))
    return err, numels, buckets, cands, budget, current, resolution, target


def _check_instances(seed, count, max_l, resolutions):
    from torch_cgx_b200.ops import allocate_bits
    from torch_cgx_b200.ops.oracle import allocate_bits_reference

    rng = np.random.default_rng(seed)
    for i in range(count):
        L = int(rng.integers(0, max_l + 1))
        K = int(rng.integers(1, 9))
        err, numels, buckets, cands, budget, current, res, target = _instance(rng, L, K, int(rng.choice(resolutions)))
        want = allocate_bits_reference(err, numels, buckets, cands, budget, current, res, target_bits=target)
        got = allocate_bits(err, numels, buckets, cands, budget, current, res, target_bits=target)
        assert got == want, (seed, i, L, K, res, budget, target)


def test_allocator_matches_reference_small():
    _check_instances(seed=10, count=3000, max_l=12, resolutions=[1, 2, 3, 5, 16, 64, 257])


def test_allocator_matches_reference_medium():
    _check_instances(seed=11, count=400, max_l=60, resolutions=[1, 7, 100, 1000, 4096])


def test_allocator_matches_reference_large():
    _check_instances(seed=12, count=60, max_l=300, resolutions=[4096])


def test_allocator_edge_instances():
    """Exact boundaries: L = 0, budgets at the uniform cost, a tie at the uniform fallback."""
    from torch_cgx_b200.ops import allocate_bits
    from torch_cgx_b200.ops.oracle import _layer_wire_bytes, allocate_bits_reference

    cases = []
    for L in (0, 1, 2, 8, 9, 128, 129, 300):
        for cands in ((4,), (2, 4, 8), (8, 4, 2), (4, 4, 2), (1, 2, 3, 4, 5, 6, 7, 8)):
            numels, buckets = [4096 + 8 * l for l in range(L)], [512 if l % 2 else 9000 for l in range(L)]
            uniform = sum(_layer_wire_bytes(n, 4, b) for n, b in zip(numels, buckets))
            for budget in (uniform - 1, uniform, uniform + 1):
                for err in (np.zeros((L, len(cands))), np.ones((L, len(cands))) * 0.1,
                            np.tile(np.linspace(1, 0, len(cands)), (L, 1))):
                    for res in (1, 4096):
                        cases.append((err, numels, buckets, cands, budget, None, res, 4))
                        cases.append((err, numels, buckets, cands, budget, [4] * L, res, None))
    for err, numels, buckets, cands, budget, current, res, target in cases:
        want = allocate_bits_reference(err, numels, buckets, cands, budget, current, res, target_bits=target)
        assert allocate_bits(err, numels, buckets, cands, budget, current, res, target_bits=target) == want


def test_allocator_arguments():
    from torch_cgx_b200.ops import allocate_bits
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes
    from torch_cgx_b200.ops.oracle import _layer_wire_bytes

    with pytest.raises(ValueError):
        allocate_bits(np.zeros((2, 2)), [8, 8], [8, 8], (2, 4, 8), 100)
    with pytest.raises(ValueError):
        allocate_bits(np.zeros((2, 0)), [8, 8], [8, 8], (), 100)
    with pytest.raises(ValueError):
        allocate_bits(np.zeros((2, 1)), [8, 8], [8, 8], (4,), 100, resolution=0)
    assert allocate_bits(np.zeros((0, 3)), [], [], (2, 4, 8), 0) == []
    # the binding's wire bytes are the Python formula, buckets above 8192 clamped
    for n in (0, 1, 7, 8, 9, 8191, 8192, 8193, 123457):
        for bits in (1, 2, 3, 4, 8, 32):
            for b in (0, 1, 3, 8, 13, 512, 8192, 8193, 20000):
                assert layer_wire_bytes(n, bits, b) == _layer_wire_bytes(n, bits, b), (n, bits, b)


# ---- native hook at world 2 -----------------------------------------------------------------------
def _train(rank, world, state, native, steps=8):
    """Like test_adaptive_bits_cpu._train, recording the whole registered table at every step."""
    import torch_cgx_b200 as cgx
    from torch.nn.parallel import DistributedDataParallel as DDP

    cgx.reset_layers()
    torch.manual_seed(0)
    ddp = DDP(_Net())
    handle = cgx.register_cgx_hook(ddp, state, native=native)
    assert (handle is not None) == native
    opt = torch.optim.SGD(ddp.parameters(), lr=0.002)
    tables = []
    for step in range(steps):
        g = torch.Generator().manual_seed(100 + step * world + rank)  # different data per rank
        x, y = torch.randn(16, 64, generator=g), torch.randint(0, 10, (16,), generator=g)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ddp(x), y).backward()
        opt.step()
        tables.append({b: [tuple(r) for r in cgx._C.registered_bucket(b)]
                       for b in range(cgx._C.num_registered_buckets())})
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    return flat, tables


def _same_on_every_rank(world, t):
    gathered = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    return all(torch.equal(gathered[0], g) for g in gathered[1:])


def _native_world2(rank, world):
    import torch_cgx_b200 as cgx

    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        params = {"bits": 4, "bucket_size": 64}
        py = cgx.AdaptiveCGXState(None, 16, params, period=3)
        flat_py, tables_py = _train(rank, world, py, native=False)
        nat = cgx.AdaptiveCGXState(None, 16, params, period=3)
        flat_nat, tables_nat = _train(rank, world, nat, native=True)
        assert tables_nat == tables_py
        assert len({r[1] for t in tables_nat[-1].values() for r in t}) > 1  # the widths did change
        assert nat.assignment == py.assignment and nat.assignment
        assert nat.adapted_layers == py.adapted_layers
        assert nat.last_errors.dtype == torch.float64 and torch.equal(nat.last_errors, py.last_errors)
        assert torch.equal(flat_nat, flat_py)
        assert _same_on_every_rank(world, flat_nat)
        widths = torch.tensor([r[1] for b in sorted(tables_nat[-1]) for r in tables_nat[-1][b]])
        assert _same_on_every_rank(world, widths)
        assert nat.state_dict()["assignment"] == py.state_dict()["assignment"]

        # one candidate: the plain native CGXState trajectory, bit for bit
        one, t_one = _train(rank, world, cgx.AdaptiveCGXState(None, 16, params, candidate_bits=(4,), period=2),
                            native=True)
        plain, t_plain = _train(rank, world, cgx.CGXState(None, 16, params), native=True)
        assert torch.equal(one, plain) and t_one == t_plain

        # checkpoints cross between the hooks; a load before registration applies at registration
        for src, native in ((py, True), (nat, False)):
            st = cgx.AdaptiveCGXState(None, 16, params, period=1000)
            st.load_state_dict(src.state_dict())
            _, t = _train(rank, world, st, native=native, steps=3)
            assert st.assignment == src.assignment
            assert all(t[2][b][l][1] == bits for (b, l), bits in src.assignment.items())
        # a load after installing the native hook reaches it too
        st = cgx.AdaptiveCGXState(None, 16, params, period=1000)
        cgx.reset_layers()
        torch.manual_seed(0)
        from torch.nn.parallel import DistributedDataParallel as DDP

        ddp = DDP(_Net())
        cgx.register_cgx_hook(ddp, st, native=True)
        st.load_state_dict(py.state_dict())
        for _ in range(3):
            x = torch.randn(16, 64)
            torch.nn.functional.cross_entropy(ddp(x), torch.zeros(16, dtype=torch.long)).backward()
        assert st.assignment == py.assignment

        # the default still installs the Python hook for an adaptive state
        assert cgx.register_cgx_hook(DDP(_Net()), cgx.AdaptiveCGXState(None, 16, params)) is None

        # native=True needs a cgx group
        gloo = dist.new_group(backend="gloo")
        with pytest.raises(ValueError):
            cgx.register_cgx_hook(DDP(_Net(), process_group=gloo), cgx.AdaptiveCGXState(gloo, 16, params),
                                  native=True)
    finally:
        dist.destroy_process_group()


def test_native_adaptive_hook_world2_cpu():
    spawn(_native_world2, 2, env={"CGX_COMPRESS_CPU": "1"})
