"""Adaptive FSDP2 widths on the H100: the sharded estimator kernel against its CPU oracle bit for
bit; adapted tables through the reduce-scatter and all-gather kernels of W virtual ranks
(C.LocalSraGroup) against the simulators and the references; AdaptiveFSDPState on a real FSDP2
model at world 1; and, with several GPUs, an FSDP2 MLP whose ranks must agree on every width."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.ops.bit_allocation import allocate_bits, layer_wire_bytes
from torch_cgx_b200.ops.quantization import quantization_error
from torch_cgx_b200.parallel.adaptive import _sum_allocate_broadcast

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs
from test_all_gather_gpu import MIN_LANE, lanes_for, make_group, slot_for

pytestmark = pytest.mark.gpu
C = cgx._C
CANDS = (2, 3, 4, 5, 6, 7, 8)
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
# one shard: odd sizes, a raw bias, buckets of 100, 512 and 10000 (clamped to 8192) via the table
PARAMS = [((37, 29), 1073), ((37,), 37), ((64, 64), 4096), ((3, 3333), 9999), ((13,), 13), ((50, 401), 20050)]


def _table(bits, buckets=(100, 512, 10000)):
    t = cgx.fsdp_shard_table(PARAMS, bits, 512)
    adapted = [i for i, l in enumerate(t) if l[2] <= 8]
    return [(o, n, b, buckets[adapted.index(i) % len(buckets)] if b <= 8 else k)
            for i, (o, n, b, k) in enumerate(t)]


S = sum(n for _, n in PARAMS)


def _chunks(dtype, W, seed):
    """W chunks of S elements with the hostile cases of _edge_inputs, scaled per chunk."""
    xs, _ = edge_inputs(dtype, S, 512, seed, world=W)
    return torch.cat([x.reshape(-1) for x in xs])


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("chunks", [1, 2, 3, 8])
@pytest.mark.parametrize("stochastic", [False, True], ids=["nearest", "stochastic"])
def test_sharded_kernel_equals_cpu_oracle(dtype, chunks, stochastic):
    layers = [l for l in _table(4) if l[2] <= 8]
    t = _chunks(dtype, chunks, seed=chunks)
    for offset in (0, 1, 3):  # unaligned views
        buf = torch.zeros(offset + t.numel() + 8, dtype=dtype, device="cuda")
        view = buf[offset:offset + t.numel()]
        view.copy_(t)
        for skip in sorted({-1, 0, chunks - 1}):
            kw = dict(stochastic=stochastic, prescale=1.0 / chunks, chunks=chunks, skip_chunk=skip)
            got = quantization_error(view, layers, CANDS, **kw)
            again = quantization_error(view, layers, CANDS, **kw)
            torch.cuda.synchronize()
            assert_same(got.cpu(), quantization_error(t, layers, CANDS, **kw), f"offset {offset} skip {skip}")
            assert_same(again.cpu(), got.cpu(), "repeated call")
    if chunks == 1:
        plain = quantization_error(t.cuda(), layers, CANDS, stochastic=stochastic, prescale=1.0)
        assert_same(quantization_error(t.cuda(), layers, CANDS, stochastic=stochastic, chunks=1, skip_chunk=-1).cpu(),
                    plain.cpu(), "chunks=1")


def _decide(table, layers, target):
    """Adapted copy of `layers` from the shared decision helper on a world-1 gloo group."""
    rows = [i for i, l in enumerate(layers) if l[2] <= 8]
    numels = [layers[i][1] for i in rows]
    buckets = [layers[i][3] for i in rows]
    budget = sum(layer_wire_bytes(n, target, b) for n, b in zip(numels, buckets))
    store = dist.HashStore()
    dist.init_process_group("gloo", store=store, rank=0, world_size=1)
    try:
        summed, choice = _sum_allocate_broadcast([table.cpu()], [(numels, buckets, budget, [target] * len(rows), target)],
                                                 CANDS, dist.group.WORLD, torch.device("cpu"))
    finally:
        dist.destroy_process_group()
    out = list(layers)
    for i, bits in zip(rows, choice):
        o, n, _, k = out[i]
        out[i] = (o, n, bits, k)
    # the adapted assignment's estimated error is no larger than the uniform one
    col = {b: k for k, b in enumerate(CANDS)}
    adapted = sum(summed[r, col[b]].item() for r, b in enumerate(choice))
    uniform = sum(summed[r, col[target]].item() for r in range(len(rows)))
    assert adapted <= uniform, (adapted, uniform)
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=str)
@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("average", [False, True], ids=["sum", "avg"])
def test_adapted_tables_through_the_kernels(dtype, W, average):
    g = torch.Generator().manual_seed(W)
    scales = torch.cat([torch.full((n,), 10.0 ** (i % 3 - 1)) for i, (_, n) in enumerate(PARAMS)])
    ins = [((torch.randn(W * S, generator=g) * scales.repeat(W)) * (r + 1)).to(dtype) for r in range(W)]
    ps = 1.0 / W if average else 1.0
    # reduce-scatter: every rank's sharded estimate, summed over the ranks
    rs0 = _table(4)
    rows = [l for l in rs0 if l[2] <= 8]
    tables = [quantization_error(x.cuda(), rows, CANDS, prescale=ps, chunks=W, skip_chunk=r) for r, x in enumerate(ins)]
    rs_layers = _decide(sum(t.cpu() for t in tables), rs0, 4)
    assert len({l[2] for l in rs_layers if l[2] <= 8}) > 1, rs_layers
    grp = make_group(W, dtype, max(slot_for(rs_layers, W, S, dtype), 64 << 10))
    outs = [torch.empty(S, dtype=dtype, device="cuda") for _ in range(W)]
    grp.reduce_scatter([x.cuda() for x in ins], outs, rs_layers, average, False, False, 5, 1)
    torch.cuda.synchronize()
    grp.check()
    sim = [torch.empty(S, dtype=dtype) for _ in range(W)]
    C.reduce_scatter_simulate(ins, sim, rs_layers, lanes_for(W, dtype), average, False, False, 5, 1, MIN_LANE)
    ref = O.reduce_scatter_reference(ins, rs_layers, average=average)
    for r in range(W):
        assert_same(outs[r].cpu(), sim[r], f"rank {r} vs simulator")
        assert_same(outs[r].cpu(), ref[r], f"rank {r} vs reference")
    # all-gather of the reduced shards: every rank estimates its own shard
    ag0 = _table(6)
    shards = [o.cpu() for o in outs]
    rows = [l for l in ag0 if l[2] <= 8]
    ag_layers = _decide(sum(quantization_error(s.cuda(), rows, CANDS).cpu() for s in shards), ag0, 6)
    gathered = [torch.empty(W * S, dtype=dtype, device="cuda") for _ in range(W)]
    grp.all_gather([s.cuda() for s in shards], gathered, ag_layers, False, 5, 2)
    torch.cuda.synchronize()
    grp.check()
    sim = [torch.empty(W * S, dtype=dtype) for _ in range(W)]
    C.all_gather_simulate(shards, sim, ag_layers, False, 5, 2)
    ref = O.all_gather_reference(shards, ag_layers)
    for r in range(W):
        assert_same(gathered[r].cpu(), sim[r], f"rank {r} vs simulator")
        assert_same(gathered[r].cpu(), ref, f"rank {r} vs reference")


# ---- FSDP2 at world 1 -----------------------------------------------------------------------------
def _model():
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(256, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256),
                            torch.nn.LayerNorm(256), torch.nn.Linear(256, 64), torch.nn.Linear(64, 10))
    with torch.no_grad():
        for layer, s in ((m[0], 0.01), (m[2], 1.0), (m[4], 30.0), (m[5], 3.0)):
            layer.weight.mul_(s)
    return m.cuda()


def _flat(model):
    return torch.cat([fp._sharded_param_data.detach().reshape(-1)
                      for fp in model._get_fsdp_state()._fsdp_param_group.fsdp_params])


def _gather(comm, flat):
    out = comm.allocate((flat.numel(),), dtype=flat.dtype, device=flat.device)
    out.copy_(flat)
    comm(output_tensor=out, input_tensor=out[:flat.numel()], group=dist.group.WORLD, async_op=False)
    torch.cuda.synchronize()
    return out


def _kernels(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _fsdp_world1(rank, world):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(0)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        model = fully_shard(_model())
        st = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=4, bucket_size=512, period=1000)
        comms = cgx.set_cgx_adaptive(model, st)
        rs, ag = comms
        assert isinstance(rs, cgx.CGXReduceScatter) and isinstance(ag, cgx.CGXAllGather)
        assert st.rows("all_gather") == ["0.weight", "2.weight", "4.weight", "5.weight"]
        uniform = list(ag.layers)
        x = torch.randn(32, 256, device="cuda")
        flat = _flat(model)
        with torch.no_grad():
            model(x)  # step 0: the round opens
        assert ag.layers == uniform
        rows = [l for l in ag.layers if l[2] <= 8]
        names = _kernels(lambda: _gather(ag, flat))  # in the round: estimate, then the all-gather
        assert sum("qerr" in n for n in names) == 2, names
        assert ag.layers == uniform  # widths change only in the root pre-forward
        table = quantization_error(flat, rows, st.candidate_bits).cpu()
        with torch.no_grad():
            model(x)  # step 1: the decision
        budget = sum(layer_wire_bytes(n, 4, 512) for (_, n, _, _) in rows)
        want = allocate_bits(table.numpy(), [l[1] for l in rows], [512] * len(rows), st.candidate_bits, budget,
                             [4] * len(rows), target_bits=4)
        got = [l[2] for l in ag.layers if l[2] <= 8]
        assert got == want and len(set(want)) > 1, (got, want)
        assert torch.equal(st.last_errors["all_gather"], table)
        assert "reduce_scatter" not in st.last_errors and all(l[2] in (4, 32) for l in rs.layers)
        out = _gather(ag, flat)
        assert_same(out, O.quantize_dequantize_layers(flat.cpu(), ag.layers))
        # off-round: the same launches as a plain CGXAllGather with the same table
        plain = cgx.CGXAllGather(4, 512, ag.layers, "plain")
        adapted_names = _kernels(lambda: _gather(ag, flat))
        plain_names = _kernels(lambda: _gather(plain, flat))
        assert sorted(adapted_names) == sorted(plain_names) and not any("qerr" in n for n in adapted_names)
        be = cgx.get_backend()
        s0 = be.stats()[1]
        _gather(ag, flat)
        s1 = be.stats()[1]
        _gather(plain, flat)
        assert be.stats()[1] - s1 == s1 - s0 > 0
        # the reduce-scatter at world 1 is not adapted: it never estimates
        st._round_open = True
        rs(torch.empty(flat.numel(), device="cuda"), flat.clone(), dist.group.WORLD, dist.ReduceOp.AVG)
        assert id(rs) not in st._tables
        st._round_open = False

        # checkpoint: a fresh model gathers with the same tables before its first decision
        sd = st.state_dict()
        model2 = fully_shard(_model())
        st2 = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=4, bucket_size=512, period=1000)
        st2.load_state_dict(sd)
        _, ag2 = cgx.set_cgx_adaptive(model2, st2)
        assert ag2.layers == ag.layers
        with torch.no_grad():
            model2(x)
        assert_same(_gather(ag2, _flat(model2)), out)

        # estimate and decision steps refuse CUDA graph capture; calls outside a round are capturable
        st3 = cgx.AdaptiveFSDPState(reduce_scatter_bits=None, all_gather_bits=4, bucket_size=512, period=1)
        model3 = fully_shard(_model())
        (ag3,) = cgx.set_cgx_adaptive(model3, st3)
        with torch.no_grad():
            model3(x)  # the round opens
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            g = torch.cuda.CUDAGraph()
            with pytest.raises(RuntimeError, match="capture"):
                with torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
                    st3.maybe_estimate(ag3, _flat(model3), dist.group.WORLD, average=False)
        torch.cuda.current_stream().wait_stream(side)
        _gather(ag3, _flat(model3))  # the estimate, outside capture
        with torch.cuda.stream(side):
            g = torch.cuda.CUDAGraph()
            with pytest.raises(RuntimeError, match="capture"):
                with torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
                    st3.pre_forward()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_fsdp2_adaptive_world1():
    spawn(_fsdp_world1, 1)


def _non_root(rank, world):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(0)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        m = _model()
        fully_shard(m[0])
        fully_shard(m)
        with torch.no_grad():
            m(torch.randn(2, 256, device="cuda"))  # lazy init: m is the root
        with pytest.raises(ValueError, match="root"):
            cgx.set_cgx_adaptive(m[0], cgx.AdaptiveFSDPState())
    finally:
        dist.destroy_process_group()


def test_set_cgx_adaptive_refuses_a_non_root():
    spawn(_non_root, 1)


# ---- several GPUs ----------------------------------------------------------------------------------
def _fsdp_mlp(rank, world, steps):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        losses = {}
        for kind in ("nccl", "cgx"):
            torch.manual_seed(0)
            blocks = [torch.nn.Sequential(torch.nn.Linear(512, 512), torch.nn.GELU()) for _ in range(4)]
            model = torch.nn.Sequential(*blocks, torch.nn.Linear(512, 10)).cuda()
            for m in model[:4]:
                fully_shard(m)
            fully_shard(model)
            st = None
            if kind == "cgx":
                st = cgx.AdaptiveFSDPState(reduce_scatter_bits=6, all_gather_bits=8, bucket_size=512, period=4)
                cgx.set_cgx_adaptive(model, st)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            g = torch.Generator(device="cuda").manual_seed(rank)
            out = []
            for _ in range(steps):
                x = torch.randn(64, 512, device="cuda", generator=g) * torch.logspace(-2, 1, 512, device="cuda")
                y = (x[:, :10] > 0).float().argmax(1)
                loss = torch.nn.functional.cross_entropy(model(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad()
                out.append(loss.item())
            losses[kind] = np.array(out)
            if st is not None:
                both = [None] * world
                dist.all_gather_object(both, sorted(st.assignment.items()))
                assert all(b == both[0] for b in both)
                assert len({b for (k, _), b in st.assignment.items() if k == "reduce_scatter"}) > 1, st.assignment
                group = model[0]._get_fsdp_state()._fsdp_param_group
                rs, ag = group._reduce_scatter_comm, group._all_gather_comm
                S = rs.numel
                gen = torch.Generator().manual_seed(world)
                ins = [torch.randn(world * S, generator=gen) * (r + 1) for r in range(world)]
                o = torch.empty(S, device="cuda")
                rs(o, ins[rank].cuda(), dist.group.WORLD, dist.ReduceOp.AVG)
                ag_out = torch.empty(world * S, device="cuda")
                ag(ag_out, ins[rank][:S].cuda(), dist.group.WORLD)
                torch.cuda.synchronize()
                assert_same(ag_out.cpu(), O.all_gather_reference([x[:S] for x in ins], ag.layers))
                if int(os.environ.get("CGX_LOCAL_SIZE", world)) == world:  # one node: single stage
                    assert_same(o.cpu(), O.reduce_scatter_reference(ins, rs.layers, average=True)[rank])
        assert np.all(np.abs(losses["cgx"] - losses["nccl"]) <= 0.03 * losses["nccl"]), losses
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world,local", [(2, None), (4, None), (4, 2)])
def test_fsdp2_adaptive_tracks_nccl(world, local):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_fsdp_mlp, world, args=(12,), env={} if local is None else {"CGX_LOCAL_SIZE": str(local)}, timeout=600)
