"""Adaptive per-layer widths on the GPU: the quantization-error kernel against its CPU oracle and
the GPU round trip, and a one-GPU cgx DDP run of ResNet-18 with AdaptiveCGXState."""
import socket

import pytest
import torch
import torch.distributed as dist

from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BUCKETS = (8, 13, 100, 512, 1000, 1024, 4096, 8192)
SIZES = (1, 7, 1000, 12345, (1 << 20) + 3)
CANDS = (1, 2, 3, 4, 5, 6, 7, 8)


def _table(buckets, sizes, start=3):
    layers, off = [], start
    for b in buckets:
        for n in sizes:
            layers.append((off, n, 4, b))
            off += n + 5  # odd gaps: layer starts are not multiples of 8
    return layers, off


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("stochastic", [False, True], ids=["nearest", "stochastic"])
def test_kernel_matches_cpu(dtype, aligned, stochastic):
    from torch_cgx_b200.ops import quantization_error

    layers, n = _table(BUCKETS, SIZES, start=0 if aligned else 3)
    g = torch.Generator().manual_seed(7)
    base = (torch.randn(n + 1, generator=g) * torch.logspace(-3, 2, n + 1)[torch.randperm(n + 1, generator=g)]).to(dtype)
    t = base[:n] if aligned else base[1:]  # a view one element in: no 16-byte loads anywhere
    for skip in (False, True):
        cpu = quantization_error(t, layers, CANDS, stochastic=stochastic, prescale=0.5, skip_incomplete=skip)
        gpu = quantization_error(t.cuda(), layers, CANDS, stochastic=stochastic, prescale=0.5, skip_incomplete=skip)
        assert gpu.device.type == "cuda" and gpu.dtype == torch.float64 and gpu.shape == (len(layers), len(CANDS))
        torch.testing.assert_close(gpu.cpu(), cpu, rtol=1e-5, atol=0)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_kernel_matches_gpu_round_trip(dtype):
    from torch_cgx_b200.ops import fake_quantize, quantization_error

    layers, n = _table((8, 100, 512, 1024, 8192), (7, 1000, 70001))
    t = torch.randn(n, device="cuda", generator=torch.Generator("cuda").manual_seed(3)).to(dtype)
    err = quantization_error(t, layers, CANDS, prescale=0.25).cpu()
    xf = t.float() * 0.25  # the fp32 values the encoder sees
    for l, (off, m, _, b) in enumerate(layers):
        x = xf[off:off + m].contiguous()
        for k, bits in enumerate(CANDS):
            ref = ((fake_quantize(x, bits, b).double() - x.double()) ** 2).sum().item()
            assert err[l, k].item() == pytest.approx(ref, rel=1e-5, abs=0), (l, bits)


def test_kernel_is_reproducible_and_flags_non_finite():
    from torch_cgx_b200.ops import quantization_error

    t = torch.randn(3_000_003, device="cuda")
    layers = [(1, 1_000_000, 4, 1024), (1_000_001, 2_000_000, 4, 333)]
    a = quantization_error(t, layers, CANDS)
    for _ in range(3):
        assert torch.equal(quantization_error(t, layers, CANDS), a)
    for dtype in DTYPES:
        (x,), planted = edge_inputs(dtype, 64 * 512, 512, seed=5)
        lay = [(p.lo, p.hi - p.lo, 4, 512) for p in planted]
        row = quantization_error(x.cuda(), lay, CANDS).cpu()
        torch.testing.assert_close(row, quantization_error(x, lay, CANDS), rtol=0, atol=0, equal_nan=True)
        for p, r in zip(planted, row):
            if p.nonfinite:
                assert not torch.isfinite(r).any(), p
            elif p.case not in ("span_overflow", "wide_range"):
                # span_overflow: max - min overflows and the wire decodes NaN as well; wide_range: a
                # finite error whose square can overflow fp32
                assert torch.isfinite(r).all(), p


def test_binding_errors():
    from torch_cgx_b200 import _C

    t = torch.randn(100, device="cuda")
    with pytest.raises(RuntimeError):
        _C.quantization_error(t[::2], [(0, 10, 4, 8)], [4])
    with pytest.raises(RuntimeError):
        _C.quantization_error(t.double(), [(0, 10, 4, 8)], [4])
    with pytest.raises(RuntimeError):
        _C.quantization_error(t, [(95, 10, 4, 8)], [4])
    with pytest.raises(RuntimeError):
        _C.quantization_error(t, [(0, 10, 4, 8)], [9])
    with pytest.raises(RuntimeError):
        _C.quantization_error(t, [(0, 10, 4, 8)], [0])


# ---- one-GPU DDP run ---------------------------------------------------------------------------
def _run(adaptive, steps=5):
    import torch_cgx_b200 as cgx
    from torch.nn.parallel import DistributedDataParallel as DDP
    from torch_cgx_b200.models import resnet18
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes

    torch.manual_seed(0)
    model = resnet18(num_classes=10, cifar_stem=True).cuda().to(memory_format=torch.channels_last)
    ddp = DDP(model, device_ids=[0])
    params = {"bits": 4, "bucket_size": 512}
    state = (cgx.AdaptiveCGXState(None, 1024, params, period=1000) if adaptive
             else cgx.CGXState(None, 1024, params))
    err = {}

    def wrapper(st, bucket):  # squared error of the allreduced gradient against the local one
        local = bucket.buffer().detach().clone()
        step = st.step

        def done(fut):
            out = fut.value()
            err[step] = err.get(step, 0.0) + ((out.double() - local.double()) ** 2).sum().item()
            return out
        return cgx.cgx_hook(st, bucket).then(done)

    ddp.register_comm_hook(state, wrapper)
    opt = torch.optim.SGD(ddp.parameters(), lr=0.05, momentum=0.9)
    g = torch.Generator("cuda").manual_seed(1234)
    x = torch.randn(32, 3, 32, 32, device="cuda", generator=g).to(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), device="cuda", generator=g)
    be = cgx.get_backend()
    wire = []
    for _ in range(steps):
        be.reset_stats()
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(ddp(x), y)
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        wire.append(be.stats()[3])
    table = {b: cgx._C.registered_bucket(b) for b in range(cgx._C.num_registered_buckets())}
    sizes = 0
    if adaptive:
        sizes = sum(layer_wire_bytes(n, table[b][l][1], 512) for (b, l, _, n) in state.adapted_layers)
    else:
        sizes = sum(layer_wire_bytes(n, bits, 512) for b in table for (n, bits, _) in table[b] if bits <= 8)
    return state, err, wire, table, sizes


def test_ddp_resnet18_adaptive_one_gpu(clean_cgx_env):
    import torch_cgx_b200 as cgx

    torch.cuda.set_device(0)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        cgx.reset_layers()
        _, err_u, wire_u, _, bytes_u = _run(False)
        cgx.reset_layers()
        st, err_a, wire_a, table, bytes_a = _run(True)
        # layers registered at step 2, estimated there; the first decision applies at step 3
        assert st.assignment and len(set(st.assignment.values())) > 1, st.assignment
        for (b, l), bits in st.assignment.items():
            assert table[b][l][1] == bits
        assert st.last_errors is not None and st.last_errors.shape == (len(st.adapted_layers), 7)
        assert bytes_a <= bytes_u
        # the plan pads every block record to 16 bytes, which the allocator's costs leave out
        blocks = sum(-(-n // 8192) for (_, _, _, n) in st.adapted_layers)
        assert wire_a[3] <= wire_u[3] + 32 * blocks, (wire_a, wire_u)
        assert err_a[3] <= err_u[3], (err_a, err_u)
        assert wire_a[2] == wire_u[2] and err_a[2] == err_u[2]  # step 2 is uniform in both runs
    finally:
        dist.destroy_process_group()
