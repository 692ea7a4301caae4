"""The adaptive native DDP hook on the GPU: ResNet-18 at world 1 against the Python hook, bit for bit;
what an off-period step launches; and world 2 / 4 runs across GPUs."""
import socket

import pytest
import torch
import torch.distributed as dist

from _dist_utils import spawn

pytestmark = pytest.mark.gpu

PARAMS = {"bits": 4, "bucket_size": 512}


def _run(state, native, steps, rank=0, profile_step=None):
    """test_adaptive_bits_gpu._run's setup: ResNet-18, channels_last, bf16 autocast, SGD momentum."""
    import torch_cgx_b200 as cgx
    from torch.nn.parallel import DistributedDataParallel as DDP
    from torch_cgx_b200.models import resnet18

    cgx.reset_layers()
    torch.manual_seed(0)
    model = resnet18(num_classes=10, cifar_stem=True).cuda().to(memory_format=torch.channels_last)
    ddp = DDP(model, device_ids=[rank])
    handle = cgx.register_cgx_hook(ddp, state, native=native)
    assert (handle is not None) == native
    opt = torch.optim.SGD(ddp.parameters(), lr=0.05, momentum=0.9)
    g = torch.Generator("cuda").manual_seed(1234 + rank)
    x = torch.randn(32, 3, 32, 32, device="cuda", generator=g).to(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (32,), device="cuda", generator=g)
    be = cgx.get_backend()
    wire, tables, prof = [], [], None
    for step in range(steps):
        be.reset_stats()
        ctx = None
        if step == profile_step:
            torch.cuda.synchronize()
            ctx = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
            ctx.__enter__()
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(ddp(x), y)
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        if ctx is not None:
            ctx.__exit__(None, None, None)
            prof = ctx
        wire.append(be.stats()[3])
        tables.append({b: cgx._C.registered_bucket(b) for b in range(cgx._C.num_registered_buckets())})
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    return flat, tables, wire, prof


def _init_world1():
    torch.cuda.set_device(0)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)


def test_native_equals_python_resnet18_one_gpu(clean_cgx_env):
    import torch_cgx_b200 as cgx

    _init_world1()
    try:
        py = cgx.AdaptiveCGXState(None, 1024, PARAMS, period=2)
        flat_py, tables_py, wire_py, _ = _run(py, False, 7)
        nat = cgx.AdaptiveCGXState(None, 1024, PARAMS, period=2)
        flat_nat, tables_nat, wire_nat, _ = _run(nat, True, 7)
        assert tables_nat == tables_py
        assert nat.assignment == py.assignment and len(set(nat.assignment.values())) > 1, nat.assignment
        assert nat.adapted_layers == py.adapted_layers
        assert nat.last_errors.shape == (len(nat.adapted_layers), 7)
        assert torch.equal(nat.last_errors, py.last_errors)
        assert torch.equal(flat_nat, flat_py)
        assert wire_nat == wire_py
    finally:
        dist.destroy_process_group()


def _events(prof):
    kernels, dtoh = [], 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "Memcpy" in e.name:
            dtoh += "DtoH" in e.name
        elif "Memset" not in e.name:
            kernels.append(e.name)
    return kernels, dtoh


def test_off_period_step_launches_like_the_plain_hook(clean_cgx_env):
    import torch_cgx_b200 as cgx

    _init_world1()
    try:
        # registered and estimated at step 2, decided at step 3; step 4 does neither
        plain = cgx.CGXState(None, 1024, PARAMS)
        _, _, _, prof_plain = _run(plain, True, 5, profile_step=4)
        st = cgx.AdaptiveCGXState(None, 1024, PARAMS, period=3)
        _, _, _, prof_nat = _run(st, True, 5, profile_step=4)
        assert st.last_errors is not None  # the decision did run, at step 3
        k_plain, dtoh_plain = _events(prof_plain)
        k_nat, dtoh_nat = _events(prof_nat)
        assert not [k for k in k_nat if "qerr" in k]
        assert dtoh_nat == dtoh_plain
        # the mixed widths pick other instantiations of the fused kernel, one launch per bucket as before
        ar = lambda ks: [k for k in ks if "sra_kernel" in k or "oneshot_kernel" in k]  # noqa: E731
        assert len(ar(k_nat)) == len(ar(k_plain)) > 0
        assert len(k_nat) == len(k_plain)
    finally:
        dist.destroy_process_group()


def _multi(rank, world):
    import torch_cgx_b200 as cgx

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        py = cgx.AdaptiveCGXState(None, 1024, PARAMS, period=2)
        flat_py, tables_py, _, _ = _run(py, False, 6, rank=rank)
        nat = cgx.AdaptiveCGXState(None, 1024, PARAMS, period=2)
        flat_nat, tables_nat, _, _ = _run(nat, True, 6, rank=rank)
        assert tables_nat == tables_py and nat.assignment == py.assignment
        assert torch.equal(nat.last_errors, py.last_errors)
        assert torch.equal(flat_nat, flat_py)
        widths = torch.tensor([r[1] for b in sorted(tables_nat[-1]) for r in tables_nat[-1][b]], device="cuda")
        gathered = [torch.zeros_like(widths) for _ in range(world)]
        dist.all_gather(gathered, widths)
        assert all(torch.equal(gathered[0], w) for w in gathered[1:])
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
def test_native_equals_python_multi_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_multi, world, timeout=600)
