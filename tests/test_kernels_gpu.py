"""sm_90a kernels vs. the CPU implementation of the same op (bit-exact) and the
pure-PyTorch fp32 oracle.  Single GPU: the fused kernel is exercised with W
virtual ranks (W heaps, W streams) inside one process."""
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import fake_quantize, quantize, dequantize
from torch_cgx_b200.ops.oracle import quantize_dequantize_like

from _bitwise import assert_same

pytestmark = pytest.mark.gpu
C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def dev():
    return torch.device("cuda", 0)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bits", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("bucket", [64, 100, 512, 2048])
def test_quantize_kernel_bytes_match_cpu(dtype, bits, bucket):
    torch.manual_seed(bits * 7 + bucket)
    x = (torch.randn(50_003) * 2).to(dtype)
    w_cpu = quantize(x, bits, bucket)
    w_gpu = quantize(x.to(dev()), bits, bucket)
    assert_same(w_cpu, w_gpu.cpu())
    y_gpu = dequantize(w_gpu, x.to(dev()), bits, bucket)
    y_cpu = dequantize(w_cpu, x, bits, bucket)
    assert_same(y_cpu, y_gpu.cpu())
    # and against the independent fp32 PyTorch reference of the op
    assert_same(y_gpu.cpu(), quantize_dequantize_like(x, bits, bucket))


@pytest.mark.parametrize("dtype", DTYPES)
def test_unaligned_layers_and_mixed_config(dtype):
    torch.manual_seed(0)
    # odd offsets => 16 B-misaligned layer starts (scalar load/store paths)
    layers = [(0, 4099, 4, 512), (4099, 33, 32, 512), (4132, 10_001, 8, 64), (14_133, 7, 32, 512),
              (14_140, 9000, 2, 128), (23_140, 5, 3, 8)]
    n = 23_145
    x = torch.randn(n).to(dtype)
    w_cpu = C.quantize(x, layers, 1, 1, False, 1.0, False, 0, 0, 0, 0, 2048)
    w_gpu = C.quantize(x.to(dev()), layers, 1, 1, False, 1.0, False, 0, 0, 0, 0, 2048)
    assert_same(w_cpu, w_gpu.cpu())
    y_cpu = C.dequantize(w_cpu, x, layers, 1, 1, False, 2048)
    y_gpu = C.dequantize(w_gpu, x.to(dev()), layers, 1, 1, False, 2048)
    assert_same(y_cpu, y_gpu.cpu())


def test_stochastic_kernel_matches_cpu_philox():
    x = torch.randn(100_000)
    a = fake_quantize(x, 2, 512, stochastic=True, seed=3, seq=5)
    b = fake_quantize(x.to(dev()), 2, 512, stochastic=True, seed=3, seq=5)
    assert_same(a, b.cpu())


def test_elementwise_helpers():
    x = torch.randn(100_001, device=dev())
    y = torch.randn(100_001, device=dev())
    assert_same(C.add(x, y), x + y)
    z = x.clone()
    C.scale_(z, 0.125)
    assert_same(z, x * 0.125)
    assert_same(C.convert(x, torch.float16), x.half())
    assert_same(C.convert(x.half(), torch.float32), x.half().float())
    assert_same(C.convert(x, torch.bfloat16), x.bfloat16())


# --------------------------------------------------------------------------
def _run_local(world, layers, n, dtype, lanes=8, average=False, skip_incomplete=False, stochastic=False,
               seed=0, seq=1, min_lane_elems=256, repeats=1, group=None, gen_seed=0):
    torch.manual_seed(gen_seed)
    ins = [(torch.randn(n) * (r + 1)).to(dtype) for r in range(world)]
    cpu = [t.clone() for t in ins]
    C.sra_simulate(cpu, layers, lanes, average, skip_incomplete, stochastic, seed, seq, min_lane_elems)
    g = group or C.LocalSraGroup(world, lanes, 4 << 20, 5000, min_lane_elems)
    for _ in range(repeats):
        gpu = [t.to(dev()) for t in ins]
        g.allreduce(gpu, layers, average, skip_incomplete, stochastic, seed, seq)
        torch.cuda.synchronize()
        g.check()
        for r in range(world):
            assert_same(gpu[r].cpu(), cpu[r], f"rank {r} differs from the CPU SRA oracle")
    return g


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_sra_matches_cpu_oracle(world, dtype):
    n = 200_000
    _run_local(world, [(0, n, 4, 512)], n, dtype)


@pytest.mark.parametrize("bits", [1, 2, 3, 5, 8])
def test_fused_sra_bits(bits):
    n = 70_001
    _run_local(4, [(0, n, bits, 512)], n, torch.float32)


def test_fused_sra_mixed_layers_unaligned():
    layers = [(0, 4099, 4, 512), (4099, 33, 32, 512), (4132, 100_001, 8, 64), (104_133, 7, 32, 512),
              (104_140, 90_000, 2, 128)]
    n = 194_140
    for dtype in DTYPES:
        _run_local(4, layers, n, dtype, lanes=6)


def test_fused_sra_uncompressed_and_average():
    n = 123_457
    _run_local(8, [(0, n, 32, 512)], n, torch.float32, average=True)
    _run_local(8, [(0, n, 32, 512)], n, torch.float16, average=False)
    _run_local(2, [(0, n, 4, 512)], n, torch.bfloat16, average=True)


def test_fused_sra_skip_incomplete_and_stochastic():
    n = 50_000 + 123
    _run_local(4, [(0, n, 4, 512)], n, torch.float32, skip_incomplete=True)
    _run_local(4, [(0, n, 2, 512)], n, torch.float32, stochastic=True, seed=11, seq=3)


@pytest.mark.parametrize("stages", [1, 2, 3, 4])
def test_fused_sra_pipelined_stages_match_cpu_oracle(stages, monkeypatch):
    # the pipeline depth (pieces per chunk, one flag value each) must not change a single bit
    monkeypatch.setenv("CGX_STAGES", str(stages))
    n = 1_500_000
    _run_local(8, [(0, n, 4, 512)], n, torch.float32, repeats=2)
    _run_local(8, [(0, n, 4, 1024)], n, torch.float32, stochastic=True, seed=5, seq=9)
    layers = [(0, 4099, 4, 512), (4099, 33, 32, 512), (4132, 100_001, 8, 64), (104_133, 7, 32, 512),
              (104_140, 90_000, 2, 128), (194_140, 300_000, 32, 512)]
    _run_local(4, layers, 494_140, torch.bfloat16, lanes=6)
    _run_local(2, [(0, 3000, 4, 512)], 3000, torch.float16)   # fewer items than stages * warps


def test_fused_sra_repeated_calls_and_changing_plans():
    # epochs keep increasing across calls; plans (and lane counts) change between calls
    g = C.LocalSraGroup(4, 16, 4 << 20, 5000, 256)
    for i, n in enumerate([1000, 300_000, 17, 64_000, 300_000, 5]):
        bits = 4 if n >= 16 else 32
        _run_local(4, [(0, n, bits, 512)], n, torch.float32, lanes=16, repeats=2, group=g, gen_seed=i)


def test_fused_sra_tiny_and_exact_constant():
    for world in (2, 8):
        for n in (1, 2, 8, 128, 1024):
            ins = [torch.full((n,), float(r + 1), device=dev()) for r in range(world)]
            g = C.LocalSraGroup(world, 4, 1 << 20, 5000, 256)
            g.allreduce(ins, [(0, n, 4 if n >= 16 else 32, 512)])
            torch.cuda.synchronize()
            for t in ins:
                assert_same(t.cpu(), torch.full((n,), float(world * (world + 1) // 2)))


def test_fused_sra_large_buffer_many_lanes():
    # 16M elements, 2 ranks x 64 lanes (all 128 CTAs co-resident on one H100)
    n = 16 * 1024 * 1024
    torch.manual_seed(0)
    ins = [torch.randn(n), torch.randn(n) * 3]
    cpu = [t.clone() for t in ins]
    C.sra_simulate(cpu, [(0, n, 4, 512)], 64, False, False, False, 0, 1, 2048)
    g = C.LocalSraGroup(2, 64, 24 << 20, 10000, 2048)
    gpu = [t.to(dev()) for t in ins]
    g.allreduce(gpu, [(0, n, 4, 512)], False, False, False, 0, 1)
    torch.cuda.synchronize()
    g.check()
    assert_same(gpu[0].cpu(), cpu[0])
    assert_same(gpu[1].cpu(), cpu[1])


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_oneshot_kernel_matches_cpu_oracle(world, dtype):
    layers = [(0, 4099, 4, 512), (4099, 33, 32, 512), (4132, 60_001, 8, 64), (64_133, 7, 32, 512),
              (64_140, 50_000, 4, 1024)]
    n = 114_140
    torch.manual_seed(world)
    ins = [(torch.randn(n) * (r + 1)).to(dtype) for r in range(world)]
    for average in (False, True):
        cpu = [t.clone() for t in ins]
        C.oneshot_simulate(cpu, layers, 8, average, False, False, 0, 1, 256)
        g = C.LocalSraGroup(world, 8, 4 << 20, 5000, 256)
        for _ in range(3):  # alternating one-shot regions
            gpu = [t.to(dev()) for t in ins]
            g.allreduce_oneshot(gpu, layers, average, False, False, 0, 1)
            torch.cuda.synchronize()
            g.check()
            for r in range(world):
                assert_same(gpu[r].cpu(), cpu[r])
        # interleave with the three-phase kernel on the same heap
        gpu = [t.to(dev()) for t in ins]
        g.allreduce(gpu, layers, average, False, False, 0, 1)
        gpu = [t.to(dev()) for t in ins]
        g.allreduce_oneshot(gpu, layers, average, False, False, 0, 1)
        torch.cuda.synchronize()
        for r in range(world):
            assert_same(gpu[r].cpu(), cpu[r])
