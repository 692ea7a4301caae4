"""sm_90a kernels on hostile inputs and on every bucket shape, against the CPU code (bytes) and
the independent reference of the operation (torch_cgx_b200/ops/oracle.py).

Every comparison is NaN-aware and bitwise (tests/_bitwise.py). Every kernel runs on views at
element offsets 1, 3 and 5 into buffers filled with a sentinel: the bases are not 16-byte
aligned, and the elements around each view must be unchanged afterwards. The fused SRA and
one-shot kernels run with W virtual ranks on one GPU (C.LocalSraGroup). All parameters are
fixed lists, so a failure reproduces exactly."""
import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import fake_quantize
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _edge_inputs import CASES, FINITE, _applicable, edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
BUCKETS = [1, 3, 7, 8, 16, 32, 64, 100, 256, 512, 1000, 1024, 2048, 8192]
GUARD = 64        # sentinel elements after every view
SENTINEL = -7.25  # exact in every dtype
MIN_LANE = 256


def dev():
    return torch.device("cuda", 0)


def layer_elems(dtype, bucket):
    """Elements of the edge layer: room for every planted case (each on an odd bucket) and a
    partial last bucket, at least 8 full 512-element slices, capped for the largest buckets."""
    k = sum((len({p for p in (0, 7, 8, 15, 16, 255) if p < bucket} | {bucket - 1}) if c == "outlier" else 1)
            for c in CASES if _applicable(c, dtype))
    return min(max((2 * k + 2) * bucket, 4096), max(16 * bucket, 40_000)) + bucket // 2


def edge_table(nq, bits, bucket, extra):
    """Raw head (the edge layer starts misaligned), the edge layer, a raw layer, and optionally a
    5-bit layer so that the plan has no common bit width."""
    layers = [(0, 37, 32, 512), (37, nq, bits, bucket), (37 + nq, 301, 32, 512)]
    if extra:
        layers.append((338 + nq, 2000, 5, 64))
    return layers, layers[-1][0] + layers[-1][1]


def guarded(x, offset):
    """(buffer, view): x copied into buf[offset:offset+n] of a sentinel-filled CUDA buffer."""
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def assert_guards(buf, offset, n, what):
    b = buf.cpu()
    assert_same(b[:offset], torch.full((offset,), SENTINEL, dtype=b.dtype), f"{what}: elements before the view")
    assert_same(b[offset + n:], torch.full((GUARD,), SENTINEL, dtype=b.dtype), f"{what}: elements after the view")


def embed(x_layer, layers, total, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(total, generator=g).to(dtype)
    full[37:37 + x_layer.numel()] = x_layer
    return full


# ---- standalone quantize / dequantize ------------------------------------------------------------
@pytest.mark.parametrize("bucket", BUCKETS)
@pytest.mark.parametrize("bits", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_standalone_kernels_on_edge_inputs(dtype, bits, bucket):
    offset = (1, 3, 5)[(bits + bucket) % 3]
    nq = layer_elems(dtype, bucket)
    layers, total = edge_table(nq, bits, bucket, extra=bits % 2 == 0)
    xs, planted = edge_inputs(dtype, nq, bucket, 100 * bits + bucket, bits=bits)
    x = embed(xs[0], layers, total, dtype, bits)
    args = (1, 1, False, 1.0, False, 0, 0, 0, 0, 2048)
    w_cpu = C.quantize(x, layers, *args)
    buf, xv = guarded(x, offset)
    w_gpu = C.quantize(xv, layers, *args)
    assert_same(w_gpu, w_cpu, "wire bytes")
    assert_guards(buf, offset, total, "quantize input")
    y_cpu = C.dequantize(w_cpu, x, layers, 1, 1, False, 2048)
    y_gpu = C.dequantize(w_gpu, xv, layers, 1, 1, False, 2048)
    ref = O.quantize_dequantize_layers(x, layers)
    assert_same(y_gpu, y_cpu, "dequantize vs CPU")
    assert_same(y_gpu, ref, "dequantize vs reference")
    # the pre-planned codec writes into guarded wire and output buffers
    codec = C.PreparedCodec(layers, dtype, 0, False)
    wb = codec.wire_bytes()
    wbuf = torch.full((wb + GUARD,), 0xA5, dtype=torch.uint8, device=dev())
    codec.quantize(xv, wbuf[:wb])
    assert (wbuf[wb:] == 0xA5).all(), "codec quantize wrote past the wire buffer"
    obuf, ov = guarded(torch.zeros_like(x), offset)
    codec.dequantize(wbuf[:wb], ov)
    assert_same(ov, ref, "codec round trip vs reference")
    assert_guards(obuf, offset, total, "codec dequantize output")
    # fake_quantize of the edge layer alone: one layer, buckets from element 0
    lv = guarded(xs[0], offset)[1]
    assert_same(fake_quantize(lv, bits, bucket), O.quantize_dequantize_like(xs[0], bits, O.effective_bucket(bucket)),
                "fake_quantize vs reference")
    for p in planted:
        if p.nonfinite:
            assert not torch.isfinite(y_gpu[37 + p.lo:37 + p.hi].float()).any(), f"{p.case} did not poison its bucket"


# ---- fused SRA and one-shot kernels ----------------------------------------------------------------
def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def run_group(ins, layers, *, oneshot, average, skip_incomplete=False, stochastic=False, offset=1):
    """Allreduce CPU tensors with W virtual ranks; returns the results on the CPU.

    Every virtual rank's CTAs must be resident at once (they spin on each other's flags), and
    the slots must hold the largest chunk: both are checked before anything is launched."""
    W, dtype = len(ins), ins[0].dtype
    max_ctas = C.max_resident_ctas(DT_CODE[dtype])
    lanes = lanes_for(W, dtype)
    assert W * lanes <= max_ctas // 2, f"{W} ranks x {lanes} lanes cannot all be resident ({max_ctas} CTAs)"
    wire = max(C.build_plan(layers, world=w, lanes=lanes, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete,
                            min_lane_elems=MIN_LANE)["max_chunk_wire"] for w in (W, 1))
    g = C.LocalSraGroup(W, lanes, (wire + 255) // 256 * 256 + 256, 5000, MIN_LANE)
    n = ins[0].numel()
    bufs = [guarded(x, offset) for x in ins]
    views = [v for _, v in bufs]
    if oneshot:
        g.allreduce_oneshot(views, layers, average, skip_incomplete, stochastic, 5, 2)
    else:
        g.allreduce(views, layers, average, skip_incomplete, stochastic, 5, 2)
    torch.cuda.synchronize()
    g.check()
    for r, (buf, _) in enumerate(bufs):
        assert_guards(buf, offset, n, f"rank {r}")
    return [v.cpu() for v in views]


def _configs():
    out = []
    i = 0
    for world in (1, 2, 3, 5, 6, 7, 8, 16):
        for dtype in DTYPES:
            for average in (False, True):
                bucket = BUCKETS[(i * 5) % len(BUCKETS)]
                bits = 1 + (i * 3) % 8
                name = f"w{world}-{str(dtype)[6:]}-{'avg' if average else 'sum'}-b{bucket}-q{bits}"
                out.append(pytest.param(world, dtype, average, bucket, bits, i, id=name))
                i += 1
    return out


def check_allreduce(ins, layers, planted, *, oneshot, average, skip_incomplete, offset):
    W = len(ins)
    got = run_group(ins, layers, oneshot=oneshot, average=average, skip_incomplete=skip_incomplete, offset=offset)
    sim = [t.clone() for t in ins]
    if oneshot:
        C.oneshot_simulate(sim, layers, 1, average, skip_incomplete, False, 0, 0, MIN_LANE)
        ref = O.oneshot_reference(ins, layers, average=average, skip_incomplete=skip_incomplete)
    else:
        lanes = lanes_for(W, ins[0].dtype)
        C.sra_simulate(sim, layers, lanes, average, skip_incomplete, False, 0, 0, MIN_LANE)
        ref = O.sra_reference(ins, layers, lanes=lanes, min_lane_elems=MIN_LANE, average=average,
                              skip_incomplete=skip_incomplete)
    kind = "one-shot" if oneshot else "SRA"
    for r in range(W):
        assert_same(got[r], got[0], f"{kind}: rank {r} differs from rank 0")
        assert_same(got[r], sim[r], f"{kind}: rank {r} vs simulator")
        assert_same(got[r], ref[r], f"{kind}: rank {r} vs reference")
    # a bucket with a non-finite input on any rank is non-finite everywhere on every rank
    for p in planted:
        if p.nonfinite:
            for r in range(W):
                seg = got[r][37 + p.lo:37 + p.hi].float()
                assert not torch.isfinite(seg).any(), f"{kind}: {p.case} on rank {p.rank} leaked finite values"


@pytest.mark.parametrize("world,dtype,average,bucket,bits,i", _configs())
def test_fused_allreduce_on_edge_inputs(world, dtype, average, bucket, bits, i):
    nq = layer_elems(dtype, bucket)
    layers, total = edge_table(nq, bits, bucket, extra=i % 2 == 0)
    skip_incomplete = i % 3 == 0
    lanes = lanes_for(world, dtype)
    owners = O.block_owners(layers, total, world, lanes, dtype, skip_incomplete, MIN_LANE)[37:37 + nq]
    owners[owners < 0] = 0
    xs, planted = edge_inputs(dtype, nq, bucket, 1000 + i, world=world, bits=bits, owners=owners,
                              where="owner" if i % 2 else "peer")
    ins = [embed(x, layers, total, dtype, 7 * i + r) for r, x in enumerate(xs)]
    offset = (1, 3, 5)[i % 3]
    if skip_incomplete:  # the partial last bucket of the edge layer travels raw: nothing to poison there
        planted = [p for p in planted if p.hi - p.lo == bucket]
    check_allreduce(ins, layers, planted, oneshot=False, average=average, skip_incomplete=skip_incomplete,
                    offset=offset)
    if world > 1:
        check_allreduce(ins, layers, planted, oneshot=True, average=average, skip_incomplete=skip_incomplete,
                        offset=offset)


@pytest.mark.parametrize("bucket", [8, 16, 32, 256])
@pytest.mark.parametrize("bits", [1, 2, 3, 4, 5, 6, 7, 8])
def test_fused_sra_full_slices_small_buckets(bits, bucket):
    # lg = 0, 1, 2, 5: buckets inside a 512-element full slice (per-row meta, sub-warp min/max);
    # one common bit width so that the width-specialised kernels run
    world, dtype = 5, torch.float32
    nq = 32 * 1024 + bucket // 2  # several full slices in every lane of every rank
    layers = [(0, 37, 32, 512), (37, nq, bits, bucket)]
    lanes = lanes_for(world, dtype)
    plan = C.build_plan(layers, world=world, lanes=lanes, dtype=0, min_lane_elems=MIN_LANE)
    items = plan["items"]
    lg = {8: 0, 16: 1, 32: 2, 256: 5}[bucket]
    assert int(((items[:, 3] == 0) & (items[:, 4] == lg)).sum()) >= world * plan["lanes"], "no full slices to test"
    owners = O.block_owners(layers, 37 + nq, world, lanes, dtype, False, MIN_LANE)[37:]
    xs, planted = edge_inputs(dtype, nq, bucket, bits * 31 + bucket, world=world, bits=bits, owners=owners,
                              where="peer" if bits % 2 else "owner")
    ins = [embed(x, layers, 37 + nq, dtype, r) for r, x in enumerate(xs)]
    check_allreduce(ins, layers, planted, oneshot=False, average=bits % 2 == 0, skip_incomplete=False,
                    offset=(1, 3, 5)[bits % 3])
    check_allreduce(ins, layers, planted, oneshot=True, average=bits % 2 == 0, skip_incomplete=False,
                    offset=(1, 3, 5)[bits % 3])


@pytest.mark.parametrize("world", [3, 5, 16])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_fused_stochastic_within_exact_bound(world, dtype):
    # no bit-exact independent reference with stochastic rounding: the simulator gives the bits,
    # the reference's exact sum and bound check the values
    nq = 20_000
    layers = [(0, 37, 32, 512), (37, nq, 2, 512), (37 + nq, 5000, 4, 100)]
    total = 37 + nq + 5000
    xs, _ = edge_inputs(dtype, total, 512, world, world=world, bits=2, cases=FINITE)
    for average in (False, True):
        for oneshot in (False, True):
            got = run_group(xs, layers, oneshot=oneshot, average=average, stochastic=True, offset=3)
            lanes = lanes_for(world, dtype)
            sim = [t.clone() for t in xs]
            fn = C.oneshot_simulate if oneshot else C.sra_simulate
            fn(sim, layers, lanes, average, False, True, 5, 2, MIN_LANE)
            exact, bound = O.exact_sum_and_bound(xs, layers, lanes=lanes, min_lane_elems=MIN_LANE, average=average,
                                                 stochastic=True, oneshot=oneshot)
            for r in range(world):
                assert_same(got[r], sim[r], f"rank {r} vs simulator")
            v = got[0].double().numpy()
            ok = np.isfinite(exact) & np.isfinite(v)
            assert (np.abs(v - exact)[ok] <= bound[ok]).all(), "stochastic result outside the exact-sum bound"
