"""The generic reducers' device path (CudaBackend: quantize / accumulate / quantize_f32 /
dequantize item kernels) with W virtual ranks on ONE GPU (C.LocalReducerGroup), against the same
reducers on host memory and the independent references, bit for bit and NaN-aware.

With recording on, every message of every hop is compared byte for byte between the two backends,
so a mismatch names the exchange, the sender and the receiver; runs with recording off (the default)
check that the transport alone orders every device copy. Every rank's tensor is a view at
element offset 1, 3 or 5 of a sentinel-filled buffer whose guard bands must stay intact. Covered
besides the shared cases: stochastic rounding (Philox keyed by element index on both sides), the
width-specialised kernels (uniform 2, 4, 8 bits) and the generic one, the 1024-element slice path,
full slices of 8/16/32/256-element buckets, a grid-stride loop that wraps past one resident wave, and
repeated calls on one group with alternating tables. All parameters are fixed lists."""
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _a2a_cases import counts as a2a_counts, inputs as a2a_inputs, outputs as a2a_outputs
from _reducer_cases import (DT_CODE, OPS, check_many_layouts, config_id, configs, group_for, make_case, reference,
                            run_op)

pytestmark = pytest.mark.gpu
C = cgx._C
CONFIGS = configs()
GUARD = 64
SENTINEL = -7.25  # exact in every dtype


def guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device="cuda")
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def assert_guards(buf, offset, n, what):
    b = buf.cpu()
    assert_same(b[:offset], torch.full((offset,), SENTINEL, dtype=b.dtype), f"{what}: elements before the view")
    assert_same(b[offset + n:], torch.full((GUARD,), SENTINEL, dtype=b.dtype), f"{what}: elements after the view")


def chunk_record_bytes(plan, c, elsize):
    """Byte offsets of chunk c's wire record that carry data: per block the bucket metas, the
    packed groups, or the raw values. The 16-byte alignment padding after each of them is not part
    of the record: the host backend writes zeros there, the device kernels leave it untouched (a
    reused scratch buffer keeps older bytes), and no decoder reads it."""
    keep = []
    lf, blocks = plan["lane_first"], plan["blocks"].tolist()
    for _, n, bits, bucket, off in blocks[lf[c]:lf[c + 1]]:
        if bits >= 32:
            keep.append(torch.arange(off, off + n * elsize))
            continue
        nb = -(-n // bucket)
        groups = n // bucket * -(-bucket // 8) + -(-(n % bucket) // 8)
        keep.append(torch.arange(off, off + nb * 8))
        pay = off + (nb * 8 + 15) // 16 * 16
        keep.append(torch.arange(pay, pay + groups * bits))
    return torch.cat(keep) if keep else torch.zeros(0, dtype=torch.long)


def record_bytes(op, layers, W, dtype, skip_incomplete, e, src):
    """Data byte offsets of the message `src` sends at exchange `e` (which chunk it carries follows
    from each reducer's schedule)."""
    es = torch.empty(0, dtype=dtype).element_size()
    if op.startswith("BCAST"):
        p = C.build_plan(layers, world=1, lanes=1, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete)
        return chunk_record_bytes(p, 0, es)
    p = C.build_plan(layers, world=W, lanes=1, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete)
    if op == "ALLTOALL":  # the whole wire image, chunk c at row * c
        row = (p["max_chunk_wire"] + 255) // 256 * 256
        return torch.cat([chunk_record_bytes(p, c, es) + row * c for c in range(W)])
    return None


def message_chunk(op, W, e, src, dst):
    if op == "SRA":  # phase 1 carries the receiver's chunk, phase 2 the sender's
        return dst if e == 0 else src
    return (src - e) % W if e < W - 1 else (src + 1 - (e - (W - 1))) % W  # Ring


def compare_messages(op, hm, dm, layers, W, dtype, skip_incomplete):
    assert [m[:3] for m in dm] == [m[:3] for m in hm], f"{op}: the device moved other messages than the host"
    es = torch.empty(0, dtype=dtype).element_size()
    plan = C.build_plan(layers, world=W, lanes=1, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete)
    for (e, src, dst, hb), (_, _, _, db) in zip(hm, dm):
        assert db.numel() == hb.numel()
        keep = record_bytes(op, layers, W, dtype, skip_incomplete, e, src)
        if keep is None:
            c = message_chunk(op, W, e, src, dst)
            assert hb.numel() == plan["chunk_wire_bytes"][c], f"{op}: exchange {e} from {src} is not chunk {c}"
            keep = chunk_record_bytes(plan, c, es)
        assert_same(db[keep], hb[keep], f"{op}: message of exchange {e} from rank {src} to rank {dst}")


def compare_backends(op, ins, layers, *, offset=1, groups=None, ref=True, record=True, **kw):
    """Run `op` on the host and on the device; results and (recording on) every message must be
    identical. `groups`: a (host, device) pair of groups reused across calls."""
    W = len(ins)
    hg, dg = groups or (group_for(op, W, record=record), group_for(op, W, record=record))
    host = [t.clone() for t in ins]
    run_op(hg, op, host, layers, **kw)
    bufs = [guarded(t, offset) for t in ins]
    views = [v for _, v in bufs]
    run_op(dg, op, views, layers, **kw)
    torch.cuda.synchronize()
    for r, (buf, _) in enumerate(bufs):
        assert_guards(buf, offset, ins[0].numel(), f"{op} rank {r}")
    if record:
        compare_messages(op, hg.messages(), dg.messages(), layers, W, ins[0].dtype, kw.get("skip_incomplete", False))
    else:
        assert hg.messages() == [] and dg.messages() == []
    assert dg.bytes_sent() == hg.bytes_sent()
    got = [v.cpu() for v in views]
    for r in range(W):
        assert_same(got[r], host[r], f"{op} rank {r}: device vs host")
    if ref:
        kw.pop("stochastic", None)
        expect = reference(op, ins, layers, **{k: v for k, v in kw.items() if k in ("average", "skip_incomplete")})
        for r in range(W):
            assert_same(got[r], expect[r], f"{op} rank {r}: device vs reference")
    return got


def op_kwargs(op, average, skip_incomplete):
    kw = dict(skip_incomplete=skip_incomplete)
    if not op.startswith("BCAST"):
        kw["average"] = average
    return kw


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("c", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_device_reducers_match_host_and_reference(c, op):
    ins, layers = make_case(c)
    compare_backends(op, ins, layers, offset=(1, 3, 5)[c["seed"] % 3],
                     **op_kwargs(op, c["average"], c["skip_incomplete"]))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("c", [c for c in CONFIGS if c["dtype"] != torch.float16 and c["world"] in (2, 3, 5, 16)],
                         ids=config_id)
def test_device_reducers_without_recording(c, op):
    # the default: nothing copies a message to the host, so only the loopback transport itself orders
    # each device copy before the receiver's next kernel and before the sender's next write to its buffer
    ins, layers = make_case(c)
    compare_backends(op, ins, layers, offset=(1, 3, 5)[c["seed"] % 3], record=False,
                     **op_kwargs(op, c["average"], c["skip_incomplete"]))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("world,dtype", [(2, torch.float32), (3, torch.bfloat16), (5, torch.float16),
                                         (16, torch.float32)])
def test_device_stochastic_matches_host(world, dtype, op):
    layers = [(0, 37, 32, 512), (37, 12_000, 2, 512), (12_037, 5000, 5, 100), (17_037, 3001, 4, 1024)]
    g = torch.Generator().manual_seed(world)
    ins = [(torch.randn(20_038, generator=g) * (r + 1)).to(dtype) for r in range(world)]
    compare_backends(op, ins, layers, offset=3, ref=False, stochastic=True, seed=123, seq=world,
                     **op_kwargs(op, True, world % 2 == 1))


@pytest.mark.parametrize("bucket", [8, 16, 32, 256, 1024, 100])
@pytest.mark.parametrize("bits", [2, 4, 8, 3])
def test_device_width_and_slice_variants(bits, bucket):
    # one compressed width: the KB-specialised kernels (2, 4, 8) and the generic one (3); 1024-element
    # buckets everywhere: the 1024-element slice (GPL = 4); 8/16/32/256: full slices of small buckets
    layers = [(0, 37, 32, 512), (37, 40 * 1024 + bucket // 2, bits, bucket)]
    total = 37 + 40 * 1024 + bucket // 2
    plan = C.build_plan(layers, world=3, lanes=1, dtype=0)
    assert plan["uniform_bits"] == bits
    assert plan["slice_elems"] == (1024 if bucket == 1024 else 512)
    items = plan["items"]
    if bucket in (8, 16, 32, 256):
        lg = {8: 0, 16: 1, 32: 2, 256: 5}[bucket]
        assert int(((items[:, 3] == 0) & (items[:, 4] == lg)).sum()) >= 3, "no full slices to test"
    g = torch.Generator().manual_seed(bits * bucket)
    for op in OPS:
        ins = [(torch.randn(total, generator=g) * (r + 1)) for r in range(3)]
        compare_backends(op, ins, layers, offset=(1, 3, 5)[bits % 3], **op_kwargs(op, bits % 2 == 0, False))


@pytest.mark.parametrize("op", ["SRA", "RING", "ALLTOALL", "BCAST_LAST"])
def test_device_grid_wraps_past_one_wave(op):
    # about 4100 512-element items per chunk: more warps than one resident wave (3 CTAs of 8 warps per SM)
    n = (1 << 22) + 333
    layers = [(0, 333, 32, 512), (333, 1 << 22, 4, 512)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plan = C.build_plan(layers, world=2, lanes=1, dtype=0)
    assert plan["item_first"][2] - plan["item_first"][1] > sms * 3 * 8
    g = torch.Generator().manual_seed(2)
    ins = [torch.randn(n, generator=g) * (r + 1) for r in range(2)]
    compare_backends(op, ins, layers, offset=5, ref=op in ("SRA", "BCAST_LAST"),
                     **op_kwargs(op, True, False))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("record", [True, False], ids=["recorded", "unrecorded"])
def test_device_repeated_calls_with_alternating_tables(record, op):
    # one group per backend for the whole sequence: plan cache hits and misses, tables uploaded on a
    # plan's first use only (a, a and big, big; all-to-all also uses a raw plan inside each call) and
    # scratch buffers that grow between calls
    W, dtype = 3, torch.bfloat16
    a = [(0, 37, 32, 512), (37, 9000, 4, 512)]
    b = [(0, 4000, 8, 64), (4000, 5037, 2, 1024)]
    big = [(0, 37, 32, 512), (37, 60_000, 3, 100)]
    groups = (group_for(op, W, record=record), group_for(op, W, record=record))
    g = torch.Generator().manual_seed(7)
    for i, layers in enumerate([a, a, b, a, big, big, a, b]):
        total = max(off + m for off, m, _, _ in layers)
        ins = [(torch.randn(total, generator=g) * (r + 1)).to(dtype) for r in range(W)]
        compare_backends(op, ins, layers, offset=(1, 3, 5)[i % 3], groups=groups, record=record,
                         **op_kwargs(op, i % 2 == 0, False))


def test_device_plan_cache_is_bounded_across_many_layouts():
    check_many_layouts(3, "cuda")


def test_device_interleaved_collectives_upload_each_table_once():
    # reduce-scatter, all-to-all with fixed splits and all-to-all with new splits on one device group,
    # bitwise the host group's; after the first round the fixed calls find their tables uploaded
    W, dtype = 4, torch.bfloat16
    shard = [(0, 37, 32, 512), (37, 3000, 4, 64)]
    S = 3037
    fixed = [[1500 + 100 * q + 10 * r for r in range(W)] for q in range(W)]
    hg, dg = C.LocalReducerGroup(W, "SRA", 20_000), C.LocalReducerGroup(W, "SRA", 20_000)
    g = torch.Generator().manual_seed(3)

    def reduce_scatter(i):
        ins = [(torch.randn(W * S, generator=g) * (r + 1)).to(dtype) for r in range(W)]
        host = [torch.empty(S, dtype=dtype) for _ in range(W)]
        hg.reduce_scatter(ins, host, shard, True, False, True, 5, i)
        got = [torch.empty(S, dtype=dtype, device="cuda") for _ in range(W)]
        dg.reduce_scatter([t.cuda() for t in ins], got, shard, True, False, True, 5, i)
        return host, got

    def all_to_all(c, i):
        xs = a2a_inputs(c, dtype, i)
        host = a2a_outputs(c, dtype)
        hg.all_to_all(xs, host, c, bits=3, bucket_size=100, stochastic=True, seed=5, seq=i)
        got = a2a_outputs(c, dtype, device="cuda")
        dg.all_to_all([x.cuda() for x in xs], got, c, bits=3, bucket_size=100, stochastic=True, seed=5, seq=i)
        return host, got

    for i in range(4):
        for what, run in [("reduce_scatter", lambda: reduce_scatter(i)),
                          ("fixed splits", lambda: all_to_all(fixed, i)),
                          ("new splits", lambda: all_to_all(a2a_counts(W, "uneven", 2000, seed=i), i))]:
            before = [dg.plan_uploads(r) for r in range(W)]
            host, got = run()
            torch.cuda.synchronize()
            for r in range(W):
                assert_same(got[r].cpu(), host[r], f"round {i} {what} rank {r}: device vs host")
            uploads = [dg.plan_uploads(r) - before[r] for r in range(W)]
            if i == 0 or what == "new splits":
                assert sum(uploads) > 0, f"round {i} {what}: no table uploaded"
            else:
                assert uploads == [0] * W, f"round {i} {what}: tables uploaded again {uploads}"
