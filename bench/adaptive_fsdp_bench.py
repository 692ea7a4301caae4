"""Adaptive FSDP2 widths on one H100: the sharded estimator, the adapted all-gather, the decision.

    python bench/adaptive_fsdp_bench.py [--iters 50]

(a) ``ops.quantization_error`` on the reduce-scatter input of one GPT-2-medium block (the FSDP2
    shard table of its parameter group at W = 8 and 2, fp32 and bf16, 7 candidates, the own chunk
    skipped): one sharded launch (``chunks=W``) against W-1 per-chunk launches plus their sum.
    Time, and GB/s over the (W-1)·S elements read once.
(b) The ``CGXAllGather`` comm at world 1 on that block's shard, uniform 6-bit table against the
    table ``allocate_bits`` picks at the same budget (a mixed table leaves the specialised kernel).
(c) The host time of one decision on the whole GPT-2-medium FSDP table (one module per block plus
    the root), replayed step by step: group sum of the float64 table plus the copy to the host, the
    allocator, the broadcast of the widths, and their application to the comms' tables.
Prints the card and its power limit first; one JSON line per result. Needs a GPU.
"""
import argparse
import json
import socket
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402
from torch_cgx_b200 import models  # noqa: E402
from torch_cgx_b200.ops.bit_allocation import allocate_bits, layer_wire_bytes  # noqa: E402
from torch_cgx_b200.ops.quantization import quantization_error  # noqa: E402

CANDS = (2, 3, 4, 5, 6, 7, 8)
BUCKET = 512


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def emit(d):
    print(json.dumps(d), flush=True)


def time_events(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def shard_table(module, world, bits):
    """FSDP2's table of one parameter group: dim 0 split into world parts, padded."""
    sizes = []
    for p in module.parameters():
        rows = -(-p.shape[0] // world)
        sizes.append((tuple(p.shape), rows * (p.numel() // p.shape[0])))
    return cgx.fsdp_shard_table(sizes, bits, BUCKET)


def bench_estimator(block, iters):
    for W in (8, 2):
        table = shard_table(block, W, 4)
        rows = [l for l in table if l[2] <= 8]
        S = sum(l[1] for l in table)
        for dtype in (torch.float32, torch.bfloat16):
            x = torch.randn(W * S, device="cuda").to(dtype)
            r = 0

            def one():
                quantization_error(x, rows, CANDS, prescale=1.0 / W, chunks=W, skip_chunk=r)

            def per_chunk():
                parts = [quantization_error(x[c * S:(c + 1) * S], rows, CANDS, prescale=1.0 / W)
                         for c in range(W) if c != r]
                torch.stack(parts).sum(0)

            t1, tn = time_events(one, iters), time_events(per_chunk, iters)
            read = (W - 1) * S * x.element_size()
            emit({"bench": "sharded_estimator", "world": W, "dtype": str(dtype).split(".")[-1], "rows": len(rows),
                  "shard_elems": S, "one_launch_us": round(t1 * 1e6, 1), "per_chunk_us": round(tn * 1e6, 1),
                  "speedup": round(tn / t1, 2), "one_launch_GBps": round(read / t1 / 1e9, 1),
                  "per_chunk_GBps": round(read / tn / 1e9, 1)})


def bench_all_gather(block, iters):
    table = shard_table(block, 1, 6)
    rows = [l for l in table if l[2] <= 8]
    flat = torch.cat([p.detach().reshape(-1) for p in block.parameters()]).cuda()
    err = quantization_error(flat, rows, CANDS).cpu().numpy()
    budget = sum(layer_wire_bytes(l[1], 6, BUCKET) for l in rows)
    picked = iter(allocate_bits(err, [l[1] for l in rows], [BUCKET] * len(rows), CANDS, budget, target_bits=6))
    adapted = [(o, n, next(picked), b) if bits <= 8 else (o, n, bits, b) for (o, n, bits, b) in table]
    out = torch.empty_like(flat)
    res = {}
    for name, layers in (("uniform", table), ("adapted", adapted)):
        comm = cgx.CGXAllGather(6, BUCKET, layers, name)
        res[name] = time_events(lambda: comm(output_tensor=out, input_tensor=flat, group=dist.group.WORLD), iters)
    emit({"bench": "all_gather_world1", "elems": flat.numel(), "widths": sorted({l[2] for l in adapted if l[2] <= 8}),
          "uniform_us": round(res["uniform"] * 1e6, 1), "adapted_us": round(res["adapted"] * 1e6, 1),
          "ratio": round(res["adapted"] / res["uniform"], 2)})


def bench_decision(net, reps):
    tables, comms = [], []
    for m in list(net.blocks) + [net]:
        params = list(m.parameters()) if m is not net else [p for n, p in net.named_parameters()
                                                            if not n.startswith("blocks.")]
        sizes = [(tuple(p.shape), p.numel()) for p in params]
        for bits in (4, 6):
            t = cgx.fsdp_shard_table(sizes, bits, BUCKET)
            comms.append((cgx.CGXAllGather(bits, BUCKET, t), bits))
    rows = [(c, i) for c, _ in comms for i, l in enumerate(c.layers) if l[2] <= 8]
    est = torch.rand(len(rows), len(CANDS), dtype=torch.float64, device="cuda")
    group = dist.group.WORLD
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        table = est.clone().reshape(-1)
        dist.all_reduce(table, group=group)
        table = table.view(-1, len(CANDS)).cpu()
        t1 = time.perf_counter()
        picked, r = [], 0
        for bits in (4, 6):  # one allocation per kind
            mine = [(c, i) for (c, i) in rows if c.bits == bits]
            n = [c.layers[i][1] for c, i in mine]
            budget = sum(layer_wire_bytes(v, bits, BUCKET) for v in n)
            picked += allocate_bits(table[r:r + len(mine)].numpy(), n, [BUCKET] * len(n), CANDS, budget,
                                    [bits] * len(n), target_bits=bits)
            r += len(mine)
        t2 = time.perf_counter()
        choice = torch.tensor(picked, dtype=torch.int32).cuda()
        dist.broadcast(choice, src=0, group=group)
        widths = choice.cpu().tolist()
        t3 = time.perf_counter()
        order = [(c, i) for bits in (4, 6) for (c, i) in rows if c.bits == bits]
        for (c, i), b in zip(order, widths):
            o, n, _, k = c.layers[i]
            c.layers[i] = (o, n, b, k)
        t4 = time.perf_counter()
        cur = [t1 - t0, t2 - t1, t3 - t2, t4 - t3]
        best = cur if best is None or sum(cur) < sum(best) else best
    emit({"bench": "decision_host", "rows": len(rows), "comms": len(comms), "group_sum_ms": round(best[0] * 1e3, 3),
          "allocate_ms": round(best[1] * 1e3, 3), "broadcast_ms": round(best[2] * 1e3, 3),
          "apply_ms": round(best[3] * 1e3, 3), "total_ms": round(sum(best) * 1e3, 3)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "adaptive_fsdp_bench needs a GPU"
    torch.cuda.set_device(0)
    emit({"card": card()})
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        torch.manual_seed(0)
        net = models.gpt2_medium()
        block = net.blocks[0].cuda()
        bench_estimator(block, args.iters)
        bench_all_gather(block, args.iters)
        bench_decision(net, 20)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
