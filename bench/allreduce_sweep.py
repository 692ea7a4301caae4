#!/usr/bin/env python
"""Compressed-allreduce bandwidth sweep (BASELINE.json configs[4]): message sizes
1 KB - 1 GB x bits {2,4,8,32} on N GPUs, cgx fused P2P kernel vs stock NCCL
ncclAllReduce on the same box.  Device-timed with CUDA events on the launching
stream around a batch of back-to-back calls (nccl-tests style) over a rotating
set of buffers larger than L2, MAX over ranks, median of 3 repetitions.

  torchrun --nproc-per-node N bench/allreduce_sweep.py --out gpurun_out/sweep_N.json
  torchrun --nproc-per-node N bench/allreduce_sweep.py --op reduce_scatter   # cgx.reduce_scatter_tensor
                                                                            # vs ncclReduceScatter
  torchrun --nproc-per-node N bench/allreduce_sweep.py --op all_gather       # cgx.all_gather_into_tensor
                                                                            # vs ncclAllGather
  torchrun --nproc-per-node N bench/allreduce_sweep.py --op all_to_all       # cgx.all_to_all_single
                                                                            # vs dist.all_to_all_single (NCCL)
With --op all_to_all the message is a rank's input of W equal chunks.
With --op reduce_scatter the message is the input of W shards, with --op all_gather the gathered
output of W shards; NCCL's bus bandwidth is then algbw * (W-1)/W, and wire_bytes_per_rank counts
the packed chunks this rank sends.

Reported per row:
  time_us        median device time of one allreduce (max over ranks)
  algbw_gbs      message bytes / time
  busbw_gbs      algbw * 2(W-1)/W          (NCCL's "bus bandwidth" of the *uncompressed* message)
  wire_gbs       bytes this rank actually pushed over NVLink / time (packed bytes, per direction)
  speedup_vs_nccl
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402
from torch_cgx_b200.utils.clocks import ClockSampler  # noqa: E402


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def time_allreduce(fn, bufs, iters, warmup, dev):
    """nccl-tests style: `iters` calls enqueued back to back between two CUDA events on the
    launching stream (no host sync inside), each call on a different buffer of a rotating set
    that is larger than L2 (or 64 buffers for tiny messages), MAX over ranks."""
    nb = len(bufs)
    for i in range(warmup):
        fn(bufs[i % nb])
    torch.cuda.synchronize()
    reps = []
    for _ in range(3):
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            fn(bufs[i % nb])
        e1.record()
        torch.cuda.synchronize()
        reps.append(e0.elapsed_time(e1) * 1e3 / iters)
    t = torch.tensor(reps, device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)  # max over ranks, per repetition
    return median(t.tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/sweep.json")
    ap.add_argument("--min-kb", type=int, default=1)
    ap.add_argument("--max-mb", type=int, default=1024)
    ap.add_argument("--bits", default="2,4,8,32")
    ap.add_argument("--dtype", default="float32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--bucket-size", type=int, default=512)
    ap.add_argument("--sizes", default="", help="explicit comma-separated sizes in KB (overrides min/max)")
    ap.add_argument("--op", default="allreduce", choices=["allreduce", "reduce_scatter", "all_gather", "all_to_all"])
    ap.add_argument("--with-nccl-sra", action="store_true",
                    help="also time the reference-structure path: SRA over NCCL send/recv + separate kernels")
    args = ap.parse_args()

    rank, world, local = cgx.map_launcher_env()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    nccl = dist.new_group(backend="nccl")
    dtype = getattr(torch, args.dtype)
    es = torch.empty((), dtype=dtype).element_size()
    os.environ["CGX_COMPRESSION_BUCKET_SIZE"] = str(args.bucket_size)
    be = cgx.get_backend()
    nccl_sra = None
    if args.with_nccl_sra:
        # a second cgx group whose intra-node transport is NCCL send/recv with standalone
        # quantize/dequantize kernels: the structure of the reference's NCCL_Reduce
        # (/root/reference/src/common/nccl_reduce.cc:103-198), i.e. "a path that only calls NCCL"
        os.environ["CGX_INNER_COMMUNICATOR_TYPE"] = "NCCL"
        nccl_sra = dist.new_group(backend="cgx")
        os.environ.pop("CGX_INNER_COMMUNICATOR_TYPE")

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    sizes = []
    s = args.min_kb << 10
    while s <= (args.max_mb << 20):
        sizes.append(s)
        s *= 4
    if args.sizes:
        sizes = [int(x) << 10 for x in args.sizes.split(",")]
    rs = args.op in ("reduce_scatter", "all_gather", "all_to_all")  # one shard per rank: the message is W shards
    bus = (world - 1) / world if rs else 2 * (world - 1) / world
    if args.op == "reduce_scatter":
        sizes = [s for s in sizes if s // es >= world]
        outs = {}

        def out_for(x):
            return outs.setdefault(x.numel(), torch.empty(x.numel() // world, dtype=x.dtype, device=dev))

        def nccl_op(x):
            dist.reduce_scatter_tensor(out_for(x), x, group=nccl)

        def cgx_op(x, bits):
            cgx.reduce_scatter_tensor(out_for(x), x, bits=bits, bucket_size=args.bucket_size)
    elif args.op == "all_gather":
        sizes = [s for s in sizes if s // es >= world]
        outs = {}

        def out_for(x):  # x is the gathered message; rank r's input is its chunk r
            return outs.setdefault(x.numel(), torch.empty(x.numel(), dtype=x.dtype, device=dev))

        def nccl_op(x):
            s = x.numel() // world
            dist.all_gather_into_tensor(out_for(x), x[rank * s:(rank + 1) * s], group=nccl)

        def cgx_op(x, bits):
            s = x.numel() // world
            cgx.all_gather_into_tensor(out_for(x), x[rank * s:(rank + 1) * s], bits=bits,
                                       bucket_size=args.bucket_size)
    elif args.op == "all_to_all":
        sizes = [s for s in sizes if s // es >= world]
        outs = {}

        def out_for(x):
            return outs.setdefault(x.numel(), torch.empty(x.numel(), dtype=x.dtype, device=dev))

        def nccl_op(x):
            dist.all_to_all_single(out_for(x), x, group=nccl)

        def cgx_op(x, bits):
            cgx.all_to_all_single(out_for(x), x, bits=bits, bucket_size=args.bucket_size)
    else:
        def nccl_op(x):
            dist.all_reduce(x, group=nccl)

        def cgx_op(x, bits):
            dist.all_reduce(x)
    rows = []
    for nbytes in sizes:
        n = nbytes // es // world * world if rs else nbytes // es
        # rotating buffers: total > 2x L2 (50 MB) so no call finds its input in cache
        nbuf = max(2, min(64, (288 << 20) // nbytes + 1))
        bufs = [torch.randn(n, device=dev).to(dtype) for _ in range(nbuf)]
        iters = args.iters if nbytes <= (64 << 20) else max(6, args.iters // 3)
        t_nccl = time_allreduce(nccl_op, bufs, iters, args.warmup, dev)
        row_base = {"op": args.op, "bytes": nbytes, "dtype": args.dtype, "world": world}
        r = dict(row_base, impl="nccl", bits=32, time_us=round(t_nccl, 2),
                 algbw_gbs=round(nbytes / t_nccl / 1e3, 2), busbw_gbs=round(nbytes / t_nccl / 1e3 * bus, 2))
        rows.append(r)
        if rank == 0:
            print(json.dumps(r), flush=True)
        for bits in [int(b) for b in args.bits.split(",")]:
            os.environ["CGX_COMPRESSION_QUANTIZATION_BITS"] = str(bits)
            for x in bufs:
                x.normal_()
            be.reset_stats()
            t = time_allreduce(lambda x: cgx_op(x, bits), bufs, iters, args.warmup, dev)
            st = be.stats()
            wire_per_call = st[3] / max(1, st[0])
            r = dict(row_base, impl="cgx", bits=bits, time_us=round(t, 2), algbw_gbs=round(nbytes / t / 1e3, 2),
                     busbw_gbs=round(nbytes / t / 1e3 * bus, 2),
                     wire_bytes_per_rank=int(wire_per_call), wire_gbs=round(wire_per_call / t / 1e3, 2),
                     kernel_launches_per_call=round(st[1] / max(1, st[0]), 2),
                     speedup_vs_nccl=round(t_nccl / t, 3))
            rows.append(r)
            if rank == 0:
                print(json.dumps(r), flush=True)
            if nccl_sra is not None and not rs and bits < 32 and nbytes >= 4096:
                t2 = time_allreduce(lambda x: dist.all_reduce(x, group=nccl_sra), bufs, iters, args.warmup, dev)
                r = dict(row_base, impl="cgx_sra_over_nccl_sendrecv", bits=bits, time_us=round(t2, 2),
                         algbw_gbs=round(nbytes / t2 / 1e3, 2),
                         busbw_gbs=round(nbytes / t2 / 1e3 * 2 * (world - 1) / world, 2),
                         speedup_vs_nccl=round(t_nccl / t2, 3), fused_speedup_over_this=round(t2 / t, 3))
                rows.append(r)
                if rank == 0:
                    print(json.dumps(r), flush=True)
        del bufs
    if rank == 0:
        clocks = sampler.stop()
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps({"world": world, "lanes": be.lanes(), "heap": be.heap_kind(),
                                              "nvls_multicast": be.uses_multicast(), "clocks": clocks, "rows": rows,
                                              "timing": "CUDA events around `iters` back-to-back calls on rotating buffers (> 2x L2 in total), max over ranks, median of 3 repetitions"}, indent=1))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
