#!/usr/bin/env python
"""The cross-node stage of the compressed all-to-all (DESIGN §2.13f) at MoE shapes.

One GPU (default): rank 0 of W ranks in nodes of L holds `--rows` bf16 rows of H elements, split
equally over the W destinations. Its W - L remote chunks are

  pack:    one launch (C.a2a_pack) quantizes all of them into one send buffer
  unpack:  one launch (C.a2a_unpack) decodes a buffer of as many received chunks into their rows
  generic: the generic reducer's per-chunk path on the same chunks, one quantize and one dequantize
           launch per chunk through a one-layer plan (C.quantize / C.dequantize)

CUDA events around each arm, arms alternating, medians over --iters after --warmup. HBM bytes from
shapes: pack reads the remote rows (n es) and writes their records; unpack reads the records and
writes the rows. The achieved rate is bytes over the median time, printed beside the H100 SXM data
sheet's 3.35 TB/s. The card's name and power limit are printed with the numbers.

Under torchrun across nodes (--dist, CGX_LOCAL_SIZE set to the ranks per node), every rank times
cgx.all_to_all_single on a cgx group against dist.all_to_all_single on NCCL at the same shapes.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402

C = cgx._C
HBM_TBS = 3.35


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def timed(fns, iters, warmup):
    """Median milliseconds of each callable, alternating them."""
    for _ in range(warmup):
        for f in fns:
            f()
    times = [[] for _ in fns]
    for _ in range(iters):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b))
    return [sorted(t)[len(t) // 2] for t in times]


def one_gpu(args):
    name, power = gpu_info()
    print(f"# {name}, power limit {power}", flush=True)
    H, dt = args.H, torch.bfloat16
    for W in args.worlds:
        L = args.local
        rows = args.rows // W * W
        counts = [rows // W * H] * W
        x = torch.randn(rows * H, device="cuda", dtype=dt)
        out = torch.empty_like(x)
        remote = [q for q in range(W) if q // L != 0]
        n_remote = sum(counts[q] for q in remote)
        for bits in args.bits:
            b = 8 if isinstance(bits, str) else bits
            wire, region, total = C.a2a_remote_wire(counts, 0, L, bits, args.bucket, 2)
            buf = C.a2a_pack(x, counts, 0, L, bits, args.bucket)
            offs = [sum(counts[:q]) for q in range(W)]
            layers = lambda q: [(0, counts[q], b, args.bucket)]  # noqa: E731

            def pack():
                C.a2a_pack(x, counts, 0, L, bits, args.bucket, out=buf)

            def unpack():
                C.a2a_unpack(buf, out, counts, 0, L, bits, args.bucket)

            def generic():
                for q in remote:
                    w = C.quantize(x[offs[q]:offs[q] + counts[q]], layers(q))
                    C.dequantize(w, out[offs[q]:offs[q] + counts[q]], layers(q))

            arms = [pack, unpack] + ([generic] if not isinstance(bits, str) else [])
            ms = timed(arms, args.iters, args.warmup)
            wire_bytes = sum(wire)
            moved = n_remote * 2 + wire_bytes
            res = dict(world=W, local=L, rows=rows, H=H, bits=bits, bucket=args.bucket, remote_elems=n_remote,
                       wire_bytes=wire_bytes, hbm_bytes_per_kernel=moved,
                       pack_ms=round(ms[0], 4), unpack_ms=round(ms[1], 4),
                       pack_tbs=round(moved / ms[0] / 1e9, 3), unpack_tbs=round(moved / ms[1] / 1e9, 3),
                       hbm_peak_tbs=HBM_TBS, gpu=name, power_limit=power)
            if len(ms) > 2:
                res["generic_quantize_dequantize_ms"] = round(ms[2], 4)
                res["generic_over_pack_plus_unpack"] = round(ms[2] / (ms[0] + ms[1]), 2)
            else:
                res["generic_quantize_dequantize_ms"] = "not measured (C.quantize has no FP8 form)"
            print(json.dumps(res), flush=True)
            del buf


def distributed(args):
    import torch.distributed as dist

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dist.init_process_group("cgx")
    nccl = dist.new_group(backend="nccl")
    H, rows = args.H, args.rows // world * world
    x = torch.randn(rows, H, device="cuda", dtype=torch.bfloat16)
    out = torch.empty_like(x)
    for bits in args.bits:
        ms = timed([lambda: cgx.all_to_all_single(out, x, bits=bits, bucket_size=args.bucket),
                    lambda: dist.all_to_all_single(out, x, group=nccl)], args.iters, args.warmup)
        if rank == 0:
            print(json.dumps(dict(world=world, rows=rows, H=H, bits=bits, cgx_ms=round(ms[0], 4),
                                  nccl_ms=round(ms[1], 4), gpu=gpu_info()[0], power_limit=gpu_info()[1])), flush=True)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rows", type=int, default=32768)
    ap.add_argument("--H", type=int, default=7168)
    ap.add_argument("--worlds", type=int, nargs="+", default=[16, 32, 64])
    ap.add_argument("--local", type=int, default=8)
    ap.add_argument("--bits", nargs="+", default=["4", "8", "e4m3"])
    ap.add_argument("--bucket", type=int, default=512)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dist", action="store_true", help="run under torchrun across nodes against NCCL")
    args = ap.parse_args()
    args.bits = [b if b.startswith("e") else int(b) for b in args.bits]
    if not torch.cuda.is_available():
        sys.exit("a2a_nodes_bench.py needs a GPU")
    distributed(args) if args.dist else one_gpu(args)


if __name__ == "__main__":
    main()
