#!/usr/bin/env python
"""Single-GPU proxy of a W-GPU allreduce: W *virtual* ranks (W heaps, W streams, W concurrent
kernels) on ONE device. With `mb` MB per virtual rank the GPU executes exactly the phase A / B / C
work of ONE real rank of a (W * mb) MB allreduce on W GPUs -- minus NVLink -- so it isolates the
compute / HBM efficiency of the fused kernel at W > 1 without multi-GPU time.
The same for the compressed reduce-scatter (rows with "op": "reduce_scatter"): `mb` MB of input
per virtual rank, one shard of mb / W MB out; and for the compressed all-gather (rows with
"op": "all_gather"): one shard of mb / W MB in per virtual rank, `mb` MB out.
Reports the slope between two sizes (harness overhead cancels)."""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402
from torch_cgx_b200.utils.clocks import ClockSampler  # noqa: E402

C = cgx._C


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--bits", default="4")
    ap.add_argument("--bucket", type=int, default=512)
    ap.add_argument("--mbs", default="8,32")
    ap.add_argument("--out", default="gpurun_out/virtual_world.json")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    W = args.world
    lanes = 264 // W
    rows = []
    sampler = ClockSampler(0).start()
    for bits in [int(b) for b in args.bits.split(",")]:
        res = {}
        for mb in [int(x) for x in args.mbs.split(",")]:
            n = (mb << 20) // 4
            layers = [(0, n, bits, args.bucket)]
            g = C.LocalSraGroup(W, lanes, n * 4 // W * 2 + (1 << 20), 20000, 4096)
            xs = [torch.randn(n, device=dev) for _ in range(W)]
            g.allreduce(xs, layers)
            torch.cuda.synchronize()
            g.check()
            res[mb] = timeit(lambda: g.allreduce(xs, layers))
            del g, xs
        mbs = sorted(res)
        slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])  # us per MB per virtual rank
        row = {"world": W, "bits": bits, "bucket": args.bucket, "lanes_per_rank": lanes,
               "times_us": {str(k): round(v, 1) for k, v in res.items()},
               "us_per_equivalent_64MB_allreduce": round(slope * 64 / W, 1),
               "note": "slope * (64 MB / W): device work of one real rank of a 64 MB allreduce on W GPUs, NVLink excluded"}
        rows.append(row)
        print(json.dumps(row), flush=True)
        res = {}
        for mb in [int(x) for x in args.mbs.split(",")]:
            n = (mb << 20) // 4 // W * W
            shard = [(0, n // W, bits, args.bucket)]
            g = C.LocalSraGroup(W, lanes, n * 4 // W * 2 + (1 << 20), 20000, 4096)
            xs = [torch.randn(n, device=dev) for _ in range(W)]
            outs = [torch.empty(n // W, device=dev) for _ in range(W)]
            g.reduce_scatter(xs, outs, shard)
            torch.cuda.synchronize()
            g.check()
            res[mb] = timeit(lambda: g.reduce_scatter(xs, outs, shard))
            del g, xs, outs
        slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])
        row = {"op": "reduce_scatter", "world": W, "bits": bits, "bucket": args.bucket, "lanes_per_rank": lanes,
               "times_us": {str(k): round(v, 1) for k, v in res.items()},
               "us_per_equivalent_64MB_reduce_scatter": round(slope * 64 / W, 1),
               "note": "slope * (64 MB / W): device work of one real rank of a 64 MB-input reduce-scatter on W GPUs, "
                       "NVLink excluded"}
        rows.append(row)
        print(json.dumps(row), flush=True)
        res = {}
        for mb in [int(x) for x in args.mbs.split(",")]:
            n = (mb << 20) // 4 // W * W
            shard = [(0, n // W, bits, args.bucket)]
            g = C.LocalSraGroup(W, lanes, n * 4 // W * 2 + (1 << 20), 20000, 4096)
            xs = [torch.randn(n // W, device=dev) for _ in range(W)]
            outs = [torch.empty(n, device=dev) for _ in range(W)]
            g.all_gather(xs, outs, shard)
            torch.cuda.synchronize()
            g.check()
            res[mb] = timeit(lambda: g.all_gather(xs, outs, shard))
            del g, xs, outs
        slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])
        row = {"op": "all_gather", "world": W, "bits": bits, "bucket": args.bucket, "lanes_per_rank": lanes,
               "times_us": {str(k): round(v, 1) for k, v in res.items()},
               "us_per_equivalent_64MB_all_gather": round(slope * 64 / W, 1),
               "note": "slope * (64 MB / W): device work of one real rank of a 64 MB-output all-gather on W GPUs, "
                       "NVLink excluded"}
        rows.append(row)
        print(json.dumps(row), flush=True)
    clocks = sampler.stop()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps({"clocks": clocks, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
