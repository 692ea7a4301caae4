#!/usr/bin/env python
"""Single-GPU proxy of a W-GPU allreduce: W *virtual* ranks (W heaps, W streams, W concurrent
kernels) on ONE device. With `mb` MB per virtual rank the GPU executes exactly the phase A / B / C
work of ONE real rank of a (W * mb) MB allreduce on W GPUs -- minus NVLink -- so it isolates the
compute / HBM efficiency of the fused kernel at W > 1 without multi-GPU time.
The same for the compressed reduce-scatter (rows with "op": "reduce_scatter"): `mb` MB of input
per virtual rank, one shard of mb / W MB out; and for the compressed all-gather (rows with
"op": "all_gather"): one shard of mb / W MB in per virtual rank, `mb` MB out.
Reports the slope between two sizes (harness overhead cancels).

--op all_to_all times the compressed all-to-all (a2a_kernel) instead: `mb` MB of input per virtual
rank in W chunks, with equal splits and with skewed ones (chunk q -> r gets a share proportional to
1 + (r - q) mod W, so every rank still sends and receives `mb` MB but pairs differ up to W : 1),
next to the reduce-scatter (rs_kernel) of the same `mb` MB input per rank, same dtype, bits and
bucket. Both move the same packed bytes; the reduce-scatter also accumulates. Its --bits may name
the FP8 wire formats, e4m3 and e5m2 (and e4m3_pow2 / e5m2_pow2, their power-of-two-scale twins, and
e4m3_sr / e5m2_sr, which round stochastically),
which move the bytes of bits 8 (the reduce-scatter row next to them runs at bits 8).

--op ag_codes times the FP8 all-gather's codes output (e4m3, bf16, H in --hiddens, buckets of 128
and of H, --rows rows of H per virtual rank) two ways, the arms alternating in one run:
  (c) the decoded call, all_gather_into_tensor(out, x, bits="e4m3"), then the FP8 quantize a caller
      writes in torch (amax, scale, cast) to the same scale layout;
  (d) the codes call, all_gather_into_tensor(codes, x, bits="e4m3", output_scales=scales).
Each arm's median over --iters is taken --repeats times (min, median and max reported). HBM bytes
are computed from shapes, all virtual ranks together: every rank reads its shard (S es), writes its
record to W - 1 peers and they read it (2 (W - 1) (S + 8 S / B)); (d) writes W S codes and W S / B
fp32 scales; (c) writes the W S decoded values, and its quantize reads them once and writes the same
codes and scales. The row asserts that (d) decoded, T(code * scale), equals (c)'s decoded output.

--op sra --bits may name them too: every row then runs at bits 8 with that format, the allreduce's
included. The allreduce also gets a one-shot row ("kernel": "oneshot") at --oneshot-kbs KB per
virtual rank, the sizes the engine sends through the one-shot kernel. Every row is timed for each of
--dtypes."""
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
    ap.add_argument("--op", default="sra", choices=["sra", "all_to_all", "ag_codes"],
                    help="sra: allreduce, reduce-scatter and all-gather rows; all_to_all: a2a next to rs_kernel; "
                         "ag_codes: the all-gather's FP8 codes output against decode + torch quantize")
    ap.add_argument("--hiddens", default="4096,7168", help="ag_codes: row lengths H")
    ap.add_argument("--rows", type=int, default=1024, help="ag_codes: rows of H per virtual rank's shard")
    ap.add_argument("--repeats", type=int, default=3, help="ag_codes: medians taken per arm")
    ap.add_argument("--iters", type=int, default=10, help="ag_codes: timed calls per arm and repeat")
    ap.add_argument("--dtypes", default="float32", help="comma-separated dtypes")
    ap.add_argument("--oneshot-kbs", default="256,1024", help="one-shot allreduce sizes, KB per virtual rank")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    W = args.world
    lanes = 264 // W
    rows = []
    sampler = ClockSampler(0).start()
    if args.op in ("all_to_all", "ag_codes"):
        rows = (all_to_all_rows if args.op == "all_to_all" else ag_codes_rows)(args, dev, W, lanes)
        clocks = sampler.stop()
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps({"clocks": clocks, "rows": rows}, indent=1))
        return
    for dtype in [getattr(torch, d) for d in args.dtypes.split(",")]:
        for bits in [a2a_bits(b) for b in args.bits.split(",")]:
            rows += sra_rows(args, dev, W, lanes, dtype, bits)
    clocks = sampler.stop()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps({"clocks": clocks, "rows": rows}, indent=1))


def sra_rows(args, dev, W, lanes, dtype, bits):
    """the allreduce (SRA and one-shot), reduce-scatter and all-gather rows of one dtype and --bits
    entry; an FP8 format moves the records of bits 8"""
    rows = []
    fmt = bits if isinstance(bits, str) else None
    width = 8 if fmt else bits
    es = torch.empty(0, dtype=dtype).element_size()
    dt = str(dtype).replace("torch.", "")
    mbs = sorted(int(x) for x in args.mbs.split(","))
    res = {}
    for mb in mbs:
        n = (mb << 20) // es
        layers = [(0, n, width, args.bucket)]
        g = C.LocalSraGroup(W, lanes, n * es // W * 2 + (1 << 20), 20000, 4096)
        xs = [torch.randn(n, device=dev).to(dtype) for _ in range(W)]
        g.allreduce(xs, layers, bits=fmt)
        torch.cuda.synchronize()
        g.check()
        res[mb] = timeit(lambda: g.allreduce(xs, layers, bits=fmt))
        del g, xs
    slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])  # us per MB per virtual rank
    row = {"world": W, "dtype": dt, "bits": bits, "bucket": args.bucket, "lanes_per_rank": lanes,
           "times_us": {str(k): round(v, 1) for k, v in res.items()},
           "us_per_equivalent_64MB_allreduce": round(slope * 64 / W, 1),
           "note": "slope * (64 MB / W): device work of one real rank of a 64 MB allreduce on W GPUs, NVLink excluded"}
    rows.append(row)
    print(json.dumps(row), flush=True)
    res = {}
    for kb in sorted(int(x) for x in args.oneshot_kbs.split(",")):
        n = (kb << 10) // es
        layers = [(0, n, width, args.bucket)]
        g = C.LocalSraGroup(W, lanes, n * es * 2 + (1 << 20), 20000, 4096)
        xs = [torch.randn(n, device=dev).to(dtype) for _ in range(W)]
        g.allreduce_oneshot(xs, layers, bits=fmt)
        torch.cuda.synchronize()
        g.check()
        res[kb] = timeit(lambda: g.allreduce_oneshot(xs, layers, bits=fmt), iters=50, warmup=10)
        del g, xs
    row = {"kernel": "oneshot", "world": W, "dtype": dt, "bits": bits, "bucket": args.bucket, "lanes_per_rank": lanes,
           "times_us_by_kb": {str(k): round(v, 1) for k, v in res.items()},
           "note": "one call of W virtual ranks, each `kb` KB: the one-shot kernel's latency-bound sizes"}
    rows.append(row)
    print(json.dumps(row), flush=True)
    res = {}
    for mb in mbs:
        n = (mb << 20) // es // W * W
        shard = [(0, n // W, width, args.bucket)]
        g = C.LocalSraGroup(W, lanes, n * es // W * 2 + (1 << 20), 20000, 4096)
        xs = [torch.randn(n, device=dev).to(dtype) for _ in range(W)]
        outs = [torch.empty(n // W, device=dev, dtype=dtype) for _ in range(W)]
        g.reduce_scatter(xs, outs, shard, bits=fmt)
        torch.cuda.synchronize()
        g.check()
        res[mb] = timeit(lambda: g.reduce_scatter(xs, outs, shard, bits=fmt))
        del g, xs, outs
    slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])
    row = {"op": "reduce_scatter", "world": W, "dtype": dt, "bits": bits, "bucket": args.bucket,
           "lanes_per_rank": lanes, "times_us": {str(k): round(v, 1) for k, v in res.items()},
           "us_per_equivalent_64MB_reduce_scatter": round(slope * 64 / W, 1),
           "note": "slope * (64 MB / W): device work of one real rank of a 64 MB-input reduce-scatter on W GPUs, "
                   "NVLink excluded"}
    rows.append(row)
    print(json.dumps(row), flush=True)
    res = {}
    for mb in mbs:
        n = (mb << 20) // es // W * W
        shard = [(0, n // W, width, args.bucket)]
        g = C.LocalSraGroup(W, lanes, n * es // W * 2 + (1 << 20), 20000, 4096)
        xs = [torch.randn(n // W, device=dev).to(dtype) for _ in range(W)]
        outs = [torch.empty(n, device=dev, dtype=dtype) for _ in range(W)]
        g.all_gather(xs, outs, shard, bits=fmt)
        torch.cuda.synchronize()
        g.check()
        res[mb] = timeit(lambda: g.all_gather(xs, outs, shard, bits=fmt))
        del g, xs, outs
    slope = (res[mbs[-1]] - res[mbs[0]]) / (mbs[-1] - mbs[0])
    row = {"op": "all_gather", "world": W, "dtype": dt, "bits": bits, "bucket": args.bucket,
           "lanes_per_rank": lanes, "times_us": {str(k): round(v, 1) for k, v in res.items()},
           "us_per_equivalent_64MB_all_gather": round(slope * 64 / W, 1),
           "note": "slope * (64 MB / W): device work of one real rank of a 64 MB-output all-gather on W GPUs, "
                   "NVLink excluded"}
    rows.append(row)
    print(json.dumps(row), flush=True)
    return rows


def skewed_counts(W, n):
    """counts[q][r] ~ 1 + (r - q) mod W, every row and column summing to n (a Latin square)."""
    tot = W * (W + 1) // 2
    base = [n * (1 + k) // tot for k in range(W)]
    base[-1] += n - sum(base)
    return [[base[(r - q) % W] for r in range(W)] for q in range(W)]


def a2a_bits(b):
    """an all-to-all --bits entry: an integer width, or an FP8 format name"""
    return b if b in ("e4m3", "e5m2", "e4m3_pow2", "e5m2_pow2", "e4m3_sr", "e5m2_sr") else int(b)


def all_to_all_rows(args, dev, W, lanes):
    rows = []
    for dtype in [getattr(torch, d) for d in args.dtypes.split(",")]:
        es = torch.empty((), dtype=dtype).element_size()
        for bits in [a2a_bits(b) for b in args.bits.split(",")]:
            for mb in [int(x) for x in args.mbs.split(",")]:
                n = (mb << 20) // es // W * W
                slot = n * es // W * 2 + (1 << 20)
                row = {"op": "all_to_all", "world": W, "dtype": str(dtype).replace("torch.", ""), "bits": bits,
                       "bucket": args.bucket, "mb_per_rank": mb, "lanes_per_rank": lanes}
                g = C.LocalSraGroup(W, lanes, slot, 20000, 4096)
                xs = [torch.randn(n, device=dev).to(dtype) for _ in range(W)]
                for kind, c in (("equal", [[n // W] * W for _ in range(W)]), ("skewed", skewed_counts(W, n))):
                    outs = [torch.empty(sum(c[q][r] for q in range(W)), device=dev, dtype=dtype) for r in range(W)]
                    g.all_to_all(xs, outs, c, bits=bits, bucket_size=args.bucket)
                    torch.cuda.synchronize()
                    g.check()
                    row[f"a2a_{kind}_us"] = round(timeit(lambda: g.all_to_all(xs, outs, c, bits=bits,
                                                                              bucket_size=args.bucket)), 1)
                    del outs
                shard = [(0, n // W, 8 if isinstance(bits, str) else bits, args.bucket)]
                routs = [torch.empty(n // W, device=dev, dtype=dtype) for _ in range(W)]
                g.reduce_scatter(xs, routs, shard)
                torch.cuda.synchronize()
                g.check()
                row["rs_us"] = round(timeit(lambda: g.reduce_scatter(xs, routs, shard)), 1)
                row["a2a_equal_over_rs"] = round(row["a2a_equal_us"] / row["rs_us"], 3)
                row["note"] = ("W virtual ranks on one GPU, all W kernels of a call: the device work of W real ranks, "
                               "NVLink excluded; rs = rs_kernel on the same mb MB input per rank")
                del g, xs, routs
                torch.cuda.empty_cache()
                rows.append(row)
                print(json.dumps(row), flush=True)
    return rows


def ag_codes_rows(args, dev, W, lanes):
    rows = []
    name = torch.cuda.get_device_name(0)
    dtype, es = torch.bfloat16, 2
    for H in [int(h) for h in args.hiddens.split(",")]:
        S = args.rows * H
        g = C.LocalSraGroup(W, lanes, S + S // 8 + (1 << 20), 20000, 4096)
        xs = [torch.randn(S, device=dev).to(dtype) for _ in range(W)]
        for B in (128, H):
            shard = [(0, S, 8, B)]
            dec = [torch.empty(W * S, device=dev, dtype=dtype) for _ in range(W)]
            codes = [torch.empty(W * S, device=dev, dtype=torch.float8_e4m3fn) for _ in range(W)]
            scales = [torch.empty(W * S // B, device=dev) for _ in range(W)]
            tq = [None] * W

            def arm_c():
                g.all_gather(xs, dec, shard, bits="e4m3")
                for r in range(W):
                    v = dec[r].view(-1, B).float()
                    unit = v.abs().amax(dim=1, keepdim=True) * (1.0 / 448.0)
                    inv = torch.where(unit > 0, 1.0 / unit, torch.zeros_like(unit))
                    tq[r] = ((v * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn), unit)

            def arm_d():
                g.all_gather(xs, codes, shard, bits="e4m3", output_scales=scales)

            arms = {"c": arm_c, "d": arm_d}
            meds = {k: [] for k in arms}
            for _ in range(args.repeats):
                ts = {k: [] for k in arms}
                for it in range(3 + args.iters):
                    for k, fn in arms.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        fn()
                        e1.record()
                        torch.cuda.synchronize()
                        if it >= 3:
                            ts[k].append(e0.elapsed_time(e1) * 1e3)
                for k in arms:
                    meds[k].append(sorted(ts[k])[len(ts[k]) // 2])
            g.check()
            for r in range(W):
                got = (codes[r].float() * scales[r].repeat_interleave(B)).to(dtype)
                assert torch.equal(got.view(torch.int16), dec[r].view(torch.int16)), "codes arm differs from decoded arm"
            wire = S + S // B * 8
            common = W * (S * es + 2 * (W - 1) * wire + W * S + W * S // B * 4)
            row = {"op": "ag_codes", "gpu": name, "world": W, "dtype": "bfloat16", "bits": "e4m3", "H": H, "bucket": B,
                   "rows_per_rank": args.rows, "lanes_per_rank": lanes,
                   "hbm_c_GB": round((common + 2 * W * W * S * es) / 1e9, 3), "hbm_d_GB": round(common / 1e9, 3)}
            for k in arms:
                v = sorted(meds[k])
                row[f"{k}_us"] = {"min": round(v[0], 1), "median": round(v[len(v) // 2], 1), "max": round(v[-1], 1)}
            row["c_over_d"] = round(row["c_us"]["median"] / row["d_us"]["median"], 2)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del dec, codes, scales, tq
        del g, xs
        torch.cuda.empty_cache()
    return rows


if __name__ == "__main__":
    main()
