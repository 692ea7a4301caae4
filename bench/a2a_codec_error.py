#!/usr/bin/env python
"""Error of the all-to-all wire codecs, computed on the CPU with the simulator (C.all_to_all_simulate,
bit for bit what a2a_kernel delivers) from seeded inputs: max-min 8-bit against the FP8 formats
e4m3 and e5m2, their power-of-two-scale twins e4m3_pow2 and e5m2_pow2 and their stochastic twins
e4m3_sr and e5m2_sr, at buckets of 128 and 512 elements.

Inputs, rows of H = 7168 fp32 elements (one MoE hidden state per row):
  gaussian   N(0, 1)
  outliers   N(0, 1) with 8 fixed channels scaled by 50 (the outlier channels of an FFN's input);
             the error is reported on the other channels
  student_t  Student-t with 3 degrees of freedom (heavy tails everywhere)

Reported per (input, bucket, codec): the relative L2 error ||dec - x|| / ||x|| and the largest
per-element relative error |dec - x| / |x| over elements with |x| >= 1e-3 * rms(x). For
--op all_to_all also the share of elements whose value changes when the decoded rows go through the
same codec a second time (requant_changed_pct): 0 for a codec whose decode of its encode is a
projection, and the bias: the relative L2 norm ||mean(dec) - x|| / ||x|| of the mean decoded value
over --seeds seeds of the random stream (only the _sr codecs depend on the seed; for the others
this is their deterministic error). This says nothing about training accuracy.

--op reduce_scatter / all_gather report the same for the compressed reduce-scatter and all-gather
of --world ranks (C.reduce_scatter_simulate / C.all_gather_simulate, bit for bit what rs_kernel and
ag_kernel deliver): every rank holds --rows rows of its own seeded input (rows divisible by the
world); the reduce-scatter's result is compared with the exact fp64 sum of each shard, the
all-gather's with the gathered inputs.
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402

C = cgx._C
H = 7168
OUTLIER_CHANNELS = 8


def make_rows(kind, rows, seed):
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(H, dtype=torch.bool)
    if kind == "student_t":
        x = _student_t(rows, g)
    else:
        x = torch.randn(rows, H, generator=g, dtype=torch.float64)
    if kind == "outliers":
        ch = torch.randperm(H, generator=g)[:OUTLIER_CHANNELS]
        x[:, ch] *= 50.0
        mask[ch] = True
    return x.float(), mask


def _student_t(rows, g, dof=3.0):
    """t = z / sqrt(chi2 / dof), chi2 the sum of dof squared normals (seeded, no global state)"""
    z = torch.randn(rows, H, generator=g, dtype=torch.float64)
    chi2 = (torch.randn(int(dof), rows, H, generator=g, dtype=torch.float64) ** 2).sum(0)
    return z / torch.sqrt(chi2 / dof)


def decode(x, bits, bucket, seed=0):
    """x's rows sent from rank 0 to rank 1 through the codec: what rank 1 receives"""
    n = x.numel()
    out = [torch.empty(0), torch.empty(n)]
    C.all_to_all_simulate([x.reshape(-1), torch.empty(0)], out, [[0, n], [0, 0]], bits=bits, bucket_size=bucket,
                          seed=seed)
    return out[1].reshape(x.shape)


def sharded(op, kind, rows, seed, world, bits, bucket):
    """(exact, received) of one sharded call of `world` ranks, rows of H as in make_rows; the
    received result of every rank, stacked, and the exact one of the same shape"""
    xs = [make_rows(kind, rows, seed + 1000 * q)[0] for q in range(world)]
    mask = make_rows(kind, rows, seed)[1]
    n = rows * H
    S = n // world
    fmt = bits if isinstance(bits, str) else None
    table = [(0, S, 8 if fmt else bits, bucket)]
    if op == "reduce_scatter":
        outs = [torch.empty(S) for _ in range(world)]
        C.reduce_scatter_simulate([x.reshape(-1) for x in xs], outs, table, bits=fmt)
        exact = torch.stack([x.double() for x in xs]).sum(0).reshape(-1)
        return exact.float().reshape(rows, H), torch.cat(outs).reshape(rows, H), mask
    shards = [xs[q].reshape(-1)[q * S:(q + 1) * S].clone() for q in range(world)]
    outs = [torch.empty(n) for _ in range(world)]
    C.all_gather_simulate(shards, outs, table, bits=fmt)
    return torch.cat(shards).reshape(rows, H), outs[0].reshape(rows, H), mask


def errors(x, dec, keep):
    x, dec = x[:, keep].double(), dec[:, keep].double()
    rel_l2 = float((dec - x).norm() / x.norm())
    big = x.abs() >= 1e-3 * x.pow(2).mean().sqrt()
    max_rel = float(((dec - x).abs() / x.abs())[big].max())
    return rel_l2, max_rel


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rows", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--buckets", type=int, nargs="+", default=[128, 512])
    ap.add_argument("--out", type=str, default=None, help="also write the JSON lines here")
    ap.add_argument("--op", default="all_to_all", choices=["all_to_all", "reduce_scatter", "all_gather"])
    ap.add_argument("--world", type=int, default=8, help="--op reduce_scatter / all_gather: ranks")
    ap.add_argument("--seeds", type=int, default=16, help="--op all_to_all: seeds of the bias column")
    args = ap.parse_args()
    if args.op != "all_to_all" and args.rows % args.world:
        ap.error("--rows must be divisible by --world")
    res = []
    for i, kind in enumerate(("gaussian", "outliers", "student_t")):
        x, mask = make_rows(kind, args.rows, args.seed + i)
        for bucket in args.buckets:
            for bits in (8, "e4m3", "e5m2", "e4m3_pow2", "e5m2_pow2", "e4m3_sr", "e5m2_sr"):
                extra = {}
                if args.op == "all_to_all":
                    dec = decode(x, bits, bucket)
                    rel_l2, max_rel = errors(x, dec, ~mask)
                    again = decode(dec, bits, bucket)
                    extra["requant_changed_pct"] = round(100 * float((again != dec).double().mean()), 3)
                    mean = torch.stack([decode(x, bits, bucket, s).double() for s in range(args.seeds)]).mean(0)
                    xd = x[:, ~mask].double()
                    extra["bias_rel_l2_pct"] = round(100 * float((mean[:, ~mask] - xd).norm() / xd.norm()), 4)
                else:
                    exact, got, m = sharded(args.op, kind, args.rows, args.seed + i, args.world, bits, bucket)
                    rel_l2, max_rel = errors(exact, got, ~m)
                r = {"op": args.op, "input": kind, "bucket": bucket, "codec": "maxmin8" if bits == 8 else bits,
                     "rel_l2_pct": round(100 * rel_l2, 3), "max_rel_pct": round(100 * max_rel, 2), **extra}
                res.append(r)
                print(json.dumps(r), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in res))


if __name__ == "__main__":
    main()
