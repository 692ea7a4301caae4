#!/usr/bin/env python
"""Error of the FP8 allreduce on correlated ranks, round to nearest against stochastic rounding,
computed on the CPU with the SRA simulator (C.sra_simulate, bit for bit what sra_kernel delivers).

W ranks hold g + sigma * n_r: one shared gradient g (Gaussian with a per-channel log-normal scale)
plus small independent noise n_r per rank, the situation of data-parallel gradients. Each call
averages the W tensors through e5m2 / e5m2_sr and e4m3 / e4m3_sr (buckets of --bucket elements),
with the call number as the stream's sequence. Reported per format:
  per_call_rel_l2_pct   mean over calls of ||avg - exact|| / ||exact||, exact the fp64 average
  mean_rel_l2_pct       ||mean over calls of avg - exact|| / ||exact||: the error that stays when
                        many steps' updates add up (the bias)
A numerics result: it holds on any machine and says nothing about time.
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402

C = cgx._C


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--n", type=int, default=1 << 16, help="elements per rank")
    ap.add_argument("--bucket", type=int, default=512)
    ap.add_argument("--sigma", type=float, default=0.01, help="per-rank noise relative to the shared gradient")
    ap.add_argument("--calls", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    g = torch.Generator().manual_seed(args.seed)
    scale = torch.exp(torch.randn(args.n, generator=g, dtype=torch.float64) * 1.5)
    shared = torch.randn(args.n, generator=g, dtype=torch.float64) * scale
    xs = [(shared + args.sigma * torch.randn(args.n, generator=g, dtype=torch.float64) * scale).float()
          for _ in range(args.world)]
    exact = torch.stack([x.double() for x in xs]).mean(0)
    norm = float(exact.norm())
    table = [(0, args.n, 8, args.bucket)]
    res = []
    for fmt in ("e5m2", "e5m2_sr", "e4m3", "e4m3_sr"):
        per_call, total = [], torch.zeros(args.n, dtype=torch.float64)
        for call in range(args.calls):
            bufs = [x.clone() for x in xs]
            C.sra_simulate(bufs, table, average=True, seed=args.seed, seq=call, bits=fmt)
            got = bufs[0].double()
            per_call.append(float((got - exact).norm()) / norm)
            total += got
        r = {"world": args.world, "format": fmt, "bucket": args.bucket, "sigma": args.sigma, "calls": args.calls,
             "per_call_rel_l2_pct": round(100 * sum(per_call) / len(per_call), 4),
             "mean_rel_l2_pct": round(100 * float((total / args.calls - exact).norm()) / norm, 4)}
        res.append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in res))


if __name__ == "__main__":
    main()
