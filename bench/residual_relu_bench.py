#!/usr/bin/env python
"""Device time of the ResNet residual join, native kernels against the eager ops they replace, at
the block-output shapes of ResNet-50 (bf16, channels_last, batch 128 by default).

    python bench/residual_relu_bench.py [--batch 128] [--iters 20]

forward   native: C.residual_relu_forward(a, b)            3 passes (read a, b; write y)
          eager:  relu_(a + b)                              5 passes
backward  native: C.residual_relu_backward(y, ga, gb)      4 passes (read y, ga, gb; write g)
          eager:  threshold_backward(ga + gb, y, 0)         6 passes

CUDA events around `iters` back-to-back calls over rotating operand sets (more than 2x L2 in
total), median of 3 repetitions; GB/s = the passes' bytes / time. Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=128)
    p.add_argument("--iters", type=int, default=20)
    args = p.parse_args()

    import torch

    import torch_cgx_b200 as cgx
    from torch_cgx_b200.utils.clocks import ClockSampler

    C = cgx._C
    dev = torch.device("cuda", 0)
    sampler = ClockSampler(0)
    sampler.start()
    B = args.batch
    shapes = {"layer1": (B, 256, 56, 56), "layer2": (B, 512, 28, 28), "layer3": (B, 1024, 14, 14),
              "layer4": (B, 2048, 7, 7)}
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size

    def timeit(fn, sets):
        for s in sets[:2]:
            fn(*s)
        reps = []
        for _ in range(3):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.iters):
                fn(*sets[i % len(sets)])
            e1.record()
            torch.cuda.synchronize()
            reps.append(e0.elapsed_time(e1) * 1e3 / args.iters)
        return sorted(reps)[1]

    rows = []
    for name, shape in shapes.items():
        def make():
            return torch.randn(shape, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)

        tensor_bytes = make().numel() * 2
        nsets = max(2, -(-4 * l2 // (4 * tensor_bytes)))
        sets = [(make(), make(), make(), make()) for _ in range(nsets)]  # a, b, ga, gb
        ys = [C.residual_relu_forward(a, b) for a, b, _, _ in sets]
        fsets = [(a, b) for a, b, _, _ in sets]
        bsets = [(y, ga, gb) for y, (_, _, ga, gb) in zip(ys, sets)]
        t = {
            "fwd_native": timeit(lambda a, b: C.residual_relu_forward(a, b), fsets),
            "fwd_eager": timeit(lambda a, b: torch.relu_(a + b), fsets),
            "bwd_native": timeit(lambda y, ga, gb: C.residual_relu_backward(y, ga, gb), bsets),
            "bwd_eager": timeit(lambda y, ga, gb: torch.ops.aten.threshold_backward(ga + gb, y, 0), bsets),
        }
        passes = {"fwd_native": 3, "fwd_eager": 5, "bwd_native": 4, "bwd_eager": 6}
        row = {"stage": name, "shape": list(shape), "mb_per_tensor": round(tensor_bytes / 2**20, 1)}
        for k, us in t.items():
            row[f"{k}_us"] = round(us, 1)
            row[f"{k}_gbs"] = round(passes[k] * tensor_bytes / us / 1e3, 1)
        rows.append(row)
        del sets, ys, fsets, bsets
    print(json.dumps({"rows": rows, "clocks": sampler.stop(), "dtype": "bf16", "layout": "channels_last",
                      "timing": "CUDA events, back-to-back calls over rotating operand sets (> 2x L2), median of 3"}))


if __name__ == "__main__":
    main()
