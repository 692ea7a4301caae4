"""Shared pieces of the multi-node sharded collective tests (test_sharded_hierarchy_cpu.py,
test_sharded_hierarchy_gpu.py): shard tables and inputs of the generic reducers' cases, the bytes
each rank sends, and the engine's (W, L) topologies."""
from __future__ import annotations

import numpy as np
import torch

from torch_cgx_b200.ops import oracle as O

from _edge_inputs import edge_inputs
from _reducer_cases import C, DT_CODE

# (W, L): several nodes of several ranks, one rank per node, and the node counts 2, 3 and 4
TOPOLOGIES = [(4, 2), (6, 3), (8, 4), (4, 1), (6, 2), (8, 2)]


def shard_table(c):
    """(one shard's table, S): mixed = a raw head of 37, the main layer, a raw layer of 301 and a
    5-bit layer; plain = the main layer alone. Both tile [0, S)."""
    n = c["n_main"]
    if c["mixed"]:
        return [(0, 37, 32, 512), (37, n, c["bits"], c["bucket"]), (37 + n, 301, 32, 512),
                (338 + n, 2001, 5, 64)], 338 + n + 2001
    return [(0, n, c["bits"], c["bucket"])], n


def sharded_inputs(c, S):
    """Every rank's W * S reduce-scatter input; hostile sources plant edge_inputs into the main layer
    of every shard, non-finite values on the shard's owner or on a peer."""
    W, dtype = c["world"], c["dtype"]
    g = torch.Generator().manual_seed(c["seed"])
    full = [(torch.randn(W * S, generator=g) * (r + 1)).to(dtype) for r in range(W)]
    if c["source"] != "randn":
        off, n = (37 if c["mixed"] else 0), c["n_main"]
        for s in range(W):
            xs, _ = edge_inputs(dtype, n, O.effective_bucket(c["bucket"]), 1000 + c["seed"] + s, world=W,
                                bits=min(c["bits"], 8), owners=np.full(n, s),
                                where="owner" if c["source"] == "edge_owner" else "peer")
            for r in range(W):
                full[r][s * S + off:s * S + off + n] = xs[r]
    return full


def own_shards(full):
    """Rank r's all-gather input: shard r of its reduce-scatter input (hostile values included)."""
    W = len(full)
    S = full[0].numel() // W
    return [t[r * S:(r + 1) * S].clone() for r, t in enumerate(full)]


def replicated(layers, world, S):
    return [(o + c * S, n, b, k) for c in range(world) for o, n, b, k in layers]


def sharded_bytes_sent(op, layers, S, world, dtype, skip_incomplete):
    """Per rank: the bytes Reducer::reduce_scatter (every peer's chunk) or ::all_gather (its own chunk
    to every peer) sends, from the replicated table's plan."""
    p = C.build_plan(replicated(layers, world, S), world=world, lanes=1, dtype=DT_CODE[dtype],
                     skip_incomplete=skip_incomplete, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS)
    cw = p["chunk_wire_bytes"]
    if op == "reduce_scatter":
        return [sum(cw) - cw[r] for r in range(world)]
    return [cw[r] * (world - 1) for r in range(world)]


def gather_with_skip(shards, layers, skip_incomplete):
    """The all-gather's reference with ``skip_incomplete`` (the partial last bucket stays raw)."""
    return torch.cat([O.quantize_dequantize_layers(t, layers, skip_incomplete=skip_incomplete) for t in shards])
