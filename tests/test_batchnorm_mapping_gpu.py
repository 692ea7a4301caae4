"""The launch geometries of the channels_last BatchNorm chain kernels (statistics and backward reduction)
against ATen, bitwise, forward and backward, with the NaN-aware comparison of ``test_batchnorm_gpu.py``.

The kernels map ATen's chains onto 256-thread blocks of up to four 16-byte channel groups, with 4 or 8
rows in flight chosen from the chain length L, or onto 512-thread blocks of up to eight groups for chains
of more than 16 rows, and a grid merge that loads up to 8 staged block rows per slot before merging them. Each case below names the boundary of that mapping it exercises and that the
flagship and SMALL shapes of ``test_batchnorm_gpu.py`` do not; ``_bn_geometry.py`` prints the geometry.
"""
import pytest
import torch

import torch_cgx_b200 as cgx

from _bn_geometry import shape_geometry
from test_batchnorm_gpu import assert_same, check_forward, make_input, params

pytestmark = pytest.mark.gpu

C = cgx._C
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
VEC = {BF16: 8, F16: 8, F32: 4}

# (shape, dtype, geometry the case relies on, the branch it hits)
CASES = [
    ((8, 64, 16, 16), BF16, {"GY": 8, "U": 4}, "GY = 8: the smallest grid merge, half the slots merge no staged row"),
    ((9, 64, 16, 16), BF16, {"GY": 9, "U": 4}, "GY = 9: one slot merges two staged rows, the others one or none"),
    ((127, 32, 16, 16), BF16, {"GY": 127, "staged_per_slot": 8, "slabs": 1},
     "GY = 127: 8 staged rows per slot except 7 for the last, with a single 32-channel slab"),
    ((144, 64, 16, 16), BF16, {"GY": 128, "L": 5, "U": 8}, "L = 5 with a grid merge: 8 rows in flight, 3 of them idle"),
    ((128, 40, 28, 28), BF16, {"GY": 128, "L": 13, "slabs": 2, "partial_slab": True},
     "L = 13 and a last slab with one of its four groups valid, under the grid merge"),
    ((1, 64, 2, 2), BF16, {"GY": 1, "L": 1, "slabs": 2}, "L = 1 on the vector path, two slabs of one-row chains"),
    ((2, 64, 2, 2), BF16, {"GY": 1, "L": 2, "slabs": 2}, "L = 2 on the vector path with full slabs"),
    ((2, 64, 12, 12), BF16, {"GY": 1, "L": 5, "U": 8}, "L = 5 without a grid merge"),
    ((1, 64, 28, 28), BF16, {"GY": 1, "L": 13, "U": 8}, "L = 13 without a grid merge: two load windows of 8 rows"),
    ((16, 48, 24, 24), F32, {"GY": 36, "L": 4, "W": 16, "slabs": 3}, "fp32 vectors: three 16-channel slabs, GY = 36"),
    ((16, 40, 24, 24), F16, {"GY": 36, "slabs": 2, "partial_slab": True}, "fp16 partial last slab under the grid merge"),
    ((128, 32, 32, 32), BF16, {"GY": 128, "L": 16, "wide": False}, "L = 16: the longest chains on 256-thread blocks"),
    ((136, 72, 32, 32), BF16, {"GY": 128, "L": 17, "wide": True, "slabs": 2, "partial_slab": True},
     "L = 17: the shortest chains on 512-thread blocks, with an 8-channel last slab"),
    ((1, 64, 36, 36), BF16, {"GY": 1, "L": 21, "wide": True}, "512-thread blocks without a grid merge"),
]
# the one-element path (C not a multiple of 8): 32 channels per slab, each thread runs 8 (wide: 4) of the 64
# chains
ONE_ELEMENT = [
    ((128, 36, 28, 28), BF16, {"GY": 128, "L": 13, "U": 8, "slabs": 2, "partial_slab": True},
     "one-element path with 8 rows in flight, 8 staged rows per slot and a 4-channel last slab"),
    ((16, 44, 24, 24), F16, {"GY": 36, "L": 4, "U": 4, "slabs": 2, "partial_slab": True},
     "one-element path with 4 rows in flight and a grid merge"),
    ((136, 36, 32, 32), BF16, {"GY": 128, "L": 17, "wide": True, "slabs": 2, "partial_slab": True},
     "one-element path on 512-thread blocks"),
]


def _check_geometry(shape, vec, expect):
    geo = shape_geometry(shape, vec)
    assert {k: geo[k] for k in expect} == expect, geo


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c[0])) + "-" + str(c[1]).split(".")[-1])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("hostile", [False, True])
def test_vector_mapping_boundaries(case, relu, hostile):
    shape, dtype, expect, _ = case
    _check_geometry(shape, VEC[dtype], expect)
    check_forward(shape, dtype, relu, seed=21, hostile=hostile)


@pytest.mark.parametrize("case", ONE_ELEMENT, ids=lambda c: "x".join(map(str, c[0])) + "-" + str(c[1]).split(".")[-1])
@pytest.mark.parametrize("relu", [False, True])
def test_one_element_mapping(case, relu):
    shape, dtype, expect, _ = case
    assert shape[1] % 8 != 0
    _check_geometry(shape, 1, expect)
    check_forward(shape, dtype, relu, seed=22, hostile=True)


def test_graph_capture_then_eager():
    """a forward and backward captured in a CUDA graph and replayed twice (counters zeroed inside the capture
    and reset by the kernels), then eager calls on the same shape (the stream's cached counters)"""
    shape = (32, 64, 16, 16)
    _check_geometry(shape, 8, {"GY": 32, "U": 4, "slabs": 2})
    x = make_input(shape, BF16, 31, True)
    g = make_input(shape, BF16, 32, True)
    w, b, rm, rv = params(shape[1], 31)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y, mean, invstd = C.batchnorm_cl_forward(x, w, b, rm, rv, 0.1, 1e-5, True)
        gx, gw, gb = C.batchnorm_cl_backward(g, x, w, b, mean, invstd, True)
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for _ in range(2):
        y_ref, mean_ref, invstd_ref = torch.ops.aten.native_batch_norm(x, w, b, rm_ref, rv_ref, True, 0.1, 1e-5)
    torch.relu_(y_ref)
    g_ref = torch.ops.aten.threshold_backward(g, y_ref, 0)
    ref = torch.ops.aten.native_batch_norm_backward(g_ref, x, w, rm_ref, rv_ref, mean_ref, invstd_ref, True, 1e-5,
                                                    [True, True, True])
    for name, a, r in (("y", y, y_ref), ("save_mean", mean, mean_ref), ("save_invstd", invstd, invstd_ref),
                       ("running_mean", rm, rm_ref), ("running_var", rv, rv_ref), ("grad_input", gx, ref[0]),
                       ("grad_weight", gw, ref[1]), ("grad_bias", gb, ref[2])):
        assert_same(a, r, name)
    check_forward(shape, BF16, True, seed=33, hostile=True)
    check_forward(shape, BF16, False, seed=34)
