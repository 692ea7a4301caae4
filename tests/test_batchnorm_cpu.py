"""``batch_norm_act`` on CPU: the eager path, bitwise equal to ``relu_(bn(x))`` / ``bn(x)`` with the same
gradients and buffer updates, and ResNets whose parameter and buffer names and order are unchanged."""
import copy

import pytest
import torch
import torch.nn as nn

from torch_cgx_b200.models.batchnorm import batch_norm_act, native_ok
from torch_cgx_b200.models.resnet import resnet18, resnet50


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("channels_last", [False, True])
def test_eager_path_matches_modules(relu, channels_last):
    torch.manual_seed(0)
    bn = nn.BatchNorm2d(6)
    with torch.no_grad():
        bn.weight.normal_()
        bn.bias.normal_()
    ref = copy.deepcopy(bn)
    x = torch.randn(4, 6, 5, 3)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    assert not native_ok(bn, x)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    ya = batch_norm_act(bn, xa, relu)
    yb = ref(xb)
    if relu:
        yb = torch.relu_(yb)
    g = torch.randn_like(ya)
    ya.backward(g)
    yb.backward(g)
    assert torch.equal(ya, yb)
    assert torch.equal(xa.grad, xb.grad)
    for pa, pb in zip(bn.parameters(), ref.parameters()):
        assert torch.equal(pa.grad, pb.grad)
    for ba, bb in zip(bn.buffers(), ref.buffers()):
        assert torch.equal(ba, bb)
    assert int(bn.num_batches_tracked) == 1


@pytest.mark.parametrize("ctor,n_bn", [(resnet18, 20), (resnet50, 53)])
def test_resnet_names_and_bn_count(ctor, n_bn):
    net = ctor()
    names = [n for n, _ in net.named_parameters()] + [n for n, _ in net.named_buffers()]
    assert names[:3] == ["stem.0.weight", "stem.1.weight", "stem.1.bias"]
    assert "layer2.0.downsample.1.running_mean" in names
    assert sum(isinstance(m, nn.BatchNorm2d) for m in net.modules()) == n_bn
    assert len(names) == len(set(names))
