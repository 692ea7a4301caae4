"""NaN-aware bitwise comparison of kernel results.

``torch.equal`` is False for any tensor holding a NaN and ignores the sign of zero, so the
kernel tests compare with ``assert_same`` instead: the NaN positions must be identical and
every other element bitwise identical. Wire bytes (uint8) and integer tensors are compared
exactly. NaN payloads are not compared: the CPU and the GPU may legitimately differ there.
"""
from __future__ import annotations

import torch

_INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16,
             torch.float64: torch.int64}


def mismatch(a: torch.Tensor, b: torch.Tensor) -> str:
    """'' if a and b are the same (NaN-aware, bitwise), else a description of the first difference."""
    a, b = a.detach().cpu(), b.detach().cpu()
    if a.dtype != b.dtype or a.shape != b.shape:
        return f"dtype/shape differ: {a.dtype}{tuple(a.shape)} vs {b.dtype}{tuple(b.shape)}"
    if a.dtype not in _INT_VIEW:
        bad = (a != b).reshape(-1).nonzero()
        return "" if bad.numel() == 0 else f"{bad.numel()} elements differ, first at {int(bad[0])}: " \
                                           f"{a.reshape(-1)[bad[0]].item()} vs {b.reshape(-1)[bad[0]].item()}"
    a, b = a.contiguous().reshape(-1), b.contiguous().reshape(-1)
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        i = int((na != nb).nonzero()[0])
        return f"NaN positions differ ({int(na.sum())} vs {int(nb.sum())}), first at {i}: {a[i].item()} vs {b[i].item()}"
    iv = _INT_VIEW[a.dtype]
    diff = (a.view(iv) != b.view(iv)) & ~na
    if diff.any():
        idx = diff.nonzero().reshape(-1)
        i = int(idx[0])
        return f"{idx.numel()} of {a.numel()} non-NaN elements differ bitwise, first at {i}: " \
               f"{a[i].item()!r} vs {b[i].item()!r}"
    return ""


def assert_same(a: torch.Tensor, b: torch.Tensor, what: str = "") -> None:
    msg = mismatch(a, b)
    assert not msg, f"{what}: {msg}" if what else msg
