"""Reference ``FastAutoAugment/aug_mixup.py`` ``mixup`` on the CUDA path.

Same signature, same draws in the same order (``torch.randperm`` on the CPU generator, then
one ``np.random.beta``; reference ``aug_mixup.py:14,18``), same return tuple; the axpby runs
in the library's mixup kernel with the reference's fp32 rounding sequence.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check

_DT = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16, torch.float32: _lib.F32}


def mixup_resolved(data: torch.Tensor, indices: torch.Tensor, lam: float, out=None):
    """``data*lam + data[indices]*(1-lam)`` (reference aug_mixup.py:21) on a CUDA tensor.

    ``out`` (optional) must not overlap ``data``: mixing in place would let one sample be overwritten while another
    still reads it as its partner, so an overlapping ``out`` raises ``ValueError`` before anything is launched.  At
    most 65535 samples per call."""
    if not data.is_cuda:
        raise _lib.FaaRuntimeError("mixup needs a CUDA tensor (no CPU fallback)")
    if data.dtype not in _DT:
        raise ValueError("mixup supports float16 / bfloat16 / float32")
    data = data.contiguous()
    b = data.size(0)
    n_per = data.numel() // max(b, 1)
    if out is None:
        out = torch.empty_like(data)
    elif out.shape != data.shape or out.dtype != data.dtype or out.device != data.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous tensor of data's shape, dtype and device")
    perm = indices.to(device=data.device, dtype=torch.int64).contiguous()
    with torch.cuda.device(data.device):
        stream = C.c_void_p(torch.cuda.current_stream(data.device).cuda_stream)
        check(lib.faa_mixup(data.data_ptr(), out.data_ptr(), perm.data_ptr(), b, n_per, _DT[data.dtype],
                            float(np.float32(lam)), float(np.float32(1 - lam)), stream))
    return out


def mixup(data, targets, alpha):
    """Drop-in for reference ``mixup(data, targets, alpha)`` (aug_mixup.py:13-23)."""
    indices = torch.randperm(data.size(0))
    shuffled_targets = targets[indices.to(targets.device)]
    lam = np.random.beta(alpha, alpha)
    lam = max(lam, 1. - lam)
    assert 0.0 <= lam <= 1.0, lam
    return mixup_resolved(data, indices, lam), targets, shuffled_targets, lam
