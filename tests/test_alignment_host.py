"""Buffer alignment the policy kernels need, refused on the host before anything touches a device.

The kernels load the input as 32-bit words when W % 4 == 0 and store each output plane as one 16-byte (fp32),
8-byte (fp16 / bf16) or three 32-bit (uint8 HWC) stores when out_w % 4 == 0.  A contiguous view at an offset into a
larger allocation (`torch.empty(n + 1, ...)[1:]`) passes every shape check, so the C ABI refuses misaligned bases with
FAA_ERR_UNSUPPORTED and a message that names the alignment.  The checks come before the device is touched: refused
calls return the same status on a machine without a GPU, and they use fake device addresses that are never
dereferenced.  (The GPU side - the Python call raises and launches nothing - is in tests/test_gpu_geometries.py.)"""
import ctypes as C

import numpy as np
import pytest
import torch

from fast_autoaugment_b200 import _lib, archive
from fast_autoaugment_b200.engine import CompiledPolicy, TailSpec, make_rng

BASE = 0x7F0000000000                     # a fake, 256-byte aligned device address
F16, BF16, F32, U8 = torch.float16, torch.bfloat16, torch.float32, torch.uint8


def _pol():
    return CompiledPolicy(archive.fa_resnet50_rimagenet())


def _augment(pol, in_off, out_off, shape, dtype):
    H, W = shape
    t = TailSpec.imagenet(0, dtype).c_struct(H, W)
    r = make_rng(1, 0, TailSpec.imagenet(0, dtype))
    return _lib.lib.faa_augment(pol.handle, BASE + in_off, BASE + (1 << 30) + out_off, 4, H, W, C.byref(t), None, None,
                                C.byref(r), 0, None)


# (input offset, output offset, shape, dtype, the alignment the message names)
REFUSED = [
    (0, 8, (8, 8), F32, "16-byte"),
    (0, 4, (224, 224), F32, "16-byte"),
    (0, 4, (8, 8), F16, "8-byte"),
    (0, 2, (8, 8), BF16, "8-byte"),
    (0, 2, (8, 8), U8, "4-byte"),
    (0, 1, (8, 8), U8, "4-byte"),
    (2, 0, (8, 8), F32, "4-byte"),
    (1, 0, (375, 500), U8, "4-byte"),
]
# what the kernels accept: these reach the device check
ACCEPTED = [
    (4, 0, (8, 8), F32),                  # 4-byte aligned input
    (0, 8, (8, 8), F16), (0, 8, (8, 8), BF16), (0, 4, (8, 8), U8),
    (1, 0, (6, 6), F32),                  # W % 4 != 0: byte loads only
    (0, 4, (6, 6), F32), (0, 2, (6, 6), F16), (0, 1, (6, 6), U8),   # out_w % 4 != 0: element stores only
]


@pytest.mark.parametrize("in_off,out_off,shape,dtype,need", REFUSED)
def test_misaligned_buffers_are_refused(in_off, out_off, shape, dtype, need):
    pol = _pol()
    assert _augment(pol, in_off, out_off, shape, dtype) == _lib.ERR_UNSUPPORTED
    msg = _lib.lib.faa_last_error().decode()
    assert need in msg and "aligned" in msg, msg


@pytest.mark.skipif(torch.cuda.is_available(), reason="the accepted calls would launch on the fake addresses")
@pytest.mark.parametrize("in_off,out_off,shape,dtype", ACCEPTED)
def test_aligned_buffers_reach_the_device_check(in_off, out_off, shape, dtype):
    assert _augment(_pol(), in_off, out_off, shape, dtype) == _lib.ERR_NO_DEVICE


def test_every_entry_refuses_misaligned_buffers():
    """faa_augment_tta, faa_augment_mixup and faa_augment_many share the check; faa_augment_many refuses before its
    first step, faa_augment_host checks a caller-owned device output up front"""
    pol = _pol()
    H = W = 8
    t = TailSpec.imagenet(0, F32).c_struct(H, W)
    r = make_rng(1, 0, TailSpec.imagenet(0, F32))
    out = BASE + (1 << 30)
    assert _lib.lib.faa_augment_tta(pol.handle, BASE, out + 4, 2, 3, H, W, C.byref(t), C.byref(r), None) == _lib.ERR_UNSUPPORTED
    pol2 = CompiledPolicy([[("Invert", 1.0, 0.0), ("Color", 0.5, 0.3)]])
    assert _lib.lib.faa_augment_mixup(pol2.handle, BASE + 2, 4, 0, out, 4, H, W, C.byref(t), None, None, C.byref(r),
                                      BASE + (2 << 30), 0.5, 0.5, None) == _lib.ERR_UNSUPPORTED
    assert b"4-byte" in _lib.lib.faa_last_error()
    ins = (C.c_void_p * 3)(BASE, BASE + 4096, BASE + 8192)
    outs = (C.c_void_p * 3)(out, out + 4096, out + 8192 + 8)             # only the LAST step is misaligned
    assert _lib.lib.faa_augment_many(pol.handle, 3, ins, outs, 4, H, W, C.byref(t), C.byref(r), 4, None) == _lib.ERR_UNSUPPORTED
    assert b"16-byte" in _lib.lib.faa_last_error()
    h_in = np.zeros((4, H, W, 3), np.uint8)
    assert _lib.lib.faa_augment_host(pol.handle, h_in.ctypes.data, None, out + 8, 4, H, W, C.byref(t),
                                     C.byref(r), None) == _lib.ERR_UNSUPPORTED
    assert b"16-byte" in _lib.lib.faa_last_error()
