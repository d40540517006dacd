"""ctypes binding of ``libfaa_b200.so`` (the C ABI of ``include/faa_b200.h``).

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).
There is no Python / CPU implementation of the pixel path behind this module: if the
library is missing, importing the package fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FAA_B200_LIB") or os.path.join(_HERE, "libfaa_b200.so")   # env: tuning builds only

# ---- status codes (enum faa_status) and the reference exceptions they stand for
OK, ERR_UNKNOWN_OP, ERR_MAGNITUDE, ERR_VALUE, ERR_CUDA, ERR_NO_DEVICE, ERR_UNSUPPORTED = range(7)
F16, BF16, F32, U8_HWC = 0, 1, 2, 3
DRAW_NONE, DRAW_MIRROR, DRAW_BOX = 0, 1, 2
MAX_FUSED_OPS, MAX_POLICY_OPS = 2, 8

SAMPLE_DTYPE = np.dtype([("sub", "<u2"), ("gate", "u1"), ("sign", "u1"), ("crop_dy", "i1"),
                         ("crop_dx", "i1"), ("flip", "u1"), ("reserved", "u1"),
                         ("zero_box", "<i2", (4,))])
BOX_DTYPE = np.dtype([("x0", "<i2"), ("y0", "<i2"), ("x1", "<i2"), ("y1", "<i2")])
JITTER_DTYPE = np.dtype([("alpha", "<f4", (3,)), ("order", "u1", (4,))])          # faa_jitter_t
CROP_BOX_DTYPE = np.dtype([("x0", "<i4"), ("y0", "<i4"), ("w", "<i4"), ("h", "<i4")])  # faa_crop_box_t
IMAGE_DTYPE = np.dtype([("data", "<u8"), ("h", "<i4"), ("w", "<i4")])              # faa_image_t
CROP_RANDOM, CROP_CENTER = 0, 1
JPEG_HEADER_DTYPE = np.dtype([("offset", "<i8"), ("len", "<i8"), ("scan_off", "<i8"), ("scan_len", "<i8"),
                              ("h", "<i4"), ("w", "<i4"), ("ncomp", "<i4"), ("hs", "<i4"), ("vs", "<i4"),
                              ("restart", "<i4"), ("mcu_x", "<i4"), ("mcu_y", "<i4"), ("table_at", "<i4", (9,)),
                              ("pool", "<i4", (9,)), ("qprec", "<i4"), ("reserved", "<i4")])   # faa_jpeg_header_t
JPEG_TABLE_DTYPE = np.dtype([("q", "<u2", (64,)), ("bits", "u1", (16,)), ("vals", "u1", (256,))])   # faa_jpeg_table_t
JPEG_TRUNCATED, JPEG_BAD_CODE, JPEG_BAD_COEF, JPEG_BAD_RESTART = 1, 2, 4, 8                       # faa_jpeg_status
JPEG_SYNC_DTYPE = np.dtype([("mcu", "<i4"), ("byte", "<i4"), ("bit", "<i2"), ("pred", "<i2", (3,))])  # faa_jpeg_sync_t
JPEG_SCAN_DTYPE = np.dtype([("off", "<i8"), ("len", "<i8"), ("restart", "<i4"), ("ns", "<i4"), ("comp", "<i4", (3,)),
                            ("ss", "<i4"), ("se", "<i4"), ("ah", "<i4"), ("al", "<i4"), ("wave", "<i4"),
                            ("dc_at", "<i4", (3,)), ("ac_at", "<i4", (3,)), ("pool", "<i4", (6,)),
                            ("reserved", "<i4", (2,))])                                            # faa_jpeg_scan_t
JPEG_PROGRESSIVE, JPEG_MAX_SCANS = 1, 64
assert SAMPLE_DTYPE.itemsize == 16 and BOX_DTYPE.itemsize == 8 and IMAGE_DTYPE.itemsize == 16
assert JPEG_HEADER_DTYPE.itemsize == 144 and JPEG_TABLE_DTYPE.itemsize == 400 and JPEG_SYNC_DTYPE.itemsize == 16
assert JPEG_SCAN_DTYPE.itemsize == 112


class Tail(C.Structure):          # faa_tail_t
    _fields_ = [("out_h", C.c_int32), ("out_w", C.c_int32), ("out_dtype", C.c_int32),
                ("use_zero_box", C.c_int32), ("mean", C.c_float * 3), ("std", C.c_float * 3),
                ("crop_pad", C.c_int32), ("reserved", C.c_int32)]


class Rng(C.Structure):           # faa_rng_t
    _fields_ = [("seed", C.c_uint64), ("first_index", C.c_uint64), ("crop_pad", C.c_int32),
                ("hflip", C.c_int32), ("zero_box_len", C.c_int32), ("reserved", C.c_int32)]


class CropCfg(C.Structure):       # faa_crop_cfg_t
    _fields_ = [("mode", C.c_int32), ("img_size", C.c_int32), ("min_covered", C.c_double),
                ("aspect_lo", C.c_double), ("aspect_hi", C.c_double), ("area_lo", C.c_double),
                ("area_hi", C.c_double), ("max_attempts", C.c_int32), ("reserved", C.c_int32), ("rng", Rng)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "fast_autoaugment_b200: %s is missing. The augmentation path is CUDA-only (sm_90a) "
            "and has no CPU fallback - build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (needs nvcc)." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, u64, f32, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_double
    P = C.POINTER
    sig = {
        "faa_abi_version": (C.c_int, []),
        "faa_last_error": (C.c_char_p, []),
        "faa_device_count": (C.c_int, []),
        "faa_op_id_from_name": (C.c_int, [C.c_char_p]),
        "faa_op_name": (C.c_char_p, [C.c_int]),
        "faa_op_range": (C.c_int, [C.c_int, P(f64), P(f64)]),
        "faa_policy_create": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, P(vp)]),
        "faa_policy_destroy": (C.c_int, [vp]),
        "faa_policy_dims": (C.c_int, [vp, P(C.c_int), P(C.c_int)]),
        "faa_policy_compiled_op": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
        "faa_policy_draw_kind": (C.c_int, [vp, C.c_int, C.c_int]),
        "faa_cutout_box": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, f64, f64, vp]),
        "faa_sample_policy_mt": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]),
        "faa_sample_philox": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, P(Tail), P(Rng), vp, vp, vp]),
        "faa_sample_philox_at": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, P(Tail), P(Rng), vp, vp, vp, vp]),
        "faa_policy_cached_tables": (C.c_int, [vp, P(C.c_int), P(u64)]),
        "faa_augment": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), vp, vp, P(Rng), C.c_int, vp]),
        "faa_policy_set_overlap": (C.c_int, [vp, C.c_int]),
        "faa_augment_many": (C.c_int, [vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), P(Rng), C.c_uint64, vp]),
        "faa_augment_tta": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, P(Tail), P(Rng), vp]),
        "faa_augment_mixup": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, P(Tail),
                                        vp, vp, P(Rng), vp, f32, f32, vp]),
        "faa_augment_host": (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), P(Rng), vp]),
        "faa_mixup": (C.c_int, [vp, vp, vp, C.c_int, i64, C.c_int, f32, f32, vp]),
        "faa_mix_u8": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), f32, f32, vp]),
        "faa_enable_peer_access": (C.c_int, [C.c_int]),
        "faa_peer_alloc": (C.c_int, [C.c_size_t, P(C.c_void_p), vp]),
        "faa_peer_open": (C.c_int, [vp, P(C.c_void_p)]),
        "faa_peer_close": (C.c_int, [vp]),
        "faa_peer_free": (C.c_int, [vp]),
        "faa_mix_u8_peer": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), f32, f32, vp]),
        "faa_color_jitter": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp]),
        "faa_policy_set_lighting": (C.c_int, [vp, vp, C.c_int]),
        "faa_center_crop_box": (C.c_int, [C.c_int, C.c_int, C.c_int, vp]),
        "faa_crop_resize": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, P(Tail), vp, P(CropCfg), vp]),
        "faa_crop_resize_ragged": (C.c_int, [vp, vp, C.c_int, vp, P(Tail), vp, P(CropCfg), vp]),
        "faa_augment_ragged": (C.c_int, [vp, vp, vp, C.c_int, vp, vp, vp, vp, P(Rng), C.c_int, vp]),
        "faa_jpeg_parse": (C.c_int, [C.c_char_p, C.c_size_t, vp]),
        "faa_jpeg_tables": (C.c_int, [C.c_char_p, C.c_size_t, vp, vp]),
        "faa_jpeg_decoder_create": (C.c_int, [P(vp)]),
        "faa_jpeg_decoder_destroy": (C.c_int, [vp]),
        "faa_jpeg_index_capacity": (C.c_int, [vp]),
        "faa_jpeg_index_build": (C.c_int, [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp]),
        "faa_jpeg_index_find": (C.c_int, [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp]),
        "faa_jpeg_decode": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                      C.c_int, vp]),
        "faa_jpeg_parse_progressive": (C.c_int, [C.c_char_p, C.c_size_t, vp, vp, C.c_int, P(C.c_int)]),
        "faa_jpeg_scan_tables": (C.c_int, [C.c_char_p, C.c_size_t, vp, vp, C.c_int, vp]),
        "faa_jpeg_decode_progressive": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp,
                                                  vp]),
        "faa_launch_count": (u64, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)          # AttributeError here == header/library mismatch
        fn.restype = res
        fn.argtypes = args
    return lib, tuple(sig)


lib, EXPORTS = _load()


class FaaRuntimeError(RuntimeError):
    pass


def check(status: int):
    """Map a status code to the exception the reference would raise at that point."""
    if status == OK:
        return
    msg = (lib.faa_last_error() or b"").decode()
    if status == ERR_UNKNOWN_OP:
        raise KeyError(msg)                 # reference augmentations.py:189
    if status == ERR_MAGNITUDE:
        raise AssertionError(msg)           # reference augmentations.py per-op asserts
    if status == ERR_VALUE:
        raise ValueError(msg)
    raise FaaRuntimeError("faa_b200 status %d: %s" % (status, msg))


def op_id(name) -> int:
    return lib.faa_op_id_from_name(str(name).encode())


def device_count() -> int:
    return lib.faa_device_count()
