"""Host-side engine: policy handle, samplers and the batched launch.

``CompiledPolicy`` owns the C-ABI policy handle built from the reference's policy format
(``list[list[(op_name, prob, level)]]``, reference ``archive.py``).  Two samplers decide,
per image, what the reference's RNG draws decide:

* ``sample_parity``  - consumes the SAME global generators as the reference, in the same
  order (Python ``random``: sub-policy choice, gates, mirror signs - reference
  ``data.py:257-264``, ``augmentations.py:15,22,29,37,45,52,59``; ``numpy.random``: Cutout
  centres ``augmentations.py:131-132`` and CutoutDefault ``data.py:239-240``; torch CPU
  generator: RandomCrop / RandomHorizontalFlip), image after image, i.e. a
  ``num_workers=0`` DataLoader.  Seeding those generators like the reference reproduces
  the reference's output bit for bit.  Host cost ~2 us/image: for tests and drop-in use.
* Philox (``rng=``)  - the kernel draws the decisions itself (counter-based, keyed by
  (seed, global sample index)); same distributions, different stream; no host work.
"""
from __future__ import annotations

import ctypes as C
import random
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from ._lib import lib, check

CIFAR_MEAN, CIFAR_STD = (0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010)   # reference data.py:34
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)    # reference data.py:72

_DTYPES = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16, torch.float32: _lib.F32, torch.uint8: _lib.U8_HWC}


@dataclass
class TailSpec:
    """What follows the policy in ``transform_train`` (reference data.py:39-44,64,70-72,111-112)."""
    out_size: tuple | None = None      # RandomCrop size; None = same as the input
    crop_pad: int = 0                  # RandomCrop padding (data.py:40); 0 = no crop
    hflip: bool = False                # RandomHorizontalFlip (data.py:41,64)
    mean: tuple = CIFAR_MEAN
    std: tuple = CIFAR_STD
    cutout: int = 0                    # CutoutDefault length (data.py:111-112); 0 = off
    out_dtype: torch.dtype = torch.float16

    @staticmethod
    def cifar(cutout=16, out_dtype=torch.float16):
        return TailSpec((32, 32), 4, True, CIFAR_MEAN, CIFAR_STD, cutout, out_dtype)

    @staticmethod
    def imagenet(cutout=0, out_dtype=torch.float16):
        return TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, cutout, out_dtype)

    @staticmethod
    def raw_u8():
        return TailSpec(None, 0, False, CIFAR_MEAN, CIFAR_STD, 0, torch.uint8)

    def c_struct(self, h, w):
        oh, ow = self.out_size if self.out_size is not None else (h, w)
        t = _lib.Tail()
        t.out_h, t.out_w = int(oh), int(ow)
        t.out_dtype = _DTYPES[self.out_dtype]
        t.use_zero_box = 1 if self.cutout > 0 else 0
        t.crop_pad = int(self.crop_pad)
        for i in range(3):
            t.mean[i] = float(self.mean[i])
            t.std[i] = float(self.std[i])
        return t


class CompiledPolicy:
    """C-ABI policy handle for a reference-format policy list."""

    def __init__(self, policies):
        subs = [list(s) for s in policies]
        if not subs:
            raise IndexError("Cannot choose from an empty sequence")       # random.choice on []
        n_op = max(max(len(s) for s in subs), 1)
        # ragged sub-policies (the reference's Augmentation accepts them): short ones are padded with slots that never
        # fire (probability -1) and draw nothing - `pad[s][j]` marks them for the parity sampler
        self.pad = np.array([[j >= len(s) for j in range(n_op)] for s in subs], dtype=bool)
        subs = [s + [("Invert", -1.0, 0.0)] * (n_op - len(s)) for s in subs]
        self.policies = subs
        self.n_sub, self.n_op = len(subs), n_op
        self.names = [[str(op[0]) for op in s] for s in subs]
        ids = np.array([[_lib.op_id(op[0]) for op in s] for s in subs], dtype=np.int32)
        self.probs = np.array([[float(op[1]) for op in s] for s in subs], dtype=np.float64)
        self.levels = np.array([[float(op[2]) for op in s] for s in subs], dtype=np.float64)
        self.ids = ids
        h = C.c_void_p()
        check(lib.faa_policy_create(ids.ctypes.data, self.probs.ctypes.data, self.levels.ctypes.data,
                                    self.n_sub, self.n_op, C.byref(h)))
        self.handle = h
        self.draw = np.array([[lib.faa_policy_draw_kind(h, s, j) for j in range(n_op)]
                              for s in range(self.n_sub)], dtype=np.int8)

    def __del__(self):
        h = getattr(self, "handle", None)
        if h:
            try:
                lib.faa_policy_destroy(h)
            except Exception:
                pass
            self.handle = None

    # -- host-side compiled records (no GPU needed) -------------------------------------
    def compiled_op(self, h, w, sub, op, sign=0):
        out = np.zeros(8, dtype=np.int32)
        check(lib.faa_policy_compiled_op(self.handle, h, w, sub, op, int(sign), out.ctypes.data))
        return out

    def compiled_table(self, h, w):
        """[n_sub][n_op][2][8] int32; raises like the reference for the first bad op."""
        t = np.zeros((self.n_sub, self.n_op, 2, 8), dtype=np.int32)
        for s in range(self.n_sub):
            for j in range(self.n_op):
                for sg in range(2):
                    t[s, j, sg] = self.compiled_op(h, w, s, j, sg)
        return t

    def cutout_box(self, h, w, sub, op, ux, uy):
        b = np.zeros(1, dtype=_lib.BOX_DTYPE)
        check(lib.faa_cutout_box(self.handle, h, w, sub, op, float(ux), float(uy), b.ctypes.data))
        return b[0]

    # -- samplers -----------------------------------------------------------------------
    def sample_parity(self, batch, h, w, tail: TailSpec | None = None):
        """Replay the reference's draws from the global generators (see module doc)."""
        tail = tail or TailSpec.raw_u8()
        oh, ow = tail.out_size if tail.out_size is not None else (h, w)
        samples = np.zeros(batch, dtype=_lib.SAMPLE_DTYPE)
        boxes = np.zeros((batch, self.n_op), dtype=_lib.BOX_DTYPE)
        boxes["x1"] = -1
        boxes["y1"] = -1
        subs_range = range(self.n_sub)
        crop_rng_h = h + 2 * tail.crop_pad - oh + 1
        crop_rng_w = w + 2 * tail.crop_pad - ow + 1
        do_crop = tail.crop_pad > 0 or (oh, ow) != (h, w)
        if crop_rng_h < 1 or crop_rng_w < 1:
            raise ValueError("Required crop size %s is larger than input image size %s" %
                             ((oh, ow), (h + 2 * tail.crop_pad, w + 2 * tail.crop_pad)))
        if do_crop and (tail.crop_pad > 127 or crop_rng_h - 1 - tail.crop_pad > 127 or crop_rng_w - 1 - tail.crop_pad > 127):
            raise _lib.FaaRuntimeError("RandomCrop offsets beyond +-127 pixels are not supported (int8 records): "
                                       "crop on the host side")
        for i in range(batch):
            sub = random.choice(subs_range)                       # data.py:259
            gate = sign = 0
            for j in range(self.n_op):
                if self.pad[sub, j]:                              # padding of a ragged sub-policy: no op, no draw
                    continue
                if random.random() > self.probs[sub, j]:          # data.py:261
                    continue
                gate |= 1 << j
                d = self.draw[sub, j]
                if d < 0:
                    raise KeyError(self.names[sub][j])            # augmentations.py:189
                # validates the magnitude exactly when the reference would assert
                self.compiled_op(h, w, sub, j, 0)
                if d == _lib.DRAW_MIRROR:
                    if random.random() > 0.5:                     # augmentations.py:15 ...
                        sign |= 1 << j
                elif d == _lib.DRAW_BOX:
                    ux = np.random.random_sample()                # the u inside uniform(w), :131
                    uy = np.random.random_sample()                # :132
                    boxes[i, j] = self.cutout_box(h, w, sub, j, ux, uy)
            s = samples[i]
            s["sub"], s["gate"], s["sign"] = sub, gate, sign
            if do_crop and not (crop_rng_h == 1 and crop_rng_w == 1):     # torchvision RandomCrop.get_params
                top = int(torch.randint(0, crop_rng_h, size=(1,)).item())
                left = int(torch.randint(0, crop_rng_w, size=(1,)).item())
                s["crop_dy"], s["crop_dx"] = top - tail.crop_pad, left - tail.crop_pad
            if tail.hflip:
                s["flip"] = 1 if bool(torch.rand(1) < 0.5) else 0        # RandomHorizontalFlip
            if tail.cutout > 0:                                           # data.py:239-246
                cy = np.random.randint(oh)
                cx = np.random.randint(ow)
                half = tail.cutout // 2
                s["zero_box"] = (np.clip(cy - half, 0, oh), np.clip(cy + half, 0, oh),
                                 np.clip(cx - half, 0, ow), np.clip(cx + half, 0, ow))
        return samples, boxes

    def sample_policy_mt(self, batch, h, w, py_state=None, np_state=None):
        """C++ replay of the policy draws from explicit MT19937 states.  With the default
        arguments the live global states of ``random`` / ``numpy.random`` are read, advanced
        and written back - equivalent to the policy part of ``sample_parity``."""
        live = py_state is None and np_state is None
        if live:
            st = random.getstate()
            py_state = np.array(st[1], dtype=np.uint32)
            nst = np.random.get_state()
            np_state = np.concatenate([nst[1].astype(np.uint32), np.array([nst[2]], dtype=np.uint32)])
        py_state = np.ascontiguousarray(py_state, dtype=np.uint32)
        np_state = np.ascontiguousarray(np_state, dtype=np.uint32)
        samples = np.zeros(batch, dtype=_lib.SAMPLE_DTYPE)
        boxes = np.zeros((batch, self.n_op), dtype=_lib.BOX_DTYPE)
        check(lib.faa_sample_policy_mt(self.handle, batch, h, w, py_state.ctypes.data, np_state.ctypes.data,
                                       samples.ctypes.data, boxes.ctypes.data))
        if live:
            random.setstate((st[0], tuple(int(v) for v in py_state), st[2]))
            np.random.set_state((nst[0], np_state[:624].copy(), int(np_state[624]), nst[3], nst[4]))
        return samples, boxes, py_state, np_state


def make_rng(seed, first_index=0, tail: TailSpec | None = None):
    r = _lib.Rng()
    r.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    r.first_index = int(first_index)
    if tail is not None:
        r.crop_pad, r.hflip, r.zero_box_len = int(tail.crop_pad), int(bool(tail.hflip)), int(tail.cutout)
    return r


def _require_cuda(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise _lib.FaaRuntimeError("%s must be a CUDA tensor: the augmentation path is CUDA-only" % what)


def _stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def augment_batch(policy: CompiledPolicy, batch_u8: torch.Tensor, tail: TailSpec, samples=None, boxes=None,
                  rng=None, out=None, partner=None, lam=1.0, pool=None, pool_samples=None, pool_boxes=None,
                  first=0, lighting_rgb=None):
    """uint8 NHWC CUDA batch -> augmented NCHW ``tail.out_dtype`` (or uint8 NHWC).

    samples/boxes: resolved decisions (numpy structured arrays or CUDA uint8 tensors) - parity
    mode; or rng (``make_rng``) - fused Philox mode.  partner/lam: fused Mixup; ``pool`` is the
    array partner indexes into (defaults to ``batch_u8`` itself), ``first`` the position of this
    batch inside the pool (multi-GPU global pairing).

    A ``RaggedImages`` batch (differently sized images) is augmented image by image at its own size in one launch group
    (C ABI ``faa_augment_ragged``) and returned as a ``RaggedImages`` of the same sizes: ``tail`` must be
    ``TailSpec.raw_u8()``; ``out`` may be a ``RaggedImages`` of the same sizes; record i / global sample
    ``rng.first_index + i`` belongs to image i, drawn at its size.  No ``partner``, ``pool`` or ``lighting_rgb``.
    """
    if isinstance(batch_u8, RaggedImages):
        if partner is not None or pool is not None or lighting_rgb is not None:
            raise ValueError("a ragged batch takes no partner, pool or lighting_rgb: it is augmented at source size into uint8")
        return _augment_ragged(policy, batch_u8, tail, samples, boxes, rng, out)
    _require_cuda(batch_u8, "batch")
    if batch_u8.dtype != torch.uint8 or batch_u8.dim() != 4 or batch_u8.shape[-1] != 3:
        raise ValueError("batch must be uint8 [B, H, W, 3]")
    batch_u8 = batch_u8.contiguous()
    dev = batch_u8.device
    B, H, W, _ = batch_u8.shape
    t = tail.c_struct(H, W)
    if tail.out_dtype == torch.uint8:
        shape = (B, t.out_h, t.out_w, 3)
    else:
        shape = (B, 3, t.out_h, t.out_w)
    if out is None:
        out = torch.empty(shape, dtype=tail.out_dtype, device=dev)
    elif tuple(out.shape) != shape or out.dtype != tail.out_dtype or not out.is_contiguous():
        raise ValueError("out has the wrong shape/dtype")

    if lighting_rgb is not None:
        # Lighting (reference augmentations.py:197-215, between ToTensor and Normalize): per-image offsets [B,3] fp32
        lighting_rgb = lighting_rgb.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(lighting_rgb.shape) != (B, 3):
            raise ValueError("lighting_rgb must be [B, 3]")
        policy._lighting_keep = lighting_rgb                 # stays alive until the launch has run
        check(lib.faa_policy_set_lighting(policy.handle, lighting_rgb.data_ptr(), B))
    try:
        return _augment_launch(policy, batch_u8, tail, samples, boxes, rng, out, partner, lam, pool, pool_samples, pool_boxes,
                               first, dev, B, H, W, t)
    finally:
        if lighting_rgb is not None:
            check(lib.faa_policy_set_lighting(policy.handle, None, 0))


def _augment_launch(policy, batch_u8, tail, samples, boxes, rng, out, partner, lam, pool, pool_samples, pool_boxes, first, dev,
                    B, H, W, t):
    def to_dev(a, itemsize):
        if a is None:
            return None
        if isinstance(a, torch.Tensor):
            _require_cuda(a, "records")
            return a
        flat = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        return torch.from_numpy(flat.copy()).to(dev, non_blocking=False)

    with torch.cuda.device(dev):
        stream = _stream_ptr(dev)
        rng_p = C.byref(rng) if rng is not None else None
        if partner is None:
            d_s, d_b = to_dev(samples, 16), to_dev(boxes, 8)
            n_op = policy.n_op
            if n_op <= _lib.MAX_FUSED_OPS:
                check(lib.faa_augment(policy.handle, batch_u8.data_ptr(), out.data_ptr(), B, H, W, C.byref(t),
                                      d_s.data_ptr() if d_s is not None else None,
                                      d_b.data_ptr() if d_b is not None else None, rng_p, 0, stream))
            else:
                # chained launches: every window of 2 ops but the last writes uint8 HWC
                mid = _lib.Tail()
                mid.out_h, mid.out_w, mid.out_dtype, mid.use_zero_box = H, W, _lib.U8_HWC, 0
                cur = batch_u8
                base = 0
                while base + _lib.MAX_FUSED_OPS < n_op:
                    nxt = torch.empty_like(batch_u8)
                    check(lib.faa_augment(policy.handle, cur.data_ptr(), nxt.data_ptr(), B, H, W, C.byref(mid),
                                          d_s.data_ptr() if d_s is not None else None,
                                          d_b.data_ptr() if d_b is not None else None, rng_p, base, stream))
                    cur = nxt
                    base += _lib.MAX_FUSED_OPS
                check(lib.faa_augment(policy.handle, cur.data_ptr(), out.data_ptr(), B, H, W, C.byref(t),
                                      d_s.data_ptr() if d_s is not None else None,
                                      d_b.data_ptr() if d_b is not None else None, rng_p, base, stream))
        else:
            pool_t = batch_u8 if pool is None else pool.contiguous()
            _require_cuda(pool_t, "pool")
            d_s = to_dev(samples if pool_samples is None else pool_samples, 16)
            d_b = to_dev(boxes if pool_boxes is None else pool_boxes, 8)
            if isinstance(partner, torch.Tensor):
                d_p = partner.to(device=dev, dtype=torch.int32).contiguous()
            else:
                d_p = torch.as_tensor(np.asarray(partner, dtype=np.int32), device=dev)
            check(lib.faa_augment_mixup(policy.handle, pool_t.data_ptr(), int(pool_t.shape[0]), int(first),
                                        out.data_ptr(), B, H, W, C.byref(t),
                                        d_s.data_ptr() if d_s is not None else None,
                                        d_b.data_ptr() if d_b is not None else None, rng_p,
                                        d_p.data_ptr(), float(np.float32(lam)), float(np.float32(1 - lam)),
                                        stream))
    return out


class FusedAugmenter:
    """Pre-bound production launch: fused Philox sampling + augmentation in ONE kernel launch and
    one ctypes call per batch (no per-call Python allocation), for 2-op policies.

        aug = FusedAugmenter(policy, tail, h, w, seed)
        aug(batch_u8_cuda, out_cuda, first_index)     # asynchronous on the current stream
    """

    def __init__(self, policy: CompiledPolicy, tail: TailSpec, h: int, w: int, seed: int = 0, overlap_calls: bool = False):
        """``overlap_calls=True``: consecutive ``__call__``s on one stream may overlap on the GPU (C ABI
        ``faa_policy_set_overlap``) - only if every call's input batch was complete before the PREVIOUS call was issued
        (device-resident data, a producer that runs a batch ahead).  ``run_many`` overlaps its steps regardless."""
        if policy.n_op > _lib.MAX_FUSED_OPS:
            raise ValueError("FusedAugmenter handles policies of at most 2 ops; use augment_batch")
        if overlap_calls:
            check(lib.faa_policy_set_overlap(policy.handle, 1))
        self.policy, self.tail, self.h, self.w = policy, tail, h, w
        self.t = tail.c_struct(h, w)
        self.rng = make_rng(seed, 0, tail)
        self._t_ref, self._rng_ref = C.byref(self.t), C.byref(self.rng)
        self.out_shape = ((0, self.t.out_h, self.t.out_w, 3) if tail.out_dtype == torch.uint8
                          else (0, 3, self.t.out_h, self.t.out_w))

    def empty_out(self, batch, device="cuda"):
        return torch.empty((batch,) + tuple(self.out_shape[1:]), dtype=self.tail.out_dtype, device=device)

    def __call__(self, batch_u8: torch.Tensor, out: torch.Tensor, first_index: int = 0, stream=None):
        b = batch_u8.shape[0]
        if (batch_u8.dtype != torch.uint8 or not batch_u8.is_cuda or not batch_u8.is_contiguous()
                or tuple(batch_u8.shape[1:]) != (self.h, self.w, 3)):
            raise ValueError("batch must be a contiguous uint8 CUDA tensor [B, %d, %d, 3]" % (self.h, self.w))
        if (out.dtype != self.tail.out_dtype or out.device != batch_u8.device or not out.is_contiguous()
                or tuple(out.shape) != (b,) + tuple(self.out_shape[1:])):
            raise ValueError("out must be a contiguous %s tensor %s on %s" % (self.tail.out_dtype, (b,) + tuple(self.out_shape[1:]),
                                                                             batch_u8.device))
        self.rng.first_index = first_index
        dev = batch_u8.device
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        if dev.index == torch.cuda.current_device():
            check(lib.faa_augment(self.policy.handle, batch_u8.data_ptr(), out.data_ptr(), b, self.h,
                                  self.w, self._t_ref, None, None, self._rng_ref, 0, C.c_void_p(s)))
        else:
            with torch.cuda.device(dev):
                check(lib.faa_augment(self.policy.handle, batch_u8.data_ptr(), out.data_ptr(), b, self.h,
                                      self.w, self._t_ref, None, None, self._rng_ref, 0, C.c_void_p(s)))
        return out


    def plan_many(self, batches, outs):
        """Pointer tables for :meth:`run_many` (build once, reuse every epoch): validates the tensors like ``__call__``."""
        if len(batches) != len(outs) or not batches:
            raise ValueError("need as many outputs as batches (at least one)")
        b = batches[0].shape[0]
        for x, o in zip(batches, outs):
            if (x.dtype != torch.uint8 or not x.is_cuda or not x.is_contiguous() or tuple(x.shape) != (b, self.h, self.w, 3)):
                raise ValueError("every batch must be a contiguous uint8 CUDA tensor [%d, %d, %d, 3]" % (b, self.h, self.w))
            if (o.dtype != self.tail.out_dtype or o.device != x.device or x.device != batches[0].device or not o.is_contiguous()
                    or tuple(o.shape) != (b,) + tuple(self.out_shape[1:])):
                raise ValueError("every out must be a contiguous %s tensor %s on the batches' device"
                                 % (self.tail.out_dtype, (b,) + tuple(self.out_shape[1:])))
        n = len(batches)
        ins = (C.c_void_p * n)(*[x.data_ptr() for x in batches])
        dst = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
        return (n, b, ins, dst, batches[0].device, list(batches), list(outs))      # (keeps the tensors alive)

    def run_many(self, plan, first_index: int = 0, stride=None, stream=None):
        """Augment the planned batches back to back in ONE call (C ABI ``faa_augment_many``): step k == ``self(batches[k],
        outs[k], first_index + k * stride)``; ``stride`` defaults to the batch size."""
        n, b, ins, dst, dev = plan[:5]
        self.rng.first_index = first_index
        s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            check(lib.faa_augment_many(self.policy.handle, n, ins, dst, b, self.h, self.w, self._t_ref, self._rng_ref,
                                       int(b if stride is None else stride), C.c_void_p(s)))
        return plan[6]


def augment_tta(policy: CompiledPolicy, batch_u8: torch.Tensor, tail: TailSpec, replicas: int, seed: int, first_index: int = 0,
                out=None):
    """Test-time-augmentation batching for the policy search (reference search.py:87-125): the reference builds
    ``num_policy`` validation loaders that each augment the SAME validation batch with their own random draws and then
    reduces the per-sample losses over the replicas.  Here ONE launch produces all replicas:

        out[r] == augment_batch(policy, batch_u8, tail, rng=make_rng(seed, first_index + r * B, tail))

    uint8 [B,H,W,3] CUDA batch -> [replicas, B, 3, out_h, out_w] (or [replicas, B, out_h, out_w, 3] uint8).

    A ``RaggedImages`` batch (``tail`` must be ``TailSpec.raw_u8()``) gives a ``RaggedImages`` of replicas * B images
    in replica-major order, each at its source size: one ``faa_augment_ragged`` launch group over replicas * B
    descriptors (``tta_select``) into the batch's storage, so image r * B + i is
    ``augment_batch(policy, batch, tail, rng=make_rng(seed, first_index + r * B, tail))``'s image i.  ``out`` may be a
    ``RaggedImages`` of those sizes."""
    if isinstance(batch_u8, RaggedImages):
        check_tta(len(batch_u8), replicas)
        return _augment_ragged(policy, tta_select(batch_u8, replicas), tail, None, None,
                               make_rng(seed, first_index, tail), out)
    _require_cuda(batch_u8, "batch")
    if batch_u8.dtype != torch.uint8 or batch_u8.dim() != 4 or batch_u8.shape[-1] != 3:
        raise ValueError("batch must be uint8 [B, H, W, 3]")
    batch_u8 = batch_u8.contiguous()
    B, H, W, _ = batch_u8.shape
    t = tail.c_struct(H, W)
    shape = (replicas, B, t.out_h, t.out_w, 3) if tail.out_dtype == torch.uint8 else (replicas, B, 3, t.out_h, t.out_w)
    if out is None:
        out = torch.empty(shape, dtype=tail.out_dtype, device=batch_u8.device)
    elif tuple(out.shape) != shape or out.dtype != tail.out_dtype or not out.is_contiguous():
        raise ValueError("out has the wrong shape/dtype")
    rng = make_rng(seed, first_index, tail)
    with torch.cuda.device(batch_u8.device):
        check(lib.faa_augment_tta(policy.handle, batch_u8.data_ptr(), out.data_ptr(), B, int(replicas), H, W, C.byref(t),
                                  C.byref(rng), _stream_ptr(batch_u8.device)))
    return out


MAX_LAUNCH_IMAGES = 65535          # images per launch (one grid row each)


def check_tta(batch, replicas):
    """ValueError unless ``replicas`` >= 1 and the ``replicas * batch`` images of a TTA call fit in one launch"""
    if int(replicas) != replicas or replicas < 1:
        raise ValueError("replicas must be a positive integer, not %r" % (replicas,))
    if int(replicas) * int(batch) > MAX_LAUNCH_IMAGES:
        raise ValueError("replicas * batch = %d images: at most %d per launch" % (int(replicas) * int(batch),
                                                                                MAX_LAUNCH_IMAGES))


def compile_policies(policies):
    """The candidates of a multi-policy TTA call as ``CompiledPolicy`` handles: each item is a ``CompiledPolicy``, an
    object holding one as ``compiled`` (``data.Augmentation``) or a reference-format policy list (what the search's
    ``policy_decoder`` returns for one hyperopt suggestion)."""
    out = []
    for p in policies:
        if isinstance(p, CompiledPolicy):
            out.append(p)
        elif isinstance(getattr(p, "compiled", None), CompiledPolicy):
            out.append(p.compiled)
        else:
            out.append(CompiledPolicy(p))
    return out


def check_tta_policies(policies, batch, replicas):
    """ValueError for a multi-policy TTA call (``augment_tta_policies``) of ``CompiledPolicy`` candidates that the
    library refuses: what ``check_tta`` refuses, no candidate, one handle given twice, candidates of different op counts
    or of more than one fused window, and more than 65535 entries (candidates * replicas * batch) per launch"""
    check_tta(batch, replicas)
    if len(policies) == 0:
        raise ValueError("need at least one candidate policy")
    if len({id(p) for p in policies}) != len(policies):
        raise ValueError("a candidate policy is given twice: build one CompiledPolicy per candidate")
    n_op = sorted({p.n_op for p in policies})
    if len(n_op) != 1:
        raise ValueError("every candidate needs the same number of ops per sub-policy, not %s" % n_op)
    if n_op[0] > _lib.MAX_FUSED_OPS:
        raise ValueError("tta supports policies of at most %d ops per sub-policy (replicated launches)"
                         % _lib.MAX_FUSED_OPS)
    n = len(policies) * int(replicas) * int(batch)
    if n > MAX_LAUNCH_IMAGES:
        raise ValueError("candidates * replicas * batch = %d images: at most %d per launch" % (n, MAX_LAUNCH_IMAGES))


def tta_policy_entries(n_policies, batch, replicas):
    """(candidate, replica, image) int64 arrays of the n_policies * replicas * batch schedule entries of a multi-policy
    TTA call: entry v = (t * replicas + r) * batch + i"""
    v = np.arange(int(n_policies) * int(replicas) * int(batch), dtype=np.int64)
    return v // (int(replicas) * int(batch)), (v // int(batch)) % int(replicas), v % int(batch)


def augment_tta_policies(policies, batch_u8, tail: TailSpec, replicas: int, seed: int, first_index: int = 0, out=None):
    """``augment_tta`` for T candidate policies at once (the policy search scoring several suggestions against one
    validation fold): ONE resolve launch and the pixel launches of one replicated launch over T * replicas * B entries
    (C ABI ``faa_augment_tta_policies``).  ``policies``: what ``compile_policies`` takes.

        out[t] == augment_tta(policies[t], batch_u8, tail, replicas, seed, first_index + t * replicas * B)

    uint8 [B,H,W,3] CUDA batch -> [T, replicas, B, 3, out_h, out_w] (or [T, replicas, B, out_h, out_w, 3] uint8).
    A ``RaggedImages`` batch (``tail`` must be ``TailSpec.raw_u8()``) gives a ``RaggedImages`` of T * replicas * B
    images in that entry order, each at its source size (``faa_augment_ragged_policies`` over replicated descriptors).
    Raises ValueError before any device work for what ``check_tta_policies`` refuses."""
    pols = compile_policies(policies)
    B = len(batch_u8) if isinstance(batch_u8, RaggedImages) else int(batch_u8.shape[0])
    check_tta_policies(pols, B, replicas)
    T, K = len(pols), int(replicas)
    handles = (C.c_void_p * T)(*[p.handle.value for p in pols])
    rng = make_rng(seed, first_index, tail)
    if isinstance(batch_u8, RaggedImages):
        raw = TailSpec.raw_u8()
        if (tail.out_size, tail.crop_pad, tail.hflip, tail.cutout, tail.out_dtype) != \
                (raw.out_size, raw.crop_pad, raw.hflip, raw.cutout, raw.out_dtype):
            raise ValueError("a ragged batch is augmented at each image's own size into uint8: the tail must be "
                             "TailSpec.raw_u8()")
        src = tta_select(batch_u8, T * K)
        _require_cuda(src.storage, "batch")
        if out is None:
            out = RaggedImages.empty(src.sizes, src.device)
        elif not isinstance(out, RaggedImages) or not np.array_equal(out.sizes, src.sizes) or out.device != src.device:
            raise ValueError("out must be a RaggedImages of the replicated batch's sizes on its device")
        if len(src) == 0:
            return out
        cand = np.ascontiguousarray(tta_policy_entries(T, B, K)[0].astype(np.int32))
        (h_in, d_in), (h_out, d_out) = src.descriptors(), out.descriptors()
        with torch.cuda.device(src.device):
            check(lib.faa_augment_ragged_policies(handles, T, h_in.ctypes.data, d_in.data_ptr(), cand.ctypes.data, len(src),
                                                  h_out.ctypes.data, d_out.data_ptr(), C.byref(rng),
                                                  _stream_ptr(src.device)))
        return out
    _require_cuda(batch_u8, "batch")
    if batch_u8.dtype != torch.uint8 or batch_u8.dim() != 4 or batch_u8.shape[-1] != 3:
        raise ValueError("batch must be uint8 [B, H, W, 3]")
    batch_u8 = batch_u8.contiguous()
    _, H, W, _ = batch_u8.shape
    t = tail.c_struct(H, W)
    shape = (T, K, B, t.out_h, t.out_w, 3) if tail.out_dtype == torch.uint8 else (T, K, B, 3, t.out_h, t.out_w)
    if out is None:
        out = torch.empty(shape, dtype=tail.out_dtype, device=batch_u8.device)
    elif tuple(out.shape) != shape or out.dtype != tail.out_dtype or not out.is_contiguous():
        raise ValueError("out has the wrong shape/dtype")
    with torch.cuda.device(batch_u8.device):
        check(lib.faa_augment_tta_policies(handles, T, batch_u8.data_ptr(), out.data_ptr(), B, K, H, W, C.byref(t),
                                           C.byref(rng), _stream_ptr(batch_u8.device)))
    return out


def tta_positions(batch, replicas):
    """int64 [replicas * batch]: the batch position each TTA schedule entry v = r * batch + i reads (i)"""
    return np.tile(np.arange(int(batch), dtype=np.int64), int(replicas))


def tta_select(batch: RaggedImages, replicas):
    """``replicas`` copies of the batch's descriptors, replica-major, into the same storage (no pixel is copied)"""
    return batch.select(tta_positions(len(batch), replicas))


def crop_cfg(img_size, center=False, min_covered=0.1, aspect_ratio_range=(3. / 4, 4. / 3), area_range=(0.08, 1.0),
             max_attempts=10, seed=0, first_index=0):
    """``faa_crop_cfg_t`` of EfficientNetRandomCrop / EfficientNetCenterCrop(img_size) (reference data.py:267-345);
    ``seed`` / ``first_index`` key the device crop sampler (Philox, global sample index first_index + i)."""
    c = _lib.CropCfg()
    c.mode = _lib.CROP_CENTER if center else _lib.CROP_RANDOM
    c.img_size = int(img_size)
    c.min_covered = float(min_covered)
    c.aspect_lo, c.aspect_hi = float(aspect_ratio_range[0]), float(aspect_ratio_range[1])
    c.area_lo, c.area_hi = float(area_range[0]), float(area_range[1])
    c.max_attempts = int(max_attempts)
    c.rng = make_rng(seed, first_index)
    return c


def center_crop_box(h, w, img_size):
    """(x0, y0, w, h) of EfficientNetCenterCrop(img_size) on an h x w image (C ABI ``faa_center_crop_box``)."""
    b = np.zeros(1, dtype=_lib.CROP_BOX_DTYPE)
    check(lib.faa_center_crop_box(int(h), int(w), int(img_size), b.ctypes.data))
    return tuple(int(v) for v in b[0])


class RaggedImages:
    """A batch or dataset of differently sized uint8 HWC images in one byte buffer (on the device for every launch).

    ``storage``: 1-D uint8 tensor; image i is ``sizes[i] = (h, w)`` rows of ``w * 3`` bytes starting at byte
    ``offsets[i]`` (host int64 [N]; ``sizes`` host int32 [N, 2]).  Several descriptors may share bytes or leave gaps:
    ``select`` makes new descriptors into the same storage without copying a pixel."""

    def __init__(self, storage: torch.Tensor, offsets, sizes):
        if not isinstance(storage, torch.Tensor) or storage.dtype != torch.uint8 or storage.dim() != 1 \
                or not storage.is_contiguous():
            raise ValueError("storage must be a contiguous 1-D uint8 tensor")
        self.storage = storage
        self.offsets = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
        self.sizes = np.ascontiguousarray(sizes, dtype=np.int32).reshape(-1, 2)
        if len(self.offsets) != len(self.sizes):
            raise ValueError("need one offset per size")
        if len(self.sizes) and (int(self.sizes.min()) < 1 or int(self.offsets.min()) < 0 or
                                int((self.offsets + self.nbytes()).max()) > storage.numel()):
            raise ValueError("every image must be at least 1 x 1 and lie inside the storage")
        self._desc = None

    @staticmethod
    def from_list(images, device="cuda"):
        """uint8 HWC images (NumPy arrays or CUDA tensors), packed back to back with one copy."""
        sizes = np.array([tuple(int(v) for v in a.shape[:2]) for a in images], dtype=np.int32).reshape(-1, 2)
        for a in images:
            u8 = a.dtype == torch.uint8 if isinstance(a, torch.Tensor) else np.asarray(a).dtype == np.uint8
            if not u8 or a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("every image must be uint8 [H, W, 3]")
        n = sizes[:, 0].astype(np.int64) * sizes[:, 1] * 3
        offsets = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int64)
        if len(images) and all(isinstance(a, torch.Tensor) and a.device == torch.device(device) for a in images):
            storage = torch.cat([a.reshape(-1) for a in images]).to(device)
        else:
            host = np.empty(int(n.sum()), np.uint8)
            for a, o, k in zip(images, offsets, n):
                host[o:o + k] = (a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)).reshape(-1)
            storage = torch.from_numpy(host).to(device)
        return RaggedImages(storage, offsets, sizes)

    @staticmethod
    def empty(sizes, device="cuda"):
        """uninitialised images of the given (h, w) sizes, each starting on a 16-byte boundary of a fresh allocation"""
        sizes = np.ascontiguousarray(sizes, dtype=np.int32).reshape(-1, 2)
        slot = (sizes[:, 0].astype(np.int64) * sizes[:, 1] * 3 + 15) // 16 * 16
        storage = torch.empty(int(slot.sum()), dtype=torch.uint8, device=device)
        return RaggedImages(storage, np.cumsum(slot) - slot, sizes)

    def __len__(self):
        return len(self.sizes)

    @property
    def device(self):
        return self.storage.device

    def nbytes(self):
        """bytes of each image, int64 [N]"""
        return self.sizes[:, 0].astype(np.int64) * self.sizes[:, 1] * 3

    def select(self, idx):
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        return RaggedImages(self.storage, self.offsets[idx], self.sizes[idx])

    def image(self, i):
        """uint8 [h, w, 3] view of image i"""
        h, w = (int(v) for v in self.sizes[i])
        o = int(self.offsets[i])
        return self.storage[o:o + h * w * 3].view(h, w, 3)

    def groups(self):
        """[((h, w), positions)]: the batch positions of each distinct size, in batch order, sizes in order of their first
        image"""
        out = {}
        for i, (h, w) in enumerate(self.sizes.tolist()):
            out.setdefault((h, w), []).append(i)
        return [(k, np.array(v, dtype=np.int64)) for k, v in out.items()]

    def descriptors(self):
        """(host ``IMAGE_DTYPE`` [N], device uint8 copy of it): the ``faa_image_t`` arrays of ``faa_crop_resize_ragged``"""
        if self._desc is None:
            d = np.zeros(len(self), dtype=_lib.IMAGE_DTYPE)
            d["data"] = self.storage.data_ptr() + self.offsets.astype(np.uint64)
            d["h"], d["w"] = self.sizes[:, 0], self.sizes[:, 1]
            self._desc = (d, torch.from_numpy(d.view(np.uint8).copy()).to(self.device))
        return self._desc


def parse_jpeg(f):
    """(header ``JPEG_HEADER_DTYPE`` [1], its tables ``JPEG_TABLE_DTYPE`` [9]) of one file (C ABI ``faa_jpeg_parse`` +
    ``faa_jpeg_tables``; ctypes releases the GIL during both), or (None, reason) when the decoder does not take it"""
    hdr = np.zeros(1, dtype=_lib.JPEG_HEADER_DTYPE)
    if lib.faa_jpeg_parse(f, len(f), hdr.ctypes.data) != _lib.OK:
        return None, (lib.faa_last_error() or b"").decode()
    tabs = np.zeros(9, dtype=_lib.JPEG_TABLE_DTYPE)
    check(lib.faa_jpeg_tables(f, len(f), hdr.ctypes.data, tabs.ctypes.data))
    return hdr, tabs


def parse_jpeg_progressive(f):
    """(header [1], its tables ``JPEG_TABLE_DTYPE`` [3 + 6 S], its scans ``JPEG_SCAN_DTYPE`` [S]) of one progressive
    file (C ABI ``faa_jpeg_parse_progressive`` + ``faa_jpeg_scan_tables``): tables [0, 3) are the components'
    quantisation tables, 3 + 6 s + k slot k of scan s.  (None, reason, None) when the decoder does not take it."""
    hdr = np.zeros(1, dtype=_lib.JPEG_HEADER_DTYPE)
    scans = np.zeros(_lib.JPEG_MAX_SCANS, dtype=_lib.JPEG_SCAN_DTYPE)
    n = C.c_int(0)
    if lib.faa_jpeg_parse_progressive(f, len(f), hdr.ctypes.data, scans.ctypes.data, len(scans), C.byref(n)) != _lib.OK:
        return None, (lib.faa_last_error() or b"").decode(), None
    scans = scans[:n.value].copy()
    tabs = np.zeros(3 + 6 * len(scans), dtype=_lib.JPEG_TABLE_DTYPE)
    check(lib.faa_jpeg_scan_tables(f, len(f), hdr.ctypes.data, scans.ctypes.data, len(scans), tabs.ctypes.data))
    return hdr, tabs, scans


def _parse_any(f):
    """``parse_jpeg``, and for a file it refuses as progressive ``parse_jpeg_progressive``: (header, tables, scans or
    None), or (None, reason, None)"""
    hdr, tabs = parse_jpeg(f)
    if hdr is None and tabs.endswith(": progressive coding"):
        return parse_jpeg_progressive(f)
    return hdr, tabs, None


def parse_jpeg_headers(files, map=map, progressive=False, progressive_index=False):
    """JPEG files (``bytes``) -> (headers [N], table pool, refused [(position, reason)]).  The tables the files use are
    deduplicated into the pool in order of first use, which the headers' ``pool`` slots index; a refused file's header
    row stays zero and adds nothing to the pool.  ``offset`` is left 0: the caller places the files.  ``map`` runs the
    per-file parse (an executor's ``map`` parses files in parallel).

    ``progressive=True`` also takes progressive files (``parse_jpeg_progressive``; their headers' ``reserved`` is
    ``JPEG_PROGRESSIVE``), their scans' Huffman tables going into the same pool, and returns ``(headers, pool, refused,
    scans, scan_first)``: ``JPEG_SCAN_DTYPE`` scans with pool slots set, file i's being
    ``scans[scan_first[i]:scan_first[i + 1]]`` (none for the other files).

    ``progressive_index=True`` (with ``progressive``) marks progressive files as taking a scan index: ``reserved`` is
    ``JPEG_PROGRESSIVE | JPEG_SCAN_INDEXED`` and ``scan_len`` the sum of their scans' lengths (the scan axis of
    ``faa_jpeg.cuh``), so they are indexed, recorded and learned as baseline files are."""
    if progressive_index and not progressive:
        raise ValueError("progressive_index needs progressive=True")
    headers = np.zeros(len(files), dtype=_lib.JPEG_HEADER_DTYPE)
    pool, index, refused = [], {}, []
    scans, counts = [], np.zeros(len(files), np.int64)

    def slot_of(t):
        key = t.tobytes()
        if key not in index:
            index[key] = len(pool)
            pool.append(t.copy())
        return index[key]

    for i, parsed in enumerate(map(_parse_any if progressive else parse_jpeg, files)):
        hdr, tabs = parsed[0], parsed[1]
        if hdr is None:
            refused.append((i, tabs))
            continue
        headers[i] = hdr[0]
        nc = int(hdr["ncomp"][0])
        if progressive and parsed[2] is not None:
            sc = parsed[2]
            for c in range(nc):
                headers["pool"][i, c] = slot_of(tabs[c])
            for k in range(len(sc)):
                for t in range(6):
                    if (sc["dc_at"][k] if t < 3 else sc["ac_at"][k])[t % 3] != -1:
                        sc["pool"][k, t] = slot_of(tabs[3 + 6 * k + t])
            scans.append(sc)
            counts[i] = len(sc)
            if progressive_index:
                headers["reserved"][i] = _lib.JPEG_PROGRESSIVE | _lib.JPEG_SCAN_INDEXED
                headers["scan_len"][i] = int(sc["len"].sum())
            continue
        for slot in range(9):
            if slot % 3 >= nc:
                continue
            headers["pool"][i, slot] = slot_of(tabs[slot])
    pool = np.array(pool, dtype=_lib.JPEG_TABLE_DTYPE).reshape(-1)
    if not progressive:
        return headers, pool, refused
    scan_first = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    scans = np.concatenate(scans) if scans else np.zeros(0, _lib.JPEG_SCAN_DTYPE)
    return headers, pool, refused, scans, scan_first


class EncodedImages:
    """A batch or dataset of JPEG files: their bytes packed back to back in one device buffer, their headers parsed once
    on the host (C ABI ``faa_jpeg_parse``), and the quantisation and Huffman tables they use deduplicated into one table
    pool.  ``headers`` (host ``JPEG_HEADER_DTYPE`` [N]) is what ``decode_jpeg`` validates and plans from; their device
    copy and the pool's are made on first use.  ``select`` makes a batch of some of the files without copying a byte of
    them.

    Optionally the files carry a scan index (``build_jpeg_index``): ``first`` (int64 [N + 1]) and ``points``
    (``JPEG_SYNC_DTYPE``), file i's points being ``points[first[i]:first[i + 1]]``.  ``decode_jpeg`` then decodes each
    indexed file on many threads; the pixels and status are those of the decode without the index, whatever it holds.

    Progressive files (``from_bytes(..., progressive=True)``) carry their scans the same way: ``scan_first`` (int64
    [N + 1]) and ``scans`` (``JPEG_SCAN_DTYPE``), file i's being ``scans[scan_first[i]:scan_first[i + 1]]``; the other
    files have none.  Without them every header must be a baseline one."""

    def __init__(self, storage: torch.Tensor, headers, pool, _d_pool=None, _d_headers=None, first=None, points=None,
                 _d_first=None, _d_points=None, scans=None, scan_first=None, _d_scans=None, _d_scan_first=None):
        """``_d_pool`` / ``_d_headers`` / ``_d_first`` / ``_d_points`` / ``_d_scans`` / ``_d_scan_first``: device copies
        of ``pool`` / ``headers`` / ``first`` / ``points`` / ``scans`` / ``scan_first`` the caller already made (uint8
        tensors of their bytes, ``first`` and ``scan_first`` int64), used instead of uploading them on first use"""
        if not isinstance(storage, torch.Tensor) or storage.dtype != torch.uint8 or storage.dim() != 1 \
                or not storage.is_contiguous():
            raise ValueError("storage must be a contiguous 1-D uint8 tensor")
        self.storage = storage
        self.headers = np.ascontiguousarray(headers, dtype=_lib.JPEG_HEADER_DTYPE).reshape(-1)
        self.pool = np.ascontiguousarray(pool, dtype=_lib.JPEG_TABLE_DTYPE).reshape(-1)
        h = self.headers
        if len(h) and (int(h["offset"].min()) < 0 or int((h["offset"] + h["len"]).max()) > storage.numel()):
            raise ValueError("every file must lie inside the storage")
        if (first is None) != (points is None):
            raise ValueError("a scan index needs both first and points")
        self.first = self.points = None
        if first is not None:
            self.first = np.ascontiguousarray(first, dtype=np.int64).reshape(-1)
            self.points = np.ascontiguousarray(points, dtype=_lib.JPEG_SYNC_DTYPE).reshape(-1)
            f = self.first
            if len(f) != len(h) + 1 or f[0] != 0 or (np.diff(f) < 0).any() or f[-1] > len(self.points):
                raise ValueError("first must be [N + 1] non-decreasing offsets from 0 into points")
        if (scans is None) != (scan_first is None):
            raise ValueError("scans need both scans and scan_first")
        self.scans = self.scan_first = None
        if scans is not None:
            self.scans = np.ascontiguousarray(scans, dtype=_lib.JPEG_SCAN_DTYPE).reshape(-1)
            self.scan_first = np.ascontiguousarray(scan_first, dtype=np.int64).reshape(-1)
            f = self.scan_first
            if len(f) != len(h) + 1 or f[0] != 0 or (np.diff(f) < 0).any() or f[-1] > len(self.scans):
                raise ValueError("scan_first must be [N + 1] non-decreasing offsets from 0 into scans")
        if self.scans is None and self.progressive().any():
            raise ValueError("progressive files need their scans")
        self._d_pool = _d_pool
        self._d_headers = _d_headers
        self._d_first = _d_first
        self._d_points = _d_points
        self._d_scans = _d_scans
        self._d_scan_first = _d_scan_first

    @staticmethod
    def from_bytes(files, device="cuda", progressive=False, progressive_index=False):
        """JPEG files (``bytes``) -> EncodedImages on ``device``.  Raises ValueError naming every file the decoder
        does not take (progressive, arithmetic, 12-bit, CMYK, other sampling, malformed ...) and why.
        ``progressive=True`` takes progressive files too, and ``progressive_index=True`` lets them take a scan index
        (``parse_jpeg_headers``)."""
        if progressive_index and not progressive:
            raise ValueError("progressive_index needs progressive=True")
        files = [bytes(f) for f in files]
        scans = scan_first = None
        if progressive:
            headers, pool, refused, scans, scan_first = parse_jpeg_headers(files, progressive=True,
                                                                           progressive_index=progressive_index)
        else:
            headers, pool, refused = parse_jpeg_headers(files)
        if refused:
            raise ValueError("JPEG files the decoder does not take: " + "; ".join("%d: %s" % r for r in refused))
        lengths = np.array([len(f) for f in files], dtype=np.int64)
        headers["offset"] = np.cumsum(lengths) - lengths
        packed = np.frombuffer(b"".join(files), dtype=np.uint8)
        storage = torch.from_numpy(packed.copy()).to(device) if packed.size else torch.zeros(1, dtype=torch.uint8,
                                                                                              device=device)
        return EncodedImages(storage, headers, pool, scans=scans, scan_first=scan_first)

    def __len__(self):
        return len(self.headers)

    @property
    def device(self):
        return self.storage.device

    @property
    def sizes(self):
        """(h, w) of every image, int32 [N, 2]"""
        return np.stack([self.headers["h"], self.headers["w"]], axis=1).astype(np.int32).reshape(-1, 2)

    def progressive(self):
        """bool [N]: which files are progressive"""
        return (self.headers["reserved"] & _lib.JPEG_PROGRESSIVE) != 0

    def progressive_indexed(self):
        """bool [N]: which files are progressive and take a scan index (``progressive_index=True``)"""
        return self.headers["reserved"] == _lib.JPEG_PROGRESSIVE | _lib.JPEG_SCAN_INDEXED

    def with_index(self, first, points):
        """the same files carrying the scan index (first, points), e.g. ``build_jpeg_index``'s"""
        return EncodedImages(self.storage, self.headers, self.pool, self.device_pool(), self._d_headers, first, points,
                             scans=self.scans, scan_first=self.scan_first, _d_scans=self._d_scans,
                             _d_scan_first=self._d_scan_first)

    def select(self, idx):
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        first, points = _gather_ranges(self.first, self.points, idx)
        scan_first, scans = _gather_ranges(self.scan_first, self.scans, idx)
        return EncodedImages(self.storage, self.headers[idx], self.pool, self.device_pool(), first=first, points=points,
                             scans=scans, scan_first=scan_first)

    def device_pool(self):
        """the table pool on the device (shared by every ``select`` of this set)"""
        if self._d_pool is None:
            flat = self.pool.view(np.uint8).reshape(-1)
            self._d_pool = torch.from_numpy(flat.copy() if flat.size else np.zeros(1, np.uint8)).to(self.device)
        return self._d_pool

    def device_headers(self):
        if self._d_headers is None:
            flat = self.headers.view(np.uint8).reshape(-1)
            self._d_headers = torch.from_numpy(flat.copy() if flat.size else np.zeros(1, np.uint8)).to(self.device)
        return self._d_headers

    def device_scans(self):
        """(scans, scan_first) on the device: the scans' bytes and int64 [N + 1]"""
        if self._d_scans is None:
            flat = self.scans.view(np.uint8).reshape(-1)
            self._d_scans = torch.from_numpy(flat.copy() if flat.size else np.zeros(112, np.uint8)).to(self.device)
        if self._d_scan_first is None:
            self._d_scan_first = torch.from_numpy(self.scan_first.copy()).to(self.device)
        return self._d_scans, self._d_scan_first

    def device_index(self):
        """(first, points) on the device: int64 [N + 1] and the points' bytes"""
        if self._d_first is None:
            self._d_first = torch.from_numpy(self.first.copy()).to(self.device)
        if self._d_points is None:
            flat = self.points.view(np.uint8).reshape(-1)
            self._d_points = torch.from_numpy(flat.copy() if flat.size else np.zeros(16, np.uint8)).to(self.device)
        return self._d_first, self._d_points


def _gather_ranges(first, items, idx):
    """(first, items) of the files ``idx`` of per-file ranges ``items[first[i]:first[i + 1]]`` (None, None: none)"""
    if first is None:
        return None, None
    counts = np.diff(first)[idx]
    out = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    at = np.repeat(first[:-1][idx] - out[:-1], counts) + np.arange(int(out[-1]), dtype=np.int64)
    return out, items[at]


def build_jpeg_index(encoded: EncodedImages, find=False):
    """The scan index of every file of ``encoded`` (C ABI ``faa_jpeg_index_build``: one serial decode per file on the
    device, one thread per file): ``(first, points)``, int64 [N + 1] offsets into ``JPEG_SYNC_DTYPE`` points, file i's
    being ``points[first[i]:first[i + 1]]``.  Files with restart markers, scans under 2 KiB and files whose scan does
    not decode cleanly get none, and so do progressive files that take no scan index.  Progressive files that take one
    (``from_bytes(..., progressive_index=True)``) get the points a recording ``decode_jpeg`` places, without the points
    they carry: the index of a progressive file needs its coefficient planes, which only a decode fills.  Waits for the
    device.

    ``find=True`` finds the index in parallel instead (``faa_jpeg_index_find``: one CTA per file, no serial decode).
    Each file's points are then the verified prefix of the chain: always the first points of the serial build's for a
    file that decodes cleanly, and all of them when the chain converged (DESIGN §4.8).  Progressive files get none."""
    _require_cuda(encoded.storage, "encoded")
    prog = encoded.progressive()
    if prog.any():
        parts = [None] * len(encoded)
        groups = [(np.flatnonzero(~prog), lambda e: build_jpeg_index(e, find))]
        if not find:
            groups.append((np.flatnonzero(encoded.progressive_indexed()), _record_progressive_index))
        for at, build in groups:
            if len(at):
                first, points = build(encoded.select(at))
                for k, i in enumerate(at):
                    parts[i] = points[first[k]:first[k + 1]]
        counts = np.array([0 if q is None else len(q) for q in parts], np.int64)
        got = [q for q in parts if q is not None and len(q)]
        return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), \
            (np.concatenate(got) if got else np.zeros(0, _lib.JPEG_SYNC_DTYPE))
    dev = encoded.device
    B = len(encoded)
    if B == 0:
        return np.zeros(1, np.int64), np.zeros(0, _lib.JPEG_SYNC_DTYPE)
    hdr0 = encoded.headers.ctypes.data
    cap_first = jpeg_index_capacities(encoded.headers)
    total = int(cap_first[-1])
    with torch.cuda.device(dev):
        d_first = torch.from_numpy(cap_first).to(dev)
        d_points = torch.empty(max(total, 1) * 16, dtype=torch.uint8, device=dev)
        d_count = torch.empty(B, dtype=torch.int32, device=dev)
        args = (hdr0, encoded.device_headers().data_ptr(), encoded.device_pool().data_ptr(), len(encoded.pool),
                encoded.storage.data_ptr(), B, cap_first.ctypes.data, d_first.data_ptr(), d_points.data_ptr(),
                d_count.data_ptr())
        if find:
            check(lib.faa_jpeg_index_find(*args, _stream_ptr(dev)))
        else:
            d_status = torch.empty(B, dtype=torch.int32, device=dev)
            check(lib.faa_jpeg_index_build(*args, d_status.data_ptr(), _stream_ptr(dev)))
        count = d_count.cpu().numpy()
        pts = d_points.cpu().numpy()[:total * 16].view(_lib.JPEG_SYNC_DTYPE)
    return compact_jpeg_index(cap_first, count, pts)


def _record_progressive_index(encoded: EncodedImages):
    """``build_jpeg_index`` of scan-indexed progressive files: a recording decode without the points they carry"""
    bare = EncodedImages(encoded.storage, encoded.headers, encoded.pool, encoded.device_pool(), scans=encoded.scans,
                         scan_first=encoded.scan_first)
    _, _, count, points, cap_first = decode_jpeg(bare, record=True)
    return compact_jpeg_index(cap_first, count.cpu().numpy(), points.cpu().numpy())


def jpeg_index_capacities(headers):
    """int64 [N + 1] offsets giving each file of ``headers`` (``JPEG_HEADER_DTYPE``) room for the most points it can
    get (``faa_jpeg_index_capacity``): the layout ``faa_jpeg_index_build`` and a recording ``faa_jpeg_decode`` write into"""
    hdr0, size = headers.ctypes.data, headers.itemsize
    caps = np.array([lib.faa_jpeg_index_capacity(hdr0 + i * size) for i in range(len(headers))], np.int64)
    return np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)


def compact_jpeg_index(cap_first, count, points):
    """``(first, points)`` as ``build_jpeg_index`` returns them, from points written into the capacity layout
    ``cap_first`` (``jpeg_index_capacities``) with ``count[i]`` of them for file i (host arrays; ``points`` a
    ``JPEG_SYNC_DTYPE`` array or its bytes)"""
    cap_first = np.asarray(cap_first, np.int64)
    count = np.asarray(count).astype(np.int64)
    points = np.asarray(points)
    if points.dtype != _lib.JPEG_SYNC_DTYPE:
        points = np.ascontiguousarray(points, np.uint8).reshape(-1)[:int(cap_first[-1]) * 16].view(_lib.JPEG_SYNC_DTYPE)
    if len(count) != len(cap_first) - 1 or (count < 0).any() or (count > np.diff(cap_first)).any():
        raise ValueError("count must be [N] and within each file's capacity")
    first = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    at = np.repeat(cap_first[:-1] - first[:-1], count) + np.arange(int(first[-1]), dtype=np.int64)
    return first, points[at].copy()


class _JpegDecoder:
    """C-ABI decoder handle (scratch of the decode calls); one per device"""

    def __init__(self):
        h = C.c_void_p()
        check(lib.faa_jpeg_decoder_create(C.byref(h)))
        self.handle = h

    def __del__(self):
        if getattr(self, "handle", None):
            try:
                lib.faa_jpeg_decoder_destroy(self.handle)
            except Exception:
                pass
            self.handle = None


_DECODERS = {}


def decode_jpeg(encoded: EncodedImages, out: RaggedImages | None = None, record=False, find=False):
    """Decode every file of ``encoded`` on its device (C ABI ``faa_jpeg_decode``, with the files' scan index when they
    carry one: two launches, no host wait), bit-exact
    with ``Image.open(f).convert('RGB')`` (reference imagenet.py:80).  Returns ``(images, status)``: a ``RaggedImages``
    (``out``, by default ``RaggedImages.empty(encoded.sizes)``) and an int32 CUDA tensor of ``faa_jpeg_status`` bits per
    image, 0 where the scan decoded completely; a corrupt image still gets defined pixels.

    ``record=True`` (the call's recording outputs, same pixels and status, still no host wait) also records the scan
    index of every file the decode ran serially as a whole (no points, or points that failed their checks) and returns
    ``(images, status, count, points, cap_first)``: ``count`` int32 [N] and ``points`` (uint8, the bytes of
    ``JPEG_SYNC_DTYPE`` points) CUDA tensors, file i's ``count[i]`` new points at point ``cap_first[i]``
    (``jpeg_index_capacities``, host int64 [N + 1]).  ``count[i] > 0`` means these are file i's points now;
    ``compact_jpeg_index`` turns them into ``build_jpeg_index``'s form.

    ``find=True`` (the call's ``find`` flag: three launches, still no host wait) first finds, in parallel, the scan
    index of every restart-free file that carries none, then decodes every file with its points, so such files decode on
    many threads without a saved index.  Same pixels and status; the return values keep their shapes, with and without
    ``record``.  With ``record``, ``count[i] > 0`` still means "these are file i's points now": the found index when its
    chain converged, or the serial decode's recording when the file's points could not be used.

    Progressive files (``EncodedImages.from_bytes(..., progressive=True)``) are decoded by the same call from the scans
    they carry, one more launch when the batch mixes both kinds.  They get no scan index: count 0 with ``record=True``,
    and points given to them are not used.  Unless they take one (``progressive_index=True``): their restart-free
    scans then decode on many threads from the points they carry, checked as a baseline file's are, and ``record``
    records their points as it records a baseline file's.  Same pixels and status, same launches."""
    _require_cuda(encoded.storage, "encoded")
    dev = encoded.device
    if out is None:
        out = RaggedImages.empty(encoded.sizes, dev)
    elif not isinstance(out, RaggedImages) or not np.array_equal(out.sizes, encoded.sizes) or out.device != dev:
        raise ValueError("out must be a RaggedImages of the files' sizes on their device")
    B = len(encoded)
    status = torch.empty(max(B, 1), dtype=torch.int32, device=dev)[:B]
    if record or find:
        cap_first = jpeg_index_capacities(encoded.headers)
        count = torch.empty(max(B, 1), dtype=torch.int32, device=dev)[:B]
        points = torch.empty(max(int(cap_first[-1]), 1) * 16, dtype=torch.uint8, device=dev)
    if B == 0:
        return (out, status, count, points, cap_first) if record else (out, status)
    h_out, d_out = out.descriptors()
    with torch.cuda.device(dev):
        # the C call's optional groups: scan index in, recording out, scans in
        index, rec, scans = (None,) * 3, (None,) * 4, (None,) * 4
        if encoded.first is not None:
            d_first, d_points = encoded.device_index()
            index = (d_points.data_ptr(), encoded.first.ctypes.data, d_first.data_ptr())
        if record or find:
            d_cap_first = torch.from_numpy(cap_first).to(dev)
            rec = (cap_first.ctypes.data, d_cap_first.data_ptr(), points.data_ptr(), count.data_ptr())
        if encoded.scans is not None:
            d_scans, d_scan_first = encoded.device_scans()
            scans = (encoded.scans.ctypes.data, d_scans.data_ptr(), encoded.scan_first.ctypes.data,
                     d_scan_first.data_ptr())
        check(lib.faa_jpeg_decode(_decoder(dev).handle, encoded.headers.ctypes.data, encoded.device_headers().data_ptr(),
                                  encoded.device_pool().data_ptr(), len(encoded.pool), encoded.storage.data_ptr(), B,
                                  h_out.ctypes.data, d_out.data_ptr(), status.data_ptr(), *index, *rec, *scans,
                                  int(find), _stream_ptr(dev)))
    return (out, status, count, points, cap_first) if record else (out, status)


def _decoder(dev):
    dec = _DECODERS.get(dev.index)
    if dec is None:
        dec = _DECODERS[dev.index] = _JpegDecoder()
    return dec


def gather(jobs, d_jobs, device):
    """One launch of the byte copies ``jobs`` (host ``COPY_DTYPE`` [n]: addresses in this process, local or IPC
    mappings) on ``device``'s current stream (C ABI ``faa_gather``).  ``d_jobs``: the same table's bytes on the device,
    uploaded by the caller.  Raises ValueError before any device work for an empty table or a null address."""
    jobs = np.ascontiguousarray(jobs, dtype=_lib.COPY_DTYPE).reshape(-1)
    dev = torch.device(device)
    with torch.cuda.device(dev):
        check(lib.faa_gather(jobs.ctypes.data, d_jobs.data_ptr(), len(jobs), _stream_ptr(dev)))


def _augment_ragged(policy, batch: RaggedImages, tail, samples, boxes, rng, out):
    """augment_batch on a RaggedImages batch (C ABI ``faa_augment_ragged``); policies of more than two ops run window
    by window through uint8 intermediates, as ``_augment_launch`` does"""
    raw = TailSpec.raw_u8()
    if (tail.out_size, tail.crop_pad, tail.hflip, tail.cutout, tail.out_dtype) != \
            (raw.out_size, raw.crop_pad, raw.hflip, raw.cutout, raw.out_dtype):
        raise ValueError("a ragged batch is augmented at each image's own size into uint8: the tail must be TailSpec.raw_u8()")
    if (samples is None) == (rng is None):
        raise ValueError("give either samples (and boxes) or rng")
    _require_cuda(batch.storage, "batch")
    dev = batch.device
    if out is None:
        out = RaggedImages.empty(batch.sizes, dev)
    elif not isinstance(out, RaggedImages) or not np.array_equal(out.sizes, batch.sizes) or out.device != dev:
        raise ValueError("out must be a RaggedImages of the batch's sizes on its device")
    if len(batch) == 0:
        return out

    def to_dev(a):
        if a is None or isinstance(a, torch.Tensor):
            if a is not None:
                _require_cuda(a, "records")
            return a
        return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)

    d_s, d_b = to_dev(samples), to_dev(boxes)
    rng_p = C.byref(rng) if rng is not None else None
    B = len(batch)
    with torch.cuda.device(dev):
        stream = _stream_ptr(dev)
        cur = batch
        for base in range(0, policy.n_op, _lib.MAX_FUSED_OPS):
            nxt = out if base + _lib.MAX_FUSED_OPS >= policy.n_op else RaggedImages.empty(batch.sizes, dev)
            (h_in, d_in), (h_out, d_out) = cur.descriptors(), nxt.descriptors()
            check(lib.faa_augment_ragged(policy.handle, h_in.ctypes.data, d_in.data_ptr(), B, h_out.ctypes.data,
                                         d_out.data_ptr(), d_s.data_ptr() if d_s is not None else None,
                                         d_b.data_ptr() if d_b is not None else None, rng_p, base, stream))
            cur = nxt
    return out


def crop_resize(batch_u8, size, boxes=None, rng=None, tail: TailSpec | None = None, out=None):
    """EfficientNet crop + ``Resize((s, s), BICUBIC)`` of a uint8 [B,H,W,3] CUDA batch in ONE launch (C ABI
    ``faa_crop_resize``), bit-exact with Pillow's ``crop`` + ``resize``.  A ``RaggedImages`` batch runs the same in one
    launch too (``faa_crop_resize_ragged``), each image cropped at its own size.

    ``size``: output size (int or (h, w)).  ``boxes``: per-image crop boxes ([B] ``CROP_BOX_DTYPE`` array, or an
    int32 [B, 4] array / tensor of x0, y0, w, h); otherwise ``rng`` is a ``crop_cfg`` and the kernel draws (random
    mode) or computes (center mode) the boxes.  ``tail``: None or a uint8 ``TailSpec`` -> uint8 [B, s, s, 3]; a float
    ``TailSpec`` -> ToTensor + Normalize fused in, [B, 3, s, s] of ``tail.out_dtype`` (its crop / flip / Cutout fields
    are not used here)."""
    ragged = isinstance(batch_u8, RaggedImages)
    _require_cuda(batch_u8.storage if ragged else batch_u8, "batch")
    if not ragged:
        if batch_u8.dtype != torch.uint8 or batch_u8.dim() != 4 or batch_u8.shape[-1] != 3:
            raise ValueError("batch must be uint8 [B, H, W, 3]")
    if (boxes is None) == (rng is None):
        raise ValueError("give exactly one of boxes= and rng=")
    if ragged:
        dev, B, H, W = batch_u8.device, len(batch_u8), 1, 1
    else:
        batch_u8 = batch_u8.contiguous()
        dev = batch_u8.device
        B, H, W, _ = batch_u8.shape
    oh, ow = (size, size) if isinstance(size, int) else (int(size[0]), int(size[1]))
    tail = tail or TailSpec.raw_u8()
    t = tail.c_struct(H, W)
    t.out_h, t.out_w = oh, ow
    shape = (B, oh, ow, 3) if tail.out_dtype == torch.uint8 else (B, 3, oh, ow)
    if out is None:
        out = torch.empty(shape, dtype=tail.out_dtype, device=dev)
    elif tuple(out.shape) != shape or out.dtype != tail.out_dtype or not out.is_contiguous() or out.device != dev:
        raise ValueError("out must be a contiguous %s tensor %s on %s" % (tail.out_dtype, shape, dev))
    d_boxes = None
    if boxes is not None:
        if isinstance(boxes, torch.Tensor):
            d_boxes = boxes.to(device=dev, dtype=torch.int32).contiguous().reshape(-1)
        else:
            a = np.ascontiguousarray(boxes)
            a = a.view(np.int32) if a.dtype == _lib.CROP_BOX_DTYPE else a.astype(np.int32)
            d_boxes = torch.from_numpy(np.ascontiguousarray(a).reshape(-1).copy()).to(dev)
        if d_boxes.numel() != 4 * B:
            raise ValueError("need one box (x0, y0, w, h) per image")
    cfg = rng if rng is not None else crop_cfg(oh)
    with torch.cuda.device(dev):
        if ragged:
            h_desc, d_desc = batch_u8.descriptors()
            check(lib.faa_crop_resize_ragged(h_desc.ctypes.data, d_desc.data_ptr(), B, out.data_ptr(), C.byref(t),
                                             d_boxes.data_ptr() if d_boxes is not None else None, C.byref(cfg),
                                             _stream_ptr(dev)))
        else:
            check(lib.faa_crop_resize(batch_u8.data_ptr(), out.data_ptr(), B, H, W, C.byref(t),
                                      d_boxes.data_ptr() if d_boxes is not None else None, C.byref(cfg), _stream_ptr(dev)))
    return out


def sample_philox_at(policy: CompiledPolicy, positions, h, w, tail: TailSpec, rng, device):
    """Decisions of the global samples ``rng.first_index + positions[k]`` for h x w images, drawn on the device (C ABI
    ``faa_sample_philox_at``): (samples, boxes) as CUDA uint8 tensors for ``augment_batch``."""
    pos = torch.as_tensor(np.asarray(positions, dtype=np.int32), device=device)
    n = int(pos.numel())
    d_s = torch.empty(n * 16, dtype=torch.uint8, device=device)
    d_b = torch.empty(max(1, n * policy.n_op * 8), dtype=torch.uint8, device=device)
    t = tail.c_struct(h, w)
    with torch.cuda.device(device):
        check(lib.faa_sample_philox_at(policy.handle, n, int(h), int(w), C.byref(t), C.byref(rng), pos.data_ptr(),
                                       d_s.data_ptr(), d_b.data_ptr(), _stream_ptr(device)))
    return d_s, d_b


def cached_tables(policy: CompiledPolicy):
    """(number, bytes) of the per-size device tables of compiled ops the handle holds (C ABI ``faa_policy_cached_tables``)"""
    n, b = C.c_int(), C.c_uint64()
    check(lib.faa_policy_cached_tables(policy.handle, C.byref(n), C.byref(b)))
    return int(n.value), int(b.value)
