"""Reference ``FastAutoAugment/data.py`` surface on the CUDA path.

* ``Augmentation(policies)``   - same constructor and ``__call__(PIL) -> PIL`` as the reference
  (``data.py:253-264``), plus the batched entry ``augment_batch`` the training loop should use.
* ``CutoutDefault(length)``    - same callable as the reference (``data.py:228-250``).
* ``GpuAugmentedLoader``       - what ``get_dataloaders`` (``data.py:37-225``) hands to
  ``train.py:47`` / ``search.py:101``: an iterable of ``(data, label)`` whose ``data`` is already
  the augmented, normalised CUDA tensor, so the caller's ``.cuda()`` (``train.py:49``) is a
  no-op.  The raw uint8 dataset lives on the device; no CUDA is touched in worker processes
  because there are none.  The one exception is the ImageNet directory (``JpegFileDataset``): its files stay on disk
  and are read, staged and decoded batch by batch, one batch ahead (``FileBatchStream``), unless they are held in
  device memory (``ResidentJpegDataset``) and gathered per batch on the device.
"""
from __future__ import annotations

import contextlib
import ctypes
import io
import math
import os
import random
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import PIL.Image
import torch
import torch.distributed as dist
from torch.utils.data import Sampler, SubsetRandomSampler
from torch.utils.data.distributed import DistributedSampler

from . import _lib, archive
from .conf import Config as C
from .distributed import _RawCuda, agree, check_fit, fit_error, gather_bytes, host_ranks, share_jpeg_index
from .engine import (CIFAR_MEAN, CIFAR_STD, IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, EncodedImages, RaggedImages,
                     TailSpec, augment_batch, augment_tta, augment_tta_policies, build_jpeg_index, center_crop_box,
                     check_tta, check_tta_policies, compact_jpeg_index, compile_policies, crop_cfg, crop_resize,
                     decode_jpeg, gather, jpeg_index_capacities, make_rng, parse_jpeg_headers, sample_philox_at,
                     tta_positions, tta_select)
from .engine import _gather_ranges as engine_gather_ranges


class Augmentation(object):
    """Drop-in for reference ``Augmentation`` (data.py:253-264)."""

    def __init__(self, policies):
        self.policies = policies
        self._compiled = None

    @property
    def compiled(self) -> CompiledPolicy:
        if self._compiled is None:
            self._compiled = CompiledPolicy(self.policies)
        return self._compiled

    def __call__(self, img):
        """PIL RGB image in, new PIL image out; consumes ``random`` / ``numpy.random`` exactly
        like the reference, so identical seeds give identical pixels."""
        if not torch.cuda.is_available():
            raise _lib.FaaRuntimeError("fast_autoaugment_b200 needs a CUDA device (no CPU fallback)")
        arr = np.ascontiguousarray(np.asarray(img.convert("RGB")))
        h, w = arr.shape[:2]
        samples, boxes = self.compiled.sample_parity(1, h, w, TailSpec.raw_u8())
        y = augment_batch(self.compiled, torch.from_numpy(arr[None].copy()).cuda(), TailSpec.raw_u8(), samples, boxes)
        return PIL.Image.fromarray(y[0].cpu().numpy())

    def augment_batch(self, batch_u8, tail: TailSpec | None = None, seed=None, first_index=0, parity=False,
                      out=None):
        """uint8 [B,H,W,3] CUDA tensor -> augmented batch.  ``parity=True`` replays the global
        generators like the reference's per-sample loop; otherwise the kernel draws with Philox
        keyed by (``seed``, ``first_index`` + i).  A ``RaggedImages`` batch is augmented image by image at its own
        size (uint8, ``tail`` raw) into a ``RaggedImages``; with ``parity`` each image's draws are made at its size,
        in batch order, as calling this object on the images one after another would."""
        tail = tail or TailSpec.raw_u8()
        if isinstance(batch_u8, RaggedImages):
            if parity:
                recs = [self.compiled.sample_parity(1, int(h), int(w), tail) for h, w in batch_u8.sizes]
                samples = np.concatenate([s for s, _ in recs]) if recs else np.zeros(0, _lib.SAMPLE_DTYPE)
                boxes = np.concatenate([b for _, b in recs]) if recs else np.zeros((0, self.compiled.n_op), _lib.BOX_DTYPE)
                return augment_batch(self.compiled, batch_u8, tail, samples, boxes, out=out)
            if seed is None:
                seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            return augment_batch(self.compiled, batch_u8, tail, rng=make_rng(seed, first_index, tail), out=out)
        b, h, w, _ = batch_u8.shape
        if parity:
            samples, boxes = self.compiled.sample_parity(b, h, w, tail)
            return augment_batch(self.compiled, batch_u8, tail, samples, boxes, out=out)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        return augment_batch(self.compiled, batch_u8, tail, rng=make_rng(seed, first_index, tail), out=out)


class CutoutDefault(object):
    """Drop-in for reference ``CutoutDefault`` (data.py:228-250): zero box on a CHW tensor, in
    place, centre drawn from ``numpy.random`` (y first).  In the batched path the same box is
    applied inside the fused kernel (``TailSpec.cutout``)."""

    def __init__(self, length):
        self.length = length

    def __call__(self, img):
        h, w = img.size(1), img.size(2)
        y = np.random.randint(h)
        x = np.random.randint(w)
        half = self.length // 2
        y1, y2 = int(np.clip(y - half, 0, h)), int(np.clip(y + half, 0, h))
        x1, x2 = int(np.clip(x - half, 0, w)), int(np.clip(x + half, 0, w))
        img[:, y1:y2, x1:x2] = 0.0
        return img


_IMAGENET_PCA = {                                            # reference data.py:25-32
    "eigval": [0.2175, 0.0188, 0.0045],
    "eigvec": [[-0.5675, 0.7192, 0.4009], [-0.5808, -0.0045, -0.8140], [-0.5836, -0.6948, 0.4203]],
}


class Lighting(object):
    """Drop-in for reference ``Lighting`` (augmentations.py:197-215): AlexNet-style PCA noise on a CHW float tensor,
    between ToTensor and Normalize in the ImageNet chain (data.py:70-72).  In the batched path the per-image offsets
    ``sample_rgb(n)`` go to ``augment_batch(..., lighting_rgb=...)``, which folds them into per-image normalisation tables."""

    def __init__(self, alphastd, eigval=_IMAGENET_PCA["eigval"], eigvec=_IMAGENET_PCA["eigvec"]):
        self.alphastd = alphastd
        self.eigval = torch.Tensor(eigval)
        self.eigvec = torch.Tensor(eigvec)

    def _rgb(self, like):
        alpha = like.new().resize_(3).normal_(0, self.alphastd)
        return self.eigvec.type_as(like).clone().mul(alpha.view(1, 3).expand(3, 3)) \
            .mul(self.eigval.view(1, 3).expand(3, 3)).sum(1).squeeze()

    def __call__(self, img):
        if self.alphastd == 0:
            return img
        rgb = self._rgb(img)
        return img.add(rgb.view(3, 1, 1).expand_as(img))

    def sample_rgb(self, n):
        """[n, 3] fp32 offsets, drawn from torch's CPU generator exactly like n per-image calls of the reference."""
        if self.alphastd == 0:
            return torch.zeros(n, 3)
        like = torch.empty(0)
        return torch.stack([self._rgb(like) for _ in range(n)])


class ColorJitter(object):
    """torchvision ``ColorJitter(brightness, contrast, saturation)`` of the ImageNet train chain (reference data.py:65-69)
    for uint8 NHWC CUDA batches: per image a random order (``torch.randperm(4)``) of Brightness / Contrast / Color
    ``ImageEnhance`` blends with factors uniform in ``[max(0, 1 - x), 1 + x]`` - the arithmetic of the policy ops of the
    same names (C ABI ``faa_color_jitter``)."""

    def __init__(self, brightness=0.4, contrast=0.4, saturation=0.4):
        self.ranges = [(max(0.0, 1.0 - v), 1.0 + v) if v else None for v in (brightness, contrast, saturation)]

    def sample_parity(self, n):
        """records of n images from torch's CPU generator in torchvision's order (get_params: randperm(4), then b, c, s)"""
        recs = np.zeros(n, dtype=_lib.JITTER_DTYPE)
        for i in range(n):
            order = torch.randperm(4).tolist()
            f = [None if r is None else float(torch.empty(1).uniform_(r[0], r[1])) for r in self.ranges]
            recs[i]["order"] = [o if (o < 3 and f[o] is not None) else 3 for o in order]
            recs[i]["alpha"] = [np.float32(x if x is not None else 1.0) for x in f]
        return recs

    def jitter_batch(self, batch_u8, recs=None, out=None):
        """uint8 [B,H,W,3] CUDA -> uint8 [B,H,W,3] (``out`` may be the input itself)."""
        if not (isinstance(batch_u8, torch.Tensor) and batch_u8.is_cuda and batch_u8.dtype == torch.uint8 and batch_u8.is_contiguous()):
            raise ValueError("batch must be a contiguous uint8 CUDA tensor [B, H, W, 3]")
        b, h, w, _ = batch_u8.shape
        if recs is None:
            recs = self.sample_parity(b)
        d_recs = torch.from_numpy(np.ascontiguousarray(recs).view(np.uint8).reshape(-1).copy()).to(batch_u8.device)
        if out is None:
            out = torch.empty_like(batch_u8)
        with torch.cuda.device(batch_u8.device):
            import ctypes as C
            _lib.check(_lib.lib.faa_color_jitter(batch_u8.data_ptr(), out.data_ptr(), b, h, w, d_recs.data_ptr(),
                                                 C.c_void_p(torch.cuda.current_stream(batch_u8.device).cuda_stream)))
        return out


class EfficientNetCenterCrop(object):
    """Drop-in for reference ``EfficientNetCenterCrop`` (data.py:323-345): the square of side
    ``imgsize / (imgsize + 32) * short side`` in the middle of the image.  Batched: ``cfg()`` for ``crop_resize``."""

    def __init__(self, imgsize):
        self.imgsize = imgsize

    def box(self, h, w):
        """(x0, y0, w, h) after Image.crop's rounding of the box"""
        return center_crop_box(h, w, self.imgsize)

    def __call__(self, img):
        x0, y0, w, h = self.box(img.size[1], img.size[0])
        return img.crop((x0, y0, x0 + w, y0 + h))

    def sample_parity(self, n, h, w):
        """[n] boxes (``_lib.CROP_BOX_DTYPE``); draws nothing"""
        b = np.zeros(n, dtype=_lib.CROP_BOX_DTYPE)
        b["x0"], b["y0"], b["w"], b["h"] = self.box(h, w)
        return b

    def cfg(self, seed=0, first_index=0):
        return crop_cfg(self.imgsize, center=True, seed=seed, first_index=first_index)


class EfficientNetRandomCrop(object):
    """Drop-in for reference ``EfficientNetRandomCrop`` (data.py:267-320): up to ``max_attempts`` draws of an aspect
    ratio and a height from Python's ``random``, then ``random.randint`` for x and y; the whole image or ten failed
    attempts fall back to the center crop.  ``__call__`` and ``sample_parity`` consume ``random`` exactly like the
    reference; ``cfg(seed, first_index)`` lets the kernel draw the boxes instead (Philox: same distributions, not the
    reference's stream)."""

    def __init__(self, imgsize, min_covered=0.1, aspect_ratio_range=(3. / 4, 4. / 3), area_range=(0.08, 1.0),
                 max_attempts=10):
        assert 0.0 < min_covered
        assert 0 < aspect_ratio_range[0] <= aspect_ratio_range[1]
        assert 0 < area_range[0] <= area_range[1]
        assert 1 <= max_attempts
        self.imgsize = imgsize
        self.min_covered = min_covered
        self.aspect_ratio_range = aspect_ratio_range
        self.area_range = area_range
        self.max_attempts = max_attempts
        self._fallback = EfficientNetCenterCrop(imgsize)

    def box(self, h, w):
        """one draw: (x0, y0, w, h) of the crop of an h x w image"""
        W, H = w, h
        min_area = self.area_range[0] * (W * H)
        max_area = self.area_range[1] * (W * H)
        for _ in range(self.max_attempts):
            aspect_ratio = random.uniform(*self.aspect_ratio_range)
            height = int(round(math.sqrt(min_area / aspect_ratio)))
            max_height = int(round(math.sqrt(max_area / aspect_ratio)))
            if max_height * aspect_ratio > W:
                max_height = int((W + 0.5 - 1e-7) / aspect_ratio)
                if max_height * aspect_ratio > W:
                    max_height -= 1
            if max_height > H:
                max_height = H
            if height >= max_height:
                height = max_height
            height = int(round(random.uniform(height, max_height)))
            width = int(round(height * aspect_ratio))
            area = width * height
            if area < min_area or area > max_area:
                continue
            if width > W or height > H:
                continue
            if area < self.min_covered * (W * H):
                continue
            if width == W and height == H:
                return self._fallback.box(h, w)
            x = random.randint(0, W - width)
            y = random.randint(0, H - height)
            return x, y, width, height
        return self._fallback.box(h, w)

    def __call__(self, img):
        x0, y0, w, h = self.box(img.size[1], img.size[0])
        return img.crop((x0, y0, x0 + w, y0 + h))

    def sample_parity(self, n, h, w):
        """[n] boxes (``_lib.CROP_BOX_DTYPE``) drawn one image after another from ``random``"""
        b = np.zeros(n, dtype=_lib.CROP_BOX_DTYPE)
        for i in range(n):
            b[i] = self.box(h, w)
        return b

    def cfg(self, seed=0, first_index=0):
        return crop_cfg(self.imgsize, False, self.min_covered, self.aspect_ratio_range, self.area_range,
                        self.max_attempts, seed, first_index)


# EfficientNet input resolutions, reference networks/efficientnet_pytorch/utils.py:174-181 (the `res` coefficient)
EFFICIENTNET_SIZES = {"efficientnet-b0": 224, "efficientnet-b1": 240, "efficientnet-b2": 260, "efficientnet-b3": 300,
                      "efficientnet-b4": 380, "efficientnet-b5": 456, "efficientnet-b6": 528, "efficientnet-b7": 600}


def imagenet_input_size(model_type):
    """data.py:50-55: 224, or the EfficientNet resolution when the model is an EfficientNet"""
    model_type = str(model_type or "")
    if "efficientnet" in model_type:
        return EFFICIENTNET_SIZES[model_type]
    return 224


class ImageNetChain(object):
    """The reference's ImageNet transforms (data.py:60-80) on uint8 [B,H,W,3] CUDA batches of full-size images.

    ``train``: ``Augmentation(policy)`` at source size (uint8) -> ``EfficientNetRandomCrop`` + ``Resize(BICUBIC)``
    (``faa_crop_resize``, uint8) -> ``ColorJitter(0.4, 0.4, 0.4)`` in place -> one launch of the identity policy with
    ``RandomHorizontalFlip`` + ``ToTensor`` + ``Lighting(0.1)`` + ``Normalize``.  The flip runs after the jitter here:
    the jitter is per-pixel with a whole-image mean, so the order does not change a value.
    ``test``: ``EfficientNetCenterCrop`` + ``Resize`` + ``ToTensor`` + ``Normalize`` in one launch.

    ``parity=True`` draws like the reference's per-image loop (a ``num_workers=0`` DataLoader), image after image:
    policy (``random``, ``numpy``), crop (``random``), flip (``torch.rand``), jitter (``randperm(4)`` + three
    uniforms), Lighting (three normals).  Otherwise the policy, crop and flip are drawn by the kernels (Philox keyed by
    (seed, first_index + i)) and the jitter / Lighting records by vectorised torch calls on the device.

    Both also take a ``RaggedImages`` batch of differently sized sources (the reference transforms one PIL image at a
    time, so every image is cropped at its own size).  ``test`` is then one ragged crop-resize launch.  ``train`` runs
    the policy once per distinct source size (the images of that size gathered, each with the decisions of its batch
    position: ``faa_sample_philox_at``, or its parity records) into a packed uint8 intermediate, then one ragged
    crop-resize, and the same jitter and flip + Lighting + Normalize launches as a uniform batch.  A batch of one size
    gives the bytes of the uniform chain.  The policy handle keeps one compiled table per source size it has seen.

    An ``EncodedImages`` batch (JPEG files) is decoded on the device first (``decode_jpeg``, bit-exact with the reference's
    Pillow loader) and then runs the ragged path; the decode status of its images is left in ``last_status``."""

    _EIGVAL = _IMAGENET_PCA["eigval"]
    _EIGVEC = _IMAGENET_PCA["eigvec"]

    def __init__(self, policies, input_size=224, out_dtype=torch.float32):
        self.input_size = int(input_size)
        self.crop = EfficientNetRandomCrop(self.input_size)
        self.center = EfficientNetCenterCrop(self.input_size)
        self.jitter = ColorJitter(0.4, 0.4, 0.4)
        self.lighting = Lighting(0.1)
        self.aug = Augmentation(policies) if policies is not None else None
        self.flip_policy = CompiledPolicy([[("Invert", -1.0, 0.0)]])       # a slot that never fires and draws nothing
        self.tail = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, 0, out_dtype)
        self.test_tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, out_dtype)
        self.last_status = None

    def _decoded(self, batch):
        if isinstance(batch, EncodedImages):
            batch, self.last_status = decode_jpeg(batch)
        return batch

    def sample_parity(self, n, h=None, w=None, sizes=None):
        """per-image records in the reference's draw order: (policy samples, policy boxes or None, crop boxes,
        flip samples of the identity policy, jitter records, Lighting offsets [n, 3]).  ``sizes``: [n] (h, w) of each
        image (a ragged batch) instead of one h x w for all."""
        pol = self.aug.compiled if self.aug is not None else None
        sizes = [(h, w)] * n if sizes is None else [(int(a), int(b)) for a, b in np.asarray(sizes).reshape(-1, 2)]
        if len(sizes) != n:
            raise ValueError("need one size per image")
        samples, boxes = [], []
        crops = np.zeros(n, dtype=_lib.CROP_BOX_DTYPE)
        flips = np.zeros(n, dtype=_lib.SAMPLE_DTYPE)
        jit = np.zeros(n, dtype=_lib.JITTER_DTYPE)
        rgb = torch.zeros(n, 3)
        for i in range(n):
            h, w = sizes[i]
            if pol is not None:
                s, b = pol.sample_parity(1, h, w, TailSpec.raw_u8())
                samples.append(s)
                boxes.append(b)
            crops[i] = self.crop.box(h, w)
            flips[i]["flip"] = 1 if bool(torch.rand(1) < 0.5) else 0
            jit[i] = self.jitter.sample_parity(1)[0]
            if self.lighting.alphastd != 0:
                rgb[i] = self.lighting._rgb(torch.empty(0))
        if pol is None:
            return None, None, crops, flips, jit, rgb
        return np.concatenate(samples), np.concatenate(boxes), crops, flips, jit, rgb

    def _device_records(self, n, dev, seed, first_index):
        g = torch.Generator(device=dev)
        g.manual_seed((int(seed) * 1000003 + int(first_index)) & 0x7FFFFFFFFFFFFFFF)
        order = torch.argsort(torch.rand(n, 4, device=dev, generator=g), dim=1).to(torch.int32)   # randperm(4) per image
        alpha = torch.empty(n, 3, device=dev)
        for j, r in enumerate(self.jitter.ranges):
            if r is None:
                alpha[:, j] = 1.0
            else:
                alpha[:, j].uniform_(r[0], r[1], generator=g)
        present = torch.tensor([r is not None for r in self.jitter.ranges] + [False], device=dev)
        order = torch.where(present[order.long()], order, torch.full_like(order, 3))
        packed = order[:, 0] | (order[:, 1] << 8) | (order[:, 2] << 16) | (order[:, 3] << 24)
        recs = torch.cat([alpha.view(torch.int32), packed[:, None]], dim=1).contiguous()
        a = torch.randn(n, 3, device=dev, generator=g) * float(self.lighting.alphastd)
        eigvec = torch.tensor(self._EIGVEC, device=dev)
        eigval = torch.tensor(self._EIGVAL, device=dev)
        rgb = (eigvec[None] * a[:, None, :] * eigval[None, None, :]).sum(2)
        return recs, rgb

    def train(self, batch_u8, parity=False, seed=0, first_index=0, records=None):
        """uint8 [B,H,W,3] CUDA (or ``RaggedImages``) -> [B, 3, s, s] ``out_dtype``.  ``records``: the tuple of
        ``sample_parity`` (drawn here when ``parity`` and not given)."""
        batch_u8 = self._decoded(batch_u8)
        if isinstance(batch_u8, RaggedImages):
            return self._train_ragged(batch_u8, parity, seed, first_index, records)
        b, h, w, _ = batch_u8.shape
        dev = batch_u8.device
        if parity and records is None:
            records = self.sample_parity(b, h, w)
        if records is not None:
            samples, boxes, crops, flips, jit, rgb = records
            x = batch_u8 if self.aug is None else augment_batch(self.aug.compiled, batch_u8, TailSpec.raw_u8(), samples, boxes)
            y = crop_resize(x, self.input_size, boxes=crops)
            self.jitter.jitter_batch(y, jit, out=y)
            zb = np.zeros((b, 1), dtype=_lib.BOX_DTYPE)
            return augment_batch(self.flip_policy, y, self.tail, flips, zb, lighting_rgb=rgb)
        raw = TailSpec.raw_u8()
        x = batch_u8 if self.aug is None else augment_batch(self.aug.compiled, batch_u8, raw,
                                                            rng=make_rng(seed, first_index, raw))
        y = crop_resize(x, self.input_size, rng=self.crop.cfg(seed, first_index))
        recs, rgb = self._device_records(b, dev, seed, first_index)
        with torch.cuda.device(dev):
            import ctypes as C
            _lib.check(_lib.lib.faa_color_jitter(y.data_ptr(), y.data_ptr(), b, self.input_size, self.input_size,
                                                 recs.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return augment_batch(self.flip_policy, y, self.tail, rng=make_rng(seed, first_index, self.tail), lighting_rgb=rgb)

    def _policy_ragged(self, batch, records, seed, first_index):
        """the policy at source size, one launch group per distinct size -> RaggedImages of the results (batch order).
        Each group's images are one contiguous [n, h, w, 3] starting on a 16-byte boundary: the policy kernels' word
        loads and stores need the alignment of a fresh allocation."""
        pol = self.aug.compiled
        raw = TailSpec.raw_u8()
        groups = batch.groups()
        slab = [(-(-len(pos) * h * w * 3 // 16)) * 16 for (h, w), pos in groups]
        inter = torch.empty(int(sum(slab)), dtype=torch.uint8, device=batch.device)
        offsets = np.zeros(len(batch), np.int64)
        at = 0
        for ((h, w), pos), size in zip(groups, slab):
            n = len(pos)
            src_off = batch.offsets[pos]
            if (int(src_off[0]) + batch.storage.data_ptr()) % 16 == 0 and \
                    np.array_equal(src_off, src_off[0] + np.arange(n) * h * w * 3):      # already packed in batch order
                x = batch.storage[int(src_off[0]):int(src_off[0]) + n * h * w * 3].view(n, h, w, 3)
            else:
                x = torch.stack([batch.image(int(i)) for i in pos])
            out = inter[at:at + n * h * w * 3].view(n, h, w, 3)
            if records is not None:
                samples, boxes = records[0][pos], records[1][pos]
            else:
                samples, boxes = sample_philox_at(pol, pos, h, w, raw, make_rng(seed, first_index, raw), batch.device)
            augment_batch(pol, x, raw, samples, boxes, out=out)
            offsets[pos] = at + np.arange(n) * h * w * 3
            at += size
        return RaggedImages(inter, offsets, batch.sizes)

    def _train_ragged(self, batch, parity, seed, first_index, records):
        b = len(batch)
        dev = batch.device
        if parity and records is None:
            records = self.sample_parity(b, sizes=batch.sizes)
        x = batch if self.aug is None else self._policy_ragged(batch, records, seed, first_index)
        s = self.input_size
        if records is not None:
            _, _, crops, flips, jit, rgb = records
            y = crop_resize(x, s, boxes=crops)
            self.jitter.jitter_batch(y, jit, out=y)
            zb = np.zeros((b, 1), dtype=_lib.BOX_DTYPE)
            return augment_batch(self.flip_policy, y, self.tail, flips, zb, lighting_rgb=rgb)
        y = crop_resize(x, s, rng=self.crop.cfg(seed, first_index))
        recs, rgb = self._device_records(b, dev, seed, first_index)
        with torch.cuda.device(dev):
            import ctypes as C
            _lib.check(_lib.lib.faa_color_jitter(y.data_ptr(), y.data_ptr(), b, s, s, recs.data_ptr(),
                                                 C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return augment_batch(self.flip_policy, y, self.tail, rng=make_rng(seed, first_index, self.tail), lighting_rgb=rgb)

    def _device_records_tta(self, n, dev, seed, first_index, replicas):
        """the jitter records and Lighting offsets of ``replicas`` replicas of an n-image batch, replica-major: replica r's
        are ``_device_records(n, dev, seed, first_index + r * n)``, those of ``train(first_index=first_index + r * n)``"""
        parts = [self._device_records(n, dev, seed, int(first_index) + r * n) for r in range(int(replicas))]
        return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])

    def check_tta(self, n, replicas, parity=False):
        """ValueError for a ``train_tta`` call this chain refuses: parity draws (K reference loaders have no single draw
        order), replicas < 1, more than 65535 images per launch, a policy longer than one fused window"""
        if parity:
            raise ValueError("train_tta draws with Philox only: K reference loaders have no single parity draw order")
        check_tta(n, replicas)
        if self.aug is not None and self.aug.compiled.n_op > _lib.MAX_FUSED_OPS:
            raise ValueError("train_tta supports policies of at most %d ops per sub-policy (replicated launches)"
                             % _lib.MAX_FUSED_OPS)

    def train_tta(self, batch, replicas, seed=0, first_index=0, parity=False):
        """The train chain's test-time-augmentation replicas of one batch: uint8 [B,H,W,3] CUDA, ``RaggedImages`` or
        ``EncodedImages`` (decoded once; ``last_status`` set once) -> [replicas, B, 3, s, s] ``out_dtype`` with

            out[r] == train(batch, seed=seed, first_index=first_index + r * B)      (bit for bit)

        Each stage is one launch (group) over all replicas * B images, schedule entry v = r * B + i drawing the Philox
        keys of global sample first_index + v: the policy (``augment_tta``: one replicated launch for a uniform batch,
        one ``faa_augment_ragged`` group over replicated descriptors for a ragged one), crop + resize, ColorJitter and
        HFlip + Lighting + Normalize.  Without a policy the crop reads the sources through replicated descriptors.
        Raises ValueError before any device work for what ``check_tta`` refuses."""
        B = len(batch) if isinstance(batch, (RaggedImages, EncodedImages)) else int(batch.shape[0])
        self.check_tta(B, replicas, parity)
        K = int(replicas)
        x = self._decoded(batch)
        y = None
        if self.aug is not None:
            y = augment_tta(self.aug.compiled, x, TailSpec.raw_u8(), K, seed, first_index)
            if not isinstance(y, RaggedImages):
                y = y.view(K * B, *y.shape[2:])
        out = self._tta_stages(x, y, B, K, seed, first_index)
        return out.view(K, B, *out.shape[1:])

    def _tta_stages(self, x, y, B, n, seed, first_index):
        """crop + resize, ColorJitter and HFlip + Lighting + Normalize, one launch each over the n * B entries of a TTA
        call: the policy's outputs ``y`` (n * B images in entry order), or, without a policy (``y`` None), the B
        sources ``x`` read n times through replicated descriptors -> [n * B, 3, s, s]"""
        dev = x.device
        if y is None and isinstance(x, RaggedImages):
            y = tta_select(x, n)
        elif y is None:                                     # the sources themselves, n descriptors each
            x = x.contiguous()
            h, w = int(x.shape[1]), int(x.shape[2])
            y = RaggedImages(x.view(-1), tta_positions(B, n) * (h * w * 3), [(h, w)] * (n * B))
        s = self.input_size
        z = crop_resize(y, s, rng=self.crop.cfg(seed, first_index))
        recs, rgb = self._device_records_tta(B, dev, seed, first_index, n)
        with torch.cuda.device(dev):
            import ctypes as C
            _lib.check(_lib.lib.faa_color_jitter(z.data_ptr(), z.data_ptr(), n * B, s, s, recs.data_ptr(),
                                                 C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return augment_batch(self.flip_policy, z, self.tail, rng=make_rng(seed, first_index, self.tail), lighting_rgb=rgb)

    def check_tta_policies(self, n, policies, replicas, parity=False):
        """ValueError for a ``train_tta_policies`` call this chain refuses (``policies``: ``CompiledPolicy`` handles):
        parity draws and what ``check_tta_policies`` refuses"""
        if parity:
            raise ValueError("train_tta draws with Philox only: K reference loaders have no single parity draw order")
        check_tta_policies(policies, n, replicas)

    def train_tta_policies(self, batch, policies, replicas, seed=0, first_index=0, parity=False):
        """``train_tta`` for T candidate policies in place of the chain's own (the policy search scoring several
        suggestions against one fold): uint8 [B,H,W,3] CUDA, ``RaggedImages`` or ``EncodedImages`` (decoded once) ->
        [T, replicas, B, 3, s, s] ``out_dtype`` with

            out[t] == ImageNetChain(policies[t]).train_tta(batch, replicas, seed, first_index + t * replicas * B)

        Each stage is one launch (group) over all T * replicas * B entries, entry v = (t * replicas + r) * B + i drawing
        the Philox keys of global sample first_index + v: the policy (``augment_tta_policies``), crop + resize,
        ColorJitter and HFlip + Lighting + Normalize.  ``policies``: what ``compile_policies`` takes.  Raises ValueError
        before any device work for what ``check_tta_policies`` refuses."""
        pols = compile_policies(policies)
        B = len(batch) if isinstance(batch, (RaggedImages, EncodedImages)) else int(batch.shape[0])
        self.check_tta_policies(B, pols, replicas, parity)
        T, K = len(pols), int(replicas)
        x = self._decoded(batch)
        y = augment_tta_policies(pols, x, TailSpec.raw_u8(), K, seed, first_index)
        if not isinstance(y, RaggedImages):
            y = y.view(T * K * B, *y.shape[3:])
        out = self._tta_stages(x, y, B, T * K, seed, first_index)
        return out.view(T, K, B, *out.shape[1:])

    def test(self, batch_u8, out=None):
        """uint8 [B,H,W,3] CUDA (or ``RaggedImages``) -> [B, 3, s, s]: center crop + resize + ToTensor + Normalize, one
        launch (an ``EncodedImages`` batch is decoded first)"""
        return crop_resize(self._decoded(batch_u8), self.input_size, rng=self.center.cfg(), tail=self.test_tail, out=out)


def policy_by_conf_name(aug):
    """conf['aug'] -> policy list, with the reference's error behaviour (data.py:85-109)."""
    if isinstance(aug, list):
        return aug
    if aug in archive.BY_CONF_NAME:
        return archive.BY_CONF_NAME[aug]()
    if aug in ("default",):
        return None
    raise ValueError("not found augmentations. %s" % aug)


class SubsetSampler(Sampler):
    """Reference ``SubsetSampler`` (data.py:349-362): the given indices, in order."""

    def __init__(self, indices):
        self.indices = indices

    def __iter__(self):
        return (i for i in self.indices)

    def __len__(self):
        return len(self.indices)


class DeviceDataset:
    """uint8 images [N,H,W,3] + int64 targets living on the device - the counterpart of the reference's
    torchvision dataset objects (``total_trainset`` / ``testset``, data.py:114-196); ``targets`` stays a host
    list like torchvision's so that the stratified splits see what the reference's see."""

    def __init__(self, images, targets, device="cuda"):
        self.images = torch.as_tensor(np.ascontiguousarray(images) if isinstance(images, np.ndarray) else images)
        if self.images.dtype != torch.uint8 or self.images.dim() != 4 or self.images.shape[-1] != 3:
            raise ValueError("images must be uint8 [N, H, W, 3]")
        self.images = self.images.to(device).contiguous()
        self.targets = [int(t) for t in targets]
        self.labels = torch.as_tensor(self.targets, dtype=torch.int64, device=device)

    def __len__(self):
        return self.images.shape[0]

    def subset(self, idx):
        idx = [int(i) for i in idx]
        t = torch.as_tensor(idx, dtype=torch.int64, device=self.images.device)
        d = DeviceDataset.__new__(DeviceDataset)
        d.images = self.images.index_select(0, t)
        d.targets = [self.targets[i] for i in idx]
        d.labels = self.labels.index_select(0, t)
        return d


class RaggedDeviceDataset:
    """``DeviceDataset`` of differently sized uint8 images (``RaggedImages`` on the device) + int64 targets: the
    ImageNet sources of the ``faa_crop_resize`` loaders."""

    def __init__(self, images, targets, device="cuda"):
        if isinstance(images, RaggedImages):
            self.images = RaggedImages(images.storage.to(device), images.offsets, images.sizes)
        else:
            self.images = RaggedImages.from_list(images, device)
        self.targets = [int(t) for t in targets]
        if len(self.targets) != len(self.images):
            raise ValueError("need one target per image")
        self.labels = torch.as_tensor(self.targets, dtype=torch.int64, device=device)

    def __len__(self):
        return len(self.images)

    def subset(self, idx):
        idx = [int(i) for i in idx]
        d = RaggedDeviceDataset.__new__(RaggedDeviceDataset)
        d.images = self.images.select(idx)
        d.targets = [self.targets[i] for i in idx]
        d.labels = self.labels.index_select(0, torch.as_tensor(idx, dtype=torch.int64, device=self.labels.device))
        return d


class EncodedDeviceDataset:
    """``RaggedDeviceDataset`` of JPEG files: the files' bytes stay on the device (``EncodedImages``, headers parsed
    once here) and every batch is decoded on the device before its chain runs.  ``progressive``: progressive files
    are taken too (``EncodedImages.from_bytes(..., progressive=True)``).  ``find``: each batch's restart-free files
    without a scan index get one found on the device first (``decode_jpeg(find=True)``), so they decode on many
    threads; the pixels are the same.  ``progressive_index``: progressive files take a scan index
    (``from_bytes(..., progressive_index=True)``), so the ones that carry or find none decode as they do without it."""

    def __init__(self, files, targets, device="cuda", progressive=False, find=False, progressive_index=False):
        if progressive_index and not progressive:
            raise ValueError("progressive_index needs progressive")
        self.images = files if isinstance(files, EncodedImages) else EncodedImages.from_bytes(
            files, device, progressive, progressive_index)
        self.find = bool(find)
        self.targets = [int(t) for t in targets]
        if len(self.targets) != len(self.images):
            raise ValueError("need one target per image")
        self.labels = torch.as_tensor(self.targets, dtype=torch.int64, device=device)

    def __len__(self):
        return len(self.images)

    def subset(self, idx):
        idx = [int(i) for i in idx]
        d = EncodedDeviceDataset.__new__(EncodedDeviceDataset)
        d.images = self.images.select(idx)
        d.find = self.find
        d.targets = [self.targets[i] for i in idx]
        d.labels = self.labels.index_select(0, torch.as_tensor(idx, dtype=torch.int64, device=self.labels.device))
        return d


class FilePaths(list):
    """Paths of image files that stay on disk (the ImageNet directory source of ``_load_arrays``); ``split`` and
    ``folder`` name the split folder they were listed from."""
    split = folder = None


JPEG_INDEX_VERSION = 1


class JpegIndex:
    """The scan indexes of one split folder's files (``python -m fast_autoaugment_b200.jpeg_index``, file
    ``<split>.npz``: ``paths`` relative to the folder, ``sizes`` the file lengths, ``first`` / ``points`` as
    ``build_jpeg_index`` gives them, ``version``).  A file is looked up by its path relative to ``folder``; a file the
    index does not list, or whose length differs from the one indexed, gets no points.  Any other staleness (a file
    rewritten at the same length) is caught by the decoder, which then decodes that file serially.

    ``add`` enters files' points found later (``conf['faa_jpeg_index_learn']``: a loader's recording decodes); they
    replace the ones listed for the same path.  ``delta`` hands out what ``add`` entered since the last ``delta`` and
    ``merge`` enters another process's delta with the same replace semantics (``distributed.share_jpeg_index``); merged
    entries are never part of a later delta, so a rank sends only what it learned itself.  In memory an index takes
    about what its file takes on disk: 16 bytes a point, up to 127 points a file (about 1.7 KB at ImageNet's mean file
    size of about 110 KB)."""

    def __init__(self, folder, paths, sizes, first, points):
        self.folder = os.fspath(folder)
        self._added = {}                           # relative path -> (length, points) entered by add
        self._merged = {}                          # relative path -> (length, points) entered by merge
        self._unsent = {}                          # relative paths add entered since the last delta (ordered set)
        self.sizes = np.asarray(sizes, np.int64).reshape(-1)
        self.first = np.asarray(first, np.int64).reshape(-1)
        self.points = np.ascontiguousarray(points, dtype=_lib.JPEG_SYNC_DTYPE).reshape(-1)
        self._at = {os.fsdecode(bytes(p)) if isinstance(p, (bytes, np.bytes_)) else os.fspath(p): i
                    for i, p in enumerate(paths)}
        if len(self.first) != len(self._at) + 1 or len(self.sizes) != len(self._at) or \
                (np.diff(self.first) < 0).any() or self.first[0] != 0 or self.first[-1] != len(self.points):
            raise ValueError("inconsistent JPEG index")

    @staticmethod
    def load(path, folder):
        with np.load(path, allow_pickle=False) as z:
            if int(z["version"]) != JPEG_INDEX_VERSION:
                raise ValueError("%s: JPEG index version %d, this package reads version %d" % (
                    path, int(z["version"]), JPEG_INDEX_VERSION))
            return JpegIndex(folder, list(z["paths"]), z["sizes"], z["first"], z["points"])

    @staticmethod
    def empty(folder):
        """an index of ``folder`` that lists no file"""
        return JpegIndex(folder, [], np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros(0, _lib.JPEG_SYNC_DTYPE))

    def save(self, path):
        """write the index, ``add``'s and ``merge``'s files included, as ``<split>.npz`` of ``python -m
        fast_autoaugment_b200.jpeg_index``"""
        rel = sorted(self._at, key=self._at.get)
        sizes, first, points = self.sizes, self.first, self.points
        if self._added or self._merged:
            added = {**self._merged, **self._added}
            rel = [p for p in rel if p not in added]
            at = [self._at[p] for p in rel]
            parts = [self.points[self.first[i]:self.first[i + 1]] for i in at] + [q for _, q in added.values()]
            sizes = np.array([int(self.sizes[i]) for i in at] + [n for n, _ in added.values()], np.int64)
            first = np.zeros(len(parts) + 1, np.int64)
            first[1:] = np.cumsum([len(q) for q in parts])
            points = np.concatenate(parts) if parts else self.points[:0]
            rel += list(added)
        np.savez(path, paths=np.array([os.fsencode(p) for p in rel], dtype=bytes), sizes=sizes,
                 first=first, points=points, version=np.int64(JPEG_INDEX_VERSION))

    def add(self, paths, lengths, first, points):
        """enter the points of the files at ``paths`` (of ``lengths`` bytes): file k's are ``points[first[k]:first[k +
        1]]`` (``build_jpeg_index``'s form); they replace what the index lists for those paths"""
        for k, p in enumerate(paths):
            q = np.array(points[int(first[k]):int(first[k + 1])], dtype=_lib.JPEG_SYNC_DTYPE)
            rel = os.path.relpath(os.fspath(p), self.folder)
            self._added[rel] = (int(lengths[k]), q)
            self._merged.pop(rel, None)
            self._unsent[rel] = None

    def delta(self):
        """``(paths, lengths, first, points)``: the entries ``add`` entered since the last ``delta``, as ``save`` writes
        them (relative paths as bytes, file lengths, point offsets, points); what ``merge`` takes.  The call starts the
        next delta."""
        rel = list(self._unsent)
        self._unsent = {}
        parts = [self._added[p][1] for p in rel]
        first = np.zeros(len(rel) + 1, np.int64)
        first[1:] = np.cumsum([len(q) for q in parts])
        return (np.array([os.fsencode(p) for p in rel], dtype=bytes),
                np.array([self._added[p][0] for p in rel], np.int64), first,
                np.concatenate(parts) if parts else self.points[:0].copy())

    def merge(self, paths, lengths, first, points):
        """enter another index's ``delta``: file k (``paths[k]`` relative to the folder, bytes or str) of ``lengths[k]``
        bytes has points ``points[first[k]:first[k + 1]]``; they replace what the index lists for those paths.  Raises
        ValueError, entering nothing, for a delta whose parts do not fit together."""
        n = len(paths)
        lengths = np.asarray(lengths, np.int64).reshape(-1)
        first = np.asarray(first, np.int64).reshape(-1)
        points = np.asarray(points)
        if points.dtype != _lib.JPEG_SYNC_DTYPE:
            raise ValueError("JPEG index delta: points must be of JPEG_SYNC_DTYPE")
        rel = [os.fsdecode(bytes(p)) if isinstance(p, (bytes, np.bytes_)) else os.fspath(p) for p in paths]
        if len(lengths) != n or len(first) != n + 1 or first[0] != 0 or (np.diff(first) < 0).any() or \
                first[-1] != points.size or (lengths < 0).any():
            raise ValueError("JPEG index delta: inconsistent parts")
        if any(not p or os.path.isabs(p) for p in rel):
            raise ValueError("JPEG index delta: paths must be relative to the split folder")
        points = points.reshape(-1).copy()             # one copy; the entries are views of it
        first, lengths = first.tolist(), lengths.tolist()
        for k, p in enumerate(rel):
            self._merged[p] = (lengths[k], points[first[k]:first[k + 1]])
            self._added.pop(p, None)
            self._unsent.pop(p, None)

    def lookup(self, path, length):
        """the points of the file at ``path`` (of ``length`` bytes), empty when it has none here"""
        rel = os.path.relpath(os.fspath(path), self.folder)
        e = self._added.get(rel)
        if e is None:
            e = self._merged.get(rel)
        if e is not None:
            return e[1] if e[0] == int(length) else self.points[:0]
        i = self._at.get(rel)
        if i is None or int(self.sizes[i]) != int(length):
            return self.points[:0]
        return self.points[self.first[i]:self.first[i + 1]]

    def gather(self, paths, lengths):
        """(first, points) of a batch of files, as ``EncodedImages`` carries them"""
        parts = [self.lookup(p, n) for p, n in zip(paths, lengths)]
        first = np.zeros(len(parts) + 1, np.int64)
        first[1:] = np.cumsum([len(q) for q in parts])
        return first, (np.concatenate(parts) if parts else self.points[:0])


class JpegFileDataset:
    """``EncodedDeviceDataset`` whose files stay on disk: it holds paths and targets only, so no byte of the split is on
    the device.  ``GpuAugmentedLoader`` streams each batch's files through a ``FileBatchStream``.  ``index``: a
    ``JpegIndex`` of the files, whose scan indexes let the device decode each listed file on many threads.  ``learn``:
    the loaders enter into ``index`` (which it needs) the scan index of every file they decode serially, so the next
    epoch decodes it on many threads; subsets share the index, and ``index.save`` writes it.  ``progressive``: the
    loaders decode progressive files on the device instead of with Pillow (``read_jpeg_batch``).  ``find``: the loaders
    find the scan index of every restart-free file the index does not list on the device, in parallel, before decoding
    it on many threads (``decode_jpeg(find=True)``); with ``learn`` the found points are what the index learns.
    ``progressive_index`` (with ``progressive``): progressive files take a scan index as baseline files do, looked up
    in ``index`` and, with ``learn``, learned from the loaders' recording decodes."""

    def __init__(self, paths, targets, device="cuda", index=None, learn=False, progressive=False, find=False,
                 progressive_index=False):
        if learn and index is None:
            raise ValueError("learn needs an index to enter the files' points into (JpegIndex.empty)")
        if progressive_index and not progressive:
            raise ValueError("progressive_index needs progressive")
        self.progressive_index = bool(progressive_index)
        self.paths = [os.fspath(p) for p in paths]
        self.index = index
        self.learn = bool(learn)
        self.progressive = bool(progressive)
        self.find = bool(find)
        self.targets = [int(t) for t in targets]
        if len(self.targets) != len(self.paths):
            raise ValueError("need one target per image")
        self.labels = torch.as_tensor(self.targets, dtype=torch.int64, device=device)
        self.device = self.labels.device

    def __len__(self):
        return len(self.paths)

    def select(self, idx):
        """the paths of a batch"""
        return [self.paths[int(i)] for i in idx]

    def subset(self, idx):
        idx = [int(i) for i in idx]
        d = JpegFileDataset.__new__(JpegFileDataset)
        d.paths = self.select(idx)
        d.index, d.learn, d.progressive, d.find = self.index, self.learn, self.progressive, self.find
        d.progressive_index = self.progressive_index
        d.targets = [self.targets[i] for i in idx]
        d.labels = self.labels.index_select(0, torch.as_tensor(idx, dtype=torch.int64, device=self.labels.device))
        d.device = self.device
        return d


def _read_file(path):
    with open(path, "rb") as f:
        return f.read()


def _pillow_rgb(path_and_bytes):
    """``Image.open(f).convert('RGB')`` (reference imagenet.py:80, torchvision's ``pil_loader``) of a file the device
    decoder refuses; Pillow's error names the path"""
    path, b = path_and_bytes
    try:
        with PIL.Image.open(io.BytesIO(b)) as im:
            return np.ascontiguousarray(np.asarray(im.convert("RGB")))
    except OSError as e:
        raise OSError("%s: %s" % (path, e)) from e


class HostBatch:
    """The host half of staging one batch of files (``read_jpeg_batch``): ``paths``; ``files``, ``headers`` and the
    table ``pool`` of the files the device decoder takes (headers' ``offset`` places those files back to back, as
    ``EncodedImages.from_bytes`` of them would); the batch positions of those files (``accepted``) and of the rest
    (``refused``), and Pillow's pixels of the refused ones (``pixels``, uint8 [h, w, 3]); with an index, the accepted
    files' scan indexes (``first``, ``points``, as ``EncodedImages`` carries them; otherwise None); when progressive
    files were accepted, the accepted files' scans (``scans``, ``scan_first``, as ``EncodedImages`` carries them;
    otherwise None)."""

    def __init__(self, paths, files, headers, pool, accepted, refused, pixels, first=None, points=None, scans=None,
                 scan_first=None):
        self.paths, self.files, self.headers, self.pool = paths, files, headers, pool
        self.accepted, self.refused, self.pixels = accepted, refused, pixels
        self.first, self.points = first, points
        self.scans, self.scan_first = scans, scan_first

    def sizes(self):
        """(h, w) of every image of the batch, int32 [N, 2]"""
        s = np.zeros((len(self.paths), 2), np.int32)
        s[self.accepted, 0], s[self.accepted, 1] = self.headers["h"], self.headers["w"]
        for i, px in zip(self.refused, self.pixels):
            s[i] = px.shape[:2]
        return s


def read_jpeg_batch(paths, map=map, index=None, progressive=False, progressive_index=False):
    """Read a batch of files and parse their headers (``parse_jpeg_headers``); decode the files the device decoder
    refuses with Pillow; with a ``JpegIndex``, gather the accepted files' scan indexes.  No device is touched.  ``map``:
    an executor's ``map`` reads, parses and decodes in parallel.  ``progressive=True``: progressive files are accepted
    with their scans instead of decoded by Pillow; ``progressive_index=True``: they take a scan index too."""
    paths = list(paths)
    files = list(map(_read_file, paths))
    scans = scan_first = None
    if progressive:
        headers, pool, refused, scans, scan_first = parse_jpeg_headers(files, map, progressive=True,
                                                                       progressive_index=progressive_index)
    else:
        headers, pool, refused = parse_jpeg_headers(files, map)
    bad = np.array([i for i, _ in refused], np.int64)
    ok = np.setdiff1d(np.arange(len(files), dtype=np.int64), bad)
    lengths = np.array([len(files[i]) for i in ok], np.int64)
    headers = headers[ok]
    headers["offset"] = np.cumsum(lengths) - lengths
    pixels = list(map(_pillow_rgb, [(paths[i], files[i]) for i in bad]))
    first = points = None
    if index is not None:
        first, points = index.gather([paths[i] for i in ok], lengths)
    if scans is not None and len(scans):
        scan_first = np.concatenate([scan_first[ok], scan_first[-1:]]).astype(np.int64)
    else:
        scans = scan_first = None
    return HostBatch(paths, [files[i] for i in ok], headers, pool, ok, bad, pixels, first, points, scans, scan_first)


def chunked_map(pool_map, n_chunks):
    """``map`` over ``n_chunks`` contiguous chunks of the items, one ``pool_map`` task per chunk: a task per file
    costs more than parsing a header"""
    def run(fn, items):
        items = list(items)
        step = max(1, -(-len(items) // max(1, n_chunks)))
        parts = pool_map(lambda xs: [fn(x) for x in xs], [items[i:i + step] for i in range(0, len(items), step)])
        return [r for part in parts for r in part]
    return run


def _up16(n):
    return (int(n) + 15) // 16 * 16


class _Layout:
    """Byte layout of one staged batch, the same in the pinned slot and in the batch's device buffer: headers, table
    pool, the accepted files back to back, the refused files' pixels, then (with an index) the accepted files' point
    offsets and points, then (with progressive files) their scan offsets and scans, each part on a 16-byte boundary.
    A batch without progressive files has the layout it would have without the option."""

    def __init__(self, hb: HostBatch):
        self.pool = _up16(hb.headers.nbytes)
        self.files = self.pool + _up16(hb.pool.nbytes)
        self.files_end = self.files + sum(len(f) for f in hb.files)
        self.pixels, at = [], _up16(self.files_end)
        for px in hb.pixels:
            self.pixels.append(at)
            at = _up16(at + px.nbytes)
        self.first = self.points = self.points_end = None
        if hb.first is not None:
            self.first = at
            self.points = _up16(at + hb.first.nbytes)
            self.points_end = self.points + hb.points.nbytes
            at = _up16(self.points_end)
        self.scan_first = self.scans = self.scans_end = None
        if hb.scans is not None:
            self.scan_first = at
            self.scans = _up16(at + hb.scan_first.nbytes)
            self.scans_end = self.scans + hb.scans.nbytes
            at = _up16(self.scans_end)
        self.total = max(at, 16)

    def pack(self, hb: HostBatch, buf):
        buf[:hb.headers.nbytes] = hb.headers.view(np.uint8).reshape(-1)
        buf[self.pool:self.pool + hb.pool.nbytes] = hb.pool.view(np.uint8).reshape(-1)
        at = self.files
        for f in hb.files:
            buf[at:at + len(f)] = np.frombuffer(f, np.uint8)
            at += len(f)
        for o, px in zip(self.pixels, hb.pixels):
            buf[o:o + px.nbytes] = px.reshape(-1)
        if self.first is not None:
            buf[self.first:self.first + hb.first.nbytes] = hb.first.view(np.uint8)
            buf[self.points:self.points_end] = hb.points.view(np.uint8).reshape(-1)
        if self.scans is not None:
            buf[self.scan_first:self.scan_first + hb.scan_first.nbytes] = hb.scan_first.view(np.uint8)
            buf[self.scans:self.scans_end] = hb.scans.view(np.uint8).reshape(-1)


_STATUS_BITS = ((_lib.JPEG_TRUNCATED, "scan truncated"), (_lib.JPEG_BAD_CODE, "bad Huffman code"),
                (_lib.JPEG_BAD_COEF, "run past coefficient 63"), (_lib.JPEG_BAD_RESTART, "bad restart marker"))


class FileBatchStream:
    """Batches of JPEG files read from disk, decoded into ``RaggedImages`` on the device, staged one batch ahead.

    While the device runs batch k, a host thread stages batch k + 1: a small thread pool reads its files and parses
    their headers (``read_jpeg_batch``; ctypes releases the GIL in ``faa_jpeg_parse``), and the thread packs headers,
    table pool, files and the Pillow pixels of refused files into one of ``SLOTS`` pinned staging buffers, once the
    event recorded after that slot's previous copy shows the copy finished.  The caller's thread makes one
    ``non_blocking`` copy of the slot into a device buffer of the batch, decodes the accepted files (``decode_jpeg``)
    into their images of ``RaggedImages.empty(sizes)`` and copies the refused files' pixels into theirs.  Each batch's
    decode status is copied to pinned host memory and checked once the next batch is staged, and at the end, so no
    batch waits on its own decode: a non-zero status raises ``OSError`` naming the file.  With a ``JpegIndex`` each
    batch's scan indexes travel in the same slot and the decode uses them.  With ``learn`` as well, every batch is
    decoded in recording mode (``decode_jpeg(record=True)``): its point counts and the points they cover are copied to
    pinned memory behind the decode with its status, and at the same check the files that got points are entered into
    the index (``JpegIndex.add``), so the batches read after that decode them on many threads.  With ``progressive``,
    progressive files are decoded on the device too: their scans travel in the same slot.  With ``find``, every batch
    is decoded by ``decode_jpeg(find=True)``: files without points get a scan index found on the device first and
    decode on many threads; with ``learn``, the files whose found index converged are entered with those points.
    With ``progressive_index`` as well as ``progressive``, progressive files are looked up and learned like the others.
    """

    SLOTS = 2
    WORKERS = 2

    def __init__(self, workers=None, index=None, learn=False, progressive=False, find=False, progressive_index=False):
        if learn and index is None:
            raise ValueError("learn needs an index")
        if progressive_index and not progressive:
            raise ValueError("progressive_index needs progressive")
        self.progressive_index = bool(progressive_index)
        self.workers = int(workers or self.WORKERS)
        self.index = index
        self.learn = bool(learn)
        self.progressive = bool(progressive)
        self.find = bool(find)
        self.slots = [None] * self.SLOTS           # pinned uint8 staging buffers
        self.copied = [None] * self.SLOTS          # event recorded after each slot's last host-to-device copy

    def _stage(self, paths, slot, pool, dev):
        hb = read_jpeg_batch(paths, chunked_map(pool.map, self.workers) if self.workers > 1 else map, self.index,
                             self.progressive, self.progressive_index)
        lay = _Layout(hb)
        if self.copied[slot] is not None:
            self.copied[slot].synchronize()
        buf = self.slots[slot]
        if buf is None or buf.numel() < lay.total:
            with torch.cuda.device(dev):
                buf = self.slots[slot] = torch.empty(lay.total + lay.total // 4, dtype=torch.uint8, pin_memory=True)
        lay.pack(hb, buf.numpy())
        return hb, lay, slot

    def _decode(self, hb, lay, dbuf, dev, pending):
        sizes = hb.sizes()
        out = RaggedImages.empty(sizes, dev)
        if len(hb.accepted):
            index = {}
            if hb.first is not None:
                index = dict(first=hb.first, points=hb.points,
                             _d_first=dbuf[lay.first:lay.first + hb.first.nbytes].view(torch.int64),
                             _d_points=dbuf[lay.points:lay.points_end])
            if hb.scans is not None:
                index.update(scans=hb.scans, scan_first=hb.scan_first, _d_scans=dbuf[lay.scans:lay.scans_end],
                             _d_scan_first=dbuf[lay.scan_first:lay.scan_first + hb.scan_first.nbytes].view(torch.int64))
            enc = EncodedImages(dbuf[lay.files:lay.files_end], hb.headers, hb.pool, _d_pool=dbuf[lay.pool:lay.files],
                                _d_headers=dbuf[:lay.pool], **index)
            learned = None
            find = {"find": True} if self.find else {}
            if self.learn:
                _, status, count, points, cap_first = decode_jpeg(enc, out.select(hb.accepted), record=True, **find)
                h_count = torch.empty(len(hb.accepted), dtype=torch.int32, pin_memory=True)
                h_count.copy_(count, non_blocking=True)
                h_points = torch.empty(points.numel(), dtype=torch.uint8, pin_memory=True)
                h_points.copy_(points, non_blocking=True)
                learned = (h_count, h_points, cap_first, [len(f) for f in hb.files])
            else:
                _, status = decode_jpeg(enc, out.select(hb.accepted), **find)
            queue_status(status, [hb.paths[i] for i in hb.accepted], dev, pending, learned)
        for i, o in zip(hb.refused, lay.pixels):
            h, w = (int(v) for v in sizes[i])
            out.image(int(i)).copy_(dbuf[o:o + h * w * 3].view(h, w, 3))
        return out

    def _check(self, pending, keep=0):
        check_decodes(pending, keep, self.index)

    def __call__(self, batches, device):
        """generator of one ``RaggedImages`` per batch of paths in ``batches``"""
        dev = torch.device(device)
        pool = ThreadPoolExecutor(self.workers, thread_name_prefix="faa-read")
        ahead = ThreadPoolExecutor(1, thread_name_prefix="faa-stage")
        pending = []                               # (event, pinned status, paths, recorded points) of unchecked decodes
        try:
            fut = ahead.submit(self._stage, batches[0], 0, pool, dev) if len(batches) else None
            for k in range(len(batches)):
                hb, lay, slot = fut.result()
                dbuf = torch.empty(lay.total, dtype=torch.uint8, device=dev)
                dbuf.copy_(self.slots[slot][:lay.total], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(dev))
                self.copied[slot] = ev
                if k + 1 < len(batches):
                    fut = ahead.submit(self._stage, batches[k + 1], (k + 1) % self.SLOTS, pool, dev)
                out = self._decode(hb, lay, dbuf, dev, pending)
                self._check(pending, keep=1 if len(hb.accepted) else 0)      # the batches before this one
                yield out
            self._check(pending)
        finally:
            ahead.shutdown(wait=True, cancel_futures=True)
            pool.shutdown(wait=True, cancel_futures=True)


def queue_status(status, paths, dev, pending, learned=None):
    """copy a decode's status (and what a recording decode recorded, ``learned``) to pinned memory behind the decode and
    append it to ``pending`` for ``check_decodes``, so no batch waits on its own decode"""
    st = torch.empty(len(paths), dtype=torch.int32, pin_memory=True)
    st.copy_(status, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    pending.append((ev, st, paths, learned))


def check_decodes(pending, keep=0, index=None):
    """check (and drop) every pending status but the last ``keep``: OSError naming every file whose status is not 0;
    enter into ``index`` what recording decodes found"""
    while len(pending) > keep:
        ev, st, paths, learned = pending.pop(0)
        ev.synchronize()
        if learned is not None:
            h_count, h_points, cap_first, lengths = learned
            count = h_count.numpy()
            first, points = compact_jpeg_index(cap_first, count, h_points.numpy())
            got = np.flatnonzero(count > 0)
            index.add([paths[i] for i in got], [lengths[i] for i in got],
                      np.concatenate([[0], np.cumsum(count[got])]), points)
        codes = st.numpy()
        bad = [(paths[i], int(codes[i])) for i in np.flatnonzero(codes)]
        if bad:
            raise OSError("corrupt JPEG files (decode status): " + "; ".join(
                "%s: 0x%x (%s)" % (p, s, ", ".join(n for b, n in _STATUS_BITS if s & b)) for p, s in bad))


RESIDENT_CHUNK = 256                   # files per read_jpeg_batch call while a resident store is built
RESIDENT_INDEX_CHUNK = 1024            # files per build_jpeg_index call over a shard
RESIDENT_STAGE = 64 << 20              # bytes of host staging per upload of a shard's parts
# host metadata of one file of a resident store: its header (``offset``: its bytes in the owner's shard; ``pool``: rows
# of the owner's table region), its tables (``n_tables`` rows from row ``table_at``), its points (``n_points`` from
# byte ``points_at`` of the shard), a refused file's pixels (``refused``, h x w x 3 bytes from byte ``pixels_at``) and
# the number of its progressive scans
RESIDENT_META_DTYPE = np.dtype([("hdr", _lib.JPEG_HEADER_DTYPE), ("table_at", "<i8"), ("n_tables", "<i8"),
                                ("points_at", "<i8"), ("n_points", "<i8"), ("pixels_at", "<i8"), ("h", "<i4"),
                                ("w", "<i4"), ("refused", "<i4"), ("n_scans", "<i4")])
_TABLE_BYTES = _lib.JPEG_TABLE_DTYPE.itemsize


def resident_owned(n, local_rank, n_local):
    """the files of an n-file split that local rank ``local_rank`` of ``n_local`` ranks on its host holds: file i
    belongs to local rank i mod n_local"""
    return np.arange(int(local_rank), int(n), int(n_local), dtype=np.int64)


def _used_slots(hdr, sc):
    """(header slots, [(scan, slot)]) of a parsed file that name a table: a baseline file's slots s with s % 3 <
    ncomp; a progressive file's first ncomp header slots and its scans' slots whose DC or AC table exists"""
    nc = int(hdr["ncomp"])
    if not int(hdr["reserved"]) & _lib.JPEG_PROGRESSIVE:
        return [s for s in range(9) if s % 3 < nc], []
    return list(range(nc)), [(k, t) for k in range(len(sc)) for t in range(6)
                             if (sc["dc_at"][k] if t < 3 else sc["ac_at"][k])[t % 3] != -1]


class ShardPlan:
    """The host half of one rank's shard of a resident store, from its files' ``read_jpeg_batch`` results (``hbs``, in
    ownership order): ``meta`` (``RESIDENT_META_DTYPE`` [n]), ``scans`` (the progressive files' scans, file order, pool
    slots in shard rows), ``tables`` (``JPEG_TABLE_DTYPE``: each accepted file's own tables, in file order) and the
    byte layout of the shard: the accepted files' bytes from byte 0, the tables from ``tables_off``, room for the points
    from ``points_off``, the refused files' pixels from ``pixels_off``, each item on a 16-byte boundary; ``need`` bytes.

    ``index``: a ``JpegIndex`` whose points the files take (``points``), exactly sized; without one each accepted file
    gets room for the most points it can get (``jpeg_index_capacities``) and ``n_points`` 0 until ``build_points``."""

    def __init__(self, hbs, index=None):
        metas, scans, tables, points = [], [], [], []
        self.files, self.pixels = [], []
        n_tab = 0
        for hb in hbs:
            m = np.zeros(len(hb.paths), RESIDENT_META_DTYPE)
            m["refused"][hb.refused] = 1
            for i, px in zip(hb.refused, hb.pixels):
                m["h"][i], m["w"][i] = px.shape[:2]
            for a, i in enumerate(hb.accepted):
                hdr = hb.headers[a].copy()
                sc = hb.scans[hb.scan_first[a]:hb.scan_first[a + 1]].copy() if hb.scans is not None else hb.scans
                used_h, used_s = _used_slots(hdr, sc)
                uniq = sorted({int(hdr["pool"][s]) for s in used_h} | {int(sc["pool"][k, t]) for k, t in used_s})
                row = {s: n_tab + j for j, s in enumerate(uniq)}
                pool = np.full(9, n_tab, np.int32)            # slots that name no table point at the file's first row
                pool[used_h] = [row[int(hdr["pool"][s])] for s in used_h]
                hdr["pool"] = pool
                if sc is not None and len(sc):
                    sp = np.full((len(sc), 6), n_tab, np.int32)
                    for k, t in used_s:
                        sp[k, t] = row[int(sc["pool"][k, t])]
                    sc["pool"] = sp
                    scans.append(sc)
                    m["n_scans"][i] = len(sc)
                tables.append(hb.pool[uniq])
                m["hdr"][i] = hdr
                m["table_at"][i], m["n_tables"][i] = n_tab, len(uniq)
                m["h"][i], m["w"][i] = hdr["h"], hdr["w"]
                n_tab += len(uniq)
            if index is not None:
                first, pts = index.gather([hb.paths[i] for i in hb.accepted], [len(f) for f in hb.files])
                m["n_points"][hb.accepted] = np.diff(first)
                points.append(pts)
            metas.append(m)
            self.files += hb.files
            self.pixels += hb.pixels
        self.meta = np.concatenate(metas) if metas else np.zeros(0, RESIDENT_META_DTYPE)
        self.scans = np.concatenate(scans) if scans else np.zeros(0, _lib.JPEG_SCAN_DTYPE)
        self.tables = np.concatenate(tables) if tables else np.zeros(0, _lib.JPEG_TABLE_DTYPE)
        self.points = np.concatenate(points) if points else np.zeros(0, _lib.JPEG_SYNC_DTYPE)
        m = self.meta
        acc = np.flatnonzero(m["refused"] == 0)
        self.accepted = acc
        slot = (m["hdr"]["len"][acc] + 15) // 16 * 16
        m["hdr"]["offset"][acc] = np.cumsum(slot) - slot
        self.tables_off = int(slot.sum())
        self.points_off = self.tables_off + len(self.tables) * _TABLE_BYTES
        room = m["n_points"][acc] if index is not None else np.diff(jpeg_index_capacities(m["hdr"][acc]))
        m["points_at"][acc] = self.points_off + 16 * (np.cumsum(room) - room)
        self.pixels_off = self.points_off + 16 * int(room.sum())
        ref = np.flatnonzero(m["refused"] != 0)
        px = (m["h"][ref].astype(np.int64) * m["w"][ref] * 3 + 15) // 16 * 16
        m["pixels_at"][ref] = self.pixels_off + np.cumsum(px) - px
        self.need = max(16, self.pixels_off + int(px.sum()))

    def headers(self):
        """the accepted files' headers, ``offset`` and ``pool`` in the shard (file order)"""
        return self.meta["hdr"][self.accepted]

    def scan_first(self):
        n = self.meta["n_scans"][self.accepted].astype(np.int64)
        return np.concatenate([[0], np.cumsum(n)]).astype(np.int64)

    def parts(self):
        """[(shard byte offset, uint8 array)] of everything but room for points not yet built, in offset order"""
        m = self.meta
        out = [(int(o), np.frombuffer(f, np.uint8)) for o, f in zip(m["hdr"]["offset"][self.accepted], self.files)]
        out.append((self.tables_off, self.tables.view(np.uint8).reshape(-1)))
        if len(self.points):
            at = np.repeat(m["points_at"][self.accepted], m["n_points"][self.accepted])
            first = np.cumsum(m["n_points"][self.accepted]) - m["n_points"][self.accepted]
            rows = np.zeros(self.pixels_off - self.points_off, np.uint8).view(_lib.JPEG_SYNC_DTYPE)
            k = np.arange(len(self.points)) - np.repeat(first, m["n_points"][self.accepted])
            rows[(at - self.points_off) // 16 + k] = self.points
            out.append((self.points_off, rows.view(np.uint8)))
        ref = np.flatnonzero(m["refused"] != 0)
        out += [(int(o), p.reshape(-1)) for o, p in zip(m["pixels_at"][ref], self.pixels)]
        return out


def _upload(dst, parts):
    """copy ``parts`` ([(byte offset, uint8 array)] in offset order) into the device tensor ``dst`` through host
    staging spans of at most ``RESIDENT_STAGE`` bytes (larger parts go alone)"""
    k = 0
    while k < len(parts):
        start, j = parts[k][0], k
        while j < len(parts) and parts[j][0] + len(parts[j][1]) - start <= max(RESIDENT_STAGE, len(parts[k][1])):
            j += 1
        end = parts[j - 1][0] + len(parts[j - 1][1])
        buf = np.zeros(end - start, np.uint8)
        for o, a in parts[k:j]:
            buf[o - start:o - start + len(a)] = a
        dst[start:end].copy_(torch.from_numpy(buf))
        k = j


def pack_shard_meta(meta, scans, handle, device, tables_off):
    """one rank's part of a resident store's metadata exchange: int64 [files, scans, device, table region offset], the
    64-byte IPC handle, the files' ``RESIDENT_META_DTYPE`` rows, their scans"""
    head = np.array([len(meta), len(scans), int(device), int(tables_off)], np.int64)
    return np.concatenate([head.view(np.uint8), np.frombuffer(bytes(handle), np.uint8),
                           np.ascontiguousarray(meta).view(np.uint8).reshape(-1),
                           np.ascontiguousarray(scans).view(np.uint8).reshape(-1)])


def unpack_shard_meta(buf):
    """``pack_shard_meta``'s (meta, scans, handle, device, tables_off) of ``buf``; ValueError when its sizes do not
    add up"""
    if buf.size < 96:
        raise ValueError("%d bytes, shorter than a shard's metadata header" % buf.size)
    n, ns, device, tables_off = (int(v) for v in np.frombuffer(buf, np.int64, 4))
    if min(n, ns) < 0 or buf.size != 96 + n * RESIDENT_META_DTYPE.itemsize + ns * _lib.JPEG_SCAN_DTYPE.itemsize:
        raise ValueError("%d bytes do not hold %d files' metadata and %d scans" % (buf.size, n, ns))
    meta = np.frombuffer(buf, RESIDENT_META_DTYPE, n, 96)
    scans = np.frombuffer(buf, _lib.JPEG_SCAN_DTYPE, ns, 96 + meta.nbytes)
    if int(meta["n_scans"].sum()) != ns:
        raise ValueError("scan counts do not add up to %d scans" % ns)
    return meta, scans, buf[32:96].tobytes(), device, tables_off


class ResidentBatch:
    """The host plan of one batch of a resident store (``ResidentJpegStore.plan``): the output sizes (``sizes``), the
    batch positions of the accepted and refused files, the accepted files' headers (``offset`` in the batch's file
    region, ``pool`` in its table region), scan index (``first``; None when no file has points) and scans (``scans``,
    ``scan_first``; None when no file is progressive), the batch buffer's layout (tables from 0, files from
    ``files_at``, points from ``points_at``, ``total`` bytes) and the copies that fill it, ``jobs``."""

    def __init__(self, meta, src, scan_first, scans, sel):
        sel = np.asarray(sel, np.int64).reshape(-1)
        m = meta[sel]
        self.sizes = np.stack([m["h"], m["w"]], axis=1).astype(np.int32).reshape(-1, 2)
        self.accepted = np.flatnonzero(m["refused"] == 0)
        self.refused = np.flatnonzero(m["refused"] != 0)
        a = m[self.accepted]
        s_a, s_r = src[sel[self.accepted]], src[sel[self.refused]]
        n_tab = a["n_tables"]
        row0 = np.cumsum(n_tab) - n_tab
        self.n_tables = int(n_tab.sum())
        flen = a["hdr"]["len"]
        slot = (flen + 15) // 16 * 16
        self.files_at = self.n_tables * _TABLE_BYTES
        self.points_at = self.files_at + int(slot.sum())
        n_pts = a["n_points"]
        self.total = max(16, self.points_at + 16 * int(n_pts.sum()))
        self.headers = a["hdr"].copy()
        self.headers["offset"] = np.cumsum(slot) - slot
        self.headers["pool"] += (row0 - a["table_at"]).astype(np.int32)[:, None]
        self.first = None
        if n_pts.any():
            self.first = np.concatenate([[0], np.cumsum(n_pts)]).astype(np.int64)
        self.scans = self.scan_first = None
        n_sc = a["n_scans"].astype(np.int64)
        if n_sc.any():
            self.scan_first, self.scans = engine_gather_ranges(scan_first, scans, sel[self.accepted])
            self.scans["pool"] += np.repeat((row0 - a["table_at"]).astype(np.int32), n_sc)[:, None]
        tab_dst = _TABLE_BYTES * row0
        self._rel = (np.concatenate([s_a["tables"], s_a["file"], s_a["points"]]),
                     np.concatenate([tab_dst, self.files_at + self.headers["offset"],
                                     self.points_at + 16 * (np.cumsum(n_pts) - n_pts)]).astype(np.uint64),
                     np.concatenate([_TABLE_BYTES * n_tab, flen, 16 * n_pts]))
        self._pixels = (s_r["pixels"], m["h"][self.refused].astype(np.int64) * m["w"][self.refused] * 3)

    def jobs(self, buf_ptr, image_ptrs):
        """``COPY_DTYPE`` jobs of the batch: the accepted files' tables, bytes and points into the batch buffer at
        ``buf_ptr``, each refused file's pixels into its output image (``image_ptrs``: the refused files' image
        addresses, batch order).  Jobs of no byte are left out."""
        src, dst, n = self._rel
        out = np.zeros(len(src) + len(self._pixels[0]), _lib.COPY_DTYPE)
        out["src"] = np.concatenate([src, self._pixels[0]])
        out["dst"] = np.concatenate([dst + np.uint64(buf_ptr), np.asarray(image_ptrs, np.uint64).reshape(-1)])
        out["bytes"] = np.concatenate([n, self._pixels[1]])
        return out[out["bytes"] > 0]


_SRC_DTYPE = np.dtype([("file", "<u8"), ("tables", "<u8"), ("points", "<u8"), ("pixels", "<u8")])


class ResidentJpegStore:
    """A split's JPEG files held in device memory, sharded over the ranks of each host (``ResidentJpegDataset``).

    Construction is collective under ``multinode`` (every rank of the default group, or ``group``, calls it): the
    ranks on one host (``host_ranks``) split the files by ``resident_owned``; each reads and parses only its own
    (``read_jpeg_batch``, Pillow decoding the files the device decoder refuses), plans its shard (``ShardPlan``),
    checks it fits (``check_fit``), allocates it as one buffer the host's other processes can map (``faa_peer_alloc``),
    uploads it and, without ``index``, builds its files' scan indexes on its device (``build_jpeg_index``).  The ranks
    then all-gather their files' metadata (``gather_bytes``) and each maps its host peers' shards (``faa_peer_open``).
    Every rank enters the same collectives whatever fails locally, and a failure raises on every rank.

    After that no file is read: ``batches`` plans each batch on the host with vectorised numpy (``ResidentBatch``),
    uploads its job table, headers and scans in one pinned copy, fills the batch buffer and the refused files' output
    images with one ``faa_gather`` launch and decodes the accepted files as ``FileBatchStream`` does.  ``close`` is
    collective too."""

    def __init__(self, paths, device="cuda", index=None, progressive=False, progressive_index=False, multinode=False,
                 group=None, workers=4):
        self.paths = np.array([os.fspath(p) for p in paths], dtype=object)
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.multinode, self.group = bool(multinode), group
        self._own_ptr, self._opened = 0, []
        n = len(self.paths)
        rank = dist.get_rank(group) if self.multinode else 0
        peers = host_ranks(group) if self.multinode else [0]
        self.n_local, self.local_rank = len(peers), peers.index(rank)
        self.own = resident_owned(n, self.local_rank, self.n_local)
        t0 = time.perf_counter()
        err = plan = None
        try:
            with ThreadPoolExecutor(workers, thread_name_prefix="faa-resident") as pool:
                read = chunked_map(pool.map, workers)
                hbs = [read_jpeg_batch(self.paths[self.own[k:k + RESIDENT_CHUNK]], read, None, progressive,
                                       progressive_index) for k in range(0, len(self.own), RESIDENT_CHUNK)]
            plan = ShardPlan(hbs, index)
        except Exception as e:                                   # noqa: BLE001
            err = e
        self.timing = {"read": time.perf_counter() - t0}
        free = torch.cuda.mem_get_info(self.device)[0]
        if self.multinode:
            check_fit(None if plan is None else plan.need, free, err, group)
        elif err is not None:
            raise err
        elif plan.need > free:
            raise RuntimeError(fit_error([plan.need], [free]))
        self.device_bytes = plan.need
        self.n_tables = len(plan.tables)
        handle = None
        try:
            t0 = time.perf_counter()
            with torch.cuda.device(self.device):
                ptr, h = ctypes.c_void_p(), (ctypes.c_ubyte * 64)()
                _lib.check(_lib.lib.faa_peer_alloc(plan.need, ctypes.byref(ptr), h))
                self._own_ptr, handle = ptr.value, bytes(h)
                self.shard = torch.as_tensor(_RawCuda(self._own_ptr, (plan.need,)), device=self.device)
                _upload(self.shard, plan.parts())
                torch.cuda.synchronize(self.device)
                self.timing["upload"] = time.perf_counter() - t0
                t0 = time.perf_counter()
                if index is None:
                    self._build_points(plan)
                self.timing["index"] = time.perf_counter() - t0
        except Exception as e:                                   # noqa: BLE001
            err = e
        if not self.multinode:
            if err is not None:
                self._release()
                raise err
            self._install([(plan.meta, plan.scans, self._own_ptr, plan.tables_off)], [0])
            return
        t0 = time.perf_counter()
        try:
            self._exchange(plan, handle, err, peers, rank)
        except RuntimeError:
            self._release()
            raise
        self.timing["exchange"] = time.perf_counter() - t0

    def _exchange(self, plan, handle, err, peers, rank):
        """the collective metadata exchange and the mapping of the host peers' shards"""
        mine = None
        if err is None:
            try:
                mine = pack_shard_meta(plan.meta, plan.scans, handle, self.device.index, plan.tables_off)
            except Exception as e:                               # noqa: BLE001
                err = e
        bufs, err = gather_bytes(mine, err, self.group)
        if err is None:
            try:
                shards = []
                for r in peers:
                    meta, scans, h, dev, tables_off = unpack_shard_meta(bufs[r])
                    if r == rank:
                        base = self._own_ptr
                    else:
                        with torch.cuda.device(self.device):
                            _lib.check(_lib.lib.faa_enable_peer_access(dev))
                            p = ctypes.c_void_p()
                            _lib.check(_lib.lib.faa_peer_open((ctypes.c_ubyte * 64).from_buffer_copy(h), ctypes.byref(p)))
                        base = p.value
                        self._opened.append(base)
                    shards.append((meta, scans, base, tables_off))
                self._install(shards, peers)
            except Exception as e:                               # noqa: BLE001
                err = e
        agree(err, self.group, "resident JPEG store")

    def _build_points(self, plan):
        """the accepted files' scan indexes, built over the uploaded shard, written into their room"""
        acc = plan.accepted
        if not len(acc):
            return
        m = plan.meta
        scans = {}
        if len(plan.scans):
            scans = dict(scans=plan.scans, scan_first=plan.scan_first())
        enc = EncodedImages(self.shard[:plan.tables_off], plan.headers(), plan.tables,
                            _d_pool=self.shard[plan.tables_off:plan.points_off], **scans)
        counts, parts = [], []
        for k in range(0, len(acc), RESIDENT_INDEX_CHUNK):
            first, pts = build_jpeg_index(enc.select(np.arange(k, min(len(acc), k + RESIDENT_INDEX_CHUNK))))
            counts.append(np.diff(first))
            parts.append(pts)
        count = np.concatenate(counts)
        m["n_points"][acc] = count
        pts = np.concatenate(parts)
        if len(pts):
            rows = np.zeros((plan.pixels_off - plan.points_off) // 16, _lib.JPEG_SYNC_DTYPE)
            k = np.arange(len(pts)) - np.repeat(np.cumsum(count) - count, count)
            rows[(np.repeat(m["points_at"][acc], count) - plan.points_off) // 16 + k] = pts
            self.shard[plan.points_off:plan.pixels_off].copy_(torch.from_numpy(rows.view(np.uint8)))

    def _install(self, shards, peers):
        """the split-wide host arrays from every host peer's (meta, scans, base address, table region offset)"""
        n = len(self.paths)
        self.meta = np.zeros(n, RESIDENT_META_DTYPE)
        self.src = np.zeros(n, _SRC_DTYPE)
        self.owner = np.zeros(n, np.int64)
        own = [resident_owned(n, j, len(peers)) for j in range(len(peers))]
        for j, (meta, _, base, tables_off) in enumerate(shards):
            if len(meta) != len(own[j]):
                raise ValueError("local rank %d holds %d files, not %d" % (j, len(meta), len(own[j])))
            at = own[j]
            self.meta[at] = meta
            self.owner[at] = j
            b = np.uint64(base)
            self.src["file"][at] = b + meta["hdr"]["offset"].astype(np.uint64)
            self.src["tables"][at] = b + np.uint64(tables_off) + (meta["table_at"] * _TABLE_BYTES).astype(np.uint64)
            self.src["points"][at] = b + meta["points_at"].astype(np.uint64)
            self.src["pixels"][at] = b + meta["pixels_at"].astype(np.uint64)
        self.scan_first = np.concatenate([[0], np.cumsum(self.meta["n_scans"])]).astype(np.int64)
        self.scans = np.zeros(int(self.scan_first[-1]), _lib.JPEG_SCAN_DTYPE)
        for j, (meta, scans, _, _) in enumerate(shards):
            cnt = meta["n_scans"].astype(np.int64)
            to = np.repeat(self.scan_first[own[j]], cnt) + np.arange(len(scans)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            self.scans[to] = scans

    def plan(self, sel):
        """``ResidentBatch`` of the split's files ``sel``"""
        return ResidentBatch(self.meta, self.src, self.scan_first, self.scans, sel)

    def batches(self, batches):
        """generator of one ``RaggedImages`` per batch of split positions in ``batches``; each batch's decode status is
        checked once the next batch is queued, and at the end (``check_decodes``)"""
        dev = self.device
        pending = []
        for sel in batches:
            p = self.plan(sel)
            out = RaggedImages.empty(p.sizes, dev)
            buf = torch.empty(p.total, dtype=torch.uint8, device=dev)
            jobs = p.jobs(buf.data_ptr(), out.storage.data_ptr() + out.offsets[p.refused].astype(np.uint64))
            parts = [jobs, p.headers] + ([p.first] if p.first is not None else []) + \
                ([p.scan_first, p.scans] if p.scans is not None else [])
            at = np.cumsum([0] + [_up16(a.nbytes) for a in parts])
            host = torch.empty(int(at[-1]), dtype=torch.uint8, pin_memory=True)
            h = host.numpy()
            for o, a in zip(at, parts):
                h[o:o + a.nbytes] = a.view(np.uint8).reshape(-1)
            d = torch.empty(int(at[-1]), dtype=torch.uint8, device=dev)
            d.copy_(host, non_blocking=True)
            views = [d[o:o + a.nbytes] for o, a in zip(at, parts)]
            gather(jobs, views[0], dev)
            if len(p.accepted):
                kw = {}
                if p.first is not None:
                    kw.update(first=p.first, points=np.empty(int(p.first[-1]), _lib.JPEG_SYNC_DTYPE),
                              _d_first=views[2].view(torch.int64), _d_points=buf[p.points_at:p.total])
                if p.scans is not None:
                    k = 3 if p.first is not None else 2
                    kw.update(scans=p.scans, scan_first=p.scan_first, _d_scan_first=views[k].view(torch.int64),
                              _d_scans=views[k + 1])
                enc = EncodedImages(buf[p.files_at:p.points_at], p.headers, np.empty(p.n_tables, _lib.JPEG_TABLE_DTYPE),
                                    _d_pool=buf[:p.files_at], _d_headers=views[1], **kw)
                _, status = decode_jpeg(enc, out.select(p.accepted))
                queue_status(status, self.paths[np.asarray(sel, np.int64)[p.accepted]], dev, pending)
            check_decodes(pending, keep=1 if len(p.accepted) else 0)
            yield out
        check_decodes(pending)

    def _release(self):
        with torch.cuda.device(self.device):
            for p in self._opened:
                _lib.lib.faa_peer_close(ctypes.c_void_p(p))
            self._opened = []
            if self.multinode:
                dist.barrier(group=self.group)                   # no peer maps this rank's shard any more
            if self._own_ptr:
                self.shard = None
                _lib.lib.faa_peer_free(ctypes.c_void_p(self._own_ptr))
                self._own_ptr = 0

    def close(self):
        """free the store: collective under ``multinode``.  Every rank waits for its device, unmaps its peers' shards
        and, once no rank maps it any more, frees its own."""
        if self._own_ptr or self._opened:
            torch.cuda.synchronize(self.device)
            self._release()


class ResidentJpegDataset:
    """``JpegFileDataset`` whose files are held in device memory (``conf['faa_jpeg_resident']``): a
    ``ResidentJpegStore`` of the split, sharded over the ranks of each host under ``multinode``, so the loaders read no
    file after construction (collective under ``multinode``).  ``index``: a ``JpegIndex`` whose points the files take;
    without one each rank builds its files' scan indexes on its device.  ``progressive`` / ``progressive_index``: as
    ``JpegFileDataset``'s.  Subsets share the store; ``close`` frees it (collective under ``multinode``).
    ``device_bytes``: the bytes of this rank's shard."""

    def __init__(self, paths, targets, device="cuda", index=None, progressive=False, progressive_index=False,
                 multinode=False, group=None):
        if progressive_index and not progressive:
            raise ValueError("progressive_index needs progressive")
        self.targets = [int(t) for t in targets]
        if len(self.targets) != len(paths):
            raise ValueError("need one target per image")
        self.store = ResidentJpegStore(paths, device, index, progressive, progressive_index, multinode, group)
        self.files = np.arange(len(paths), dtype=np.int64)
        self.labels = torch.as_tensor(self.targets, dtype=torch.int64, device=self.store.device)
        self.device = self.labels.device

    @property
    def device_bytes(self):
        return self.store.device_bytes

    def __len__(self):
        return len(self.files)

    def select(self, idx):
        """the split positions of a batch"""
        return self.files[np.asarray(idx, np.int64)]

    def subset(self, idx):
        idx = [int(i) for i in idx]
        d = ResidentJpegDataset.__new__(ResidentJpegDataset)
        d.store, d.files = self.store, self.select(idx)
        d.targets = [self.targets[i] for i in idx]
        d.labels = self.labels.index_select(0, torch.as_tensor(idx, dtype=torch.int64, device=self.labels.device))
        d.device = self.device
        return d

    def close(self):
        self.store.close()


class GpuAugmentedLoader:
    """What ``get_dataloaders`` hands to ``train.py:47`` / ``search.py:101`` instead of a torch ``DataLoader``:
    an iterable of ``(data, label)`` whose ``data`` is the augmented, normalised CUDA batch (``.cuda()`` at
    train.py:49 becomes a no-op).  Batching follows ``DataLoader(dataset, batch_size, shuffle, sampler,
    drop_last)`` (reference data.py:214-224): the index stream comes from the very sampler objects the
    reference builds; the pixels of a batch are gathered on the device and go through ONE fused launch
    (policy -> RandomCrop -> HFlip -> ToTensor -> Normalize -> CutoutDefault).

    ``parity=True`` replays the reference's per-sample draws from the global ``random`` / ``numpy.random`` /
    torch generators (a ``num_workers=0`` DataLoader); the default draws on the device with Philox.
    """

    def __init__(self, dataset: DeviceDataset | RaggedDeviceDataset | EncodedDeviceDataset | JpegFileDataset, batch, policies,
                 tail: TailSpec, sampler=None, shuffle=False, drop_last=False, seed=None, parity=False, chain=None,
                 chain_mode="train"):
        """``chain``: an ``ImageNetChain`` that transforms the batches instead of the fused policy launch
        (``chain_mode`` 'train' or 'test'); a ``RaggedDeviceDataset``, ``EncodedDeviceDataset`` or ``JpegFileDataset``
        needs one.  A ``JpegFileDataset``'s batches are read from disk one batch ahead (``FileBatchStream``; the stream
        of the latest epoch is ``staging``).  When that dataset learns its index and ``sampler`` is a
        ``DistributedSampler`` under an initialised ``torch.distributed`` of more than one process, ``__iter__``
        starts every epoch with ``share_jpeg_index`` of the index, a collective, before any file is staged; ``tta``
        exchanges nothing.  A ``ResidentJpegDataset``'s batches are gathered from its store and decoded
        (``ResidentJpegStore.batches``)."""
        if not torch.cuda.is_available():
            raise _lib.FaaRuntimeError("fast_autoaugment_b200 needs a CUDA device (no CPU fallback)")
        self.dataset, self.batch_size, self.tail = dataset, int(batch), tail
        self.sampler, self.shuffle, self.drop_last, self.parity = sampler, shuffle, drop_last, parity
        self.aug = Augmentation(policies) if policies is not None else Augmentation([[("Invert", 0.0, 0.0)]])
        self.seed = int(torch.initial_seed() if seed is None else seed) & 0x7FFFFFFFFFFFFFFF
        self.chain, self.chain_mode = chain, chain_mode
        if isinstance(dataset, (RaggedDeviceDataset, EncodedDeviceDataset, JpegFileDataset, ResidentJpegDataset)) and \
                chain is None:
            raise ValueError("images of different sizes need an ImageNetChain (conf['faa_crop_resize'])")
        self._drawn = 0                   # samples drawn so far: the Philox counter never repeats across epochs
        self.staging = None

    def _n(self):
        return len(self.sampler) if self.sampler is not None else len(self.dataset)

    def __len__(self):
        n = self._n()
        return n // self.batch_size if self.drop_last else math.ceil(n / self.batch_size)

    def _indices(self):
        if self.sampler is not None:
            return list(iter(self.sampler))
        n = len(self.dataset)
        return torch.randperm(n).tolist() if self.shuffle else list(range(n))

    def _batches(self):
        """generator of (device int64 indices, source batch) over one epoch of the index stream: the gathered uint8
        images, descriptors into a ragged or encoded dataset, or a ``JpegFileDataset`` batch's files decoded on the
        device (whose decode status is checked as the epoch goes and at its end)"""
        idx_all = self._indices()
        files = None
        if isinstance(self.dataset, JpegFileDataset):
            dev = self.dataset.device
            batches = [idx_all[k * self.batch_size:(k + 1) * self.batch_size] for k in range(len(self))]
            self.staging = FileBatchStream(index=self.dataset.index, learn=self.dataset.learn,
                                           progressive=self.dataset.progressive, find=self.dataset.find,
                                           progressive_index=getattr(self.dataset, "progressive_index", False))
            files = self.staging([self.dataset.select(idx) for idx in batches], dev)
        elif isinstance(self.dataset, ResidentJpegDataset):
            dev = self.dataset.device
            batches = [idx_all[k * self.batch_size:(k + 1) * self.batch_size] for k in range(len(self))]
            files = self.dataset.store.batches([self.dataset.select(idx) for idx in batches])
        else:
            dev = self.dataset.images.device
        try:
            for k in range(len(self)):
                idx = idx_all[k * self.batch_size:(k + 1) * self.batch_size]
                t = torch.as_tensor(idx, dtype=torch.int64).to(dev, non_blocking=True)
                if files is not None:
                    raw = next(files)                            # this batch's files, decoded on the device
                elif isinstance(self.dataset, (RaggedDeviceDataset, EncodedDeviceDataset)):
                    raw = self.dataset.images.select(idx)        # descriptors into the dataset's storage: no pixel copy
                    if getattr(self.dataset, "find", False):     # decoded here, as the chain would, with found indexes
                        raw, self.chain.last_status = decode_jpeg(raw, find=True)
                else:
                    raw = self.dataset.images.index_select(0, t)
                yield t, raw
            if files is not None:
                for _ in files:                                  # the last batches' decode status
                    pass
        finally:
            if files is not None:
                files.close()

    def _shares_index(self):
        """a learning ``JpegFileDataset`` sharded by a ``DistributedSampler`` over more than one process: the ranks
        exchange what their indexes learned at the start of every epoch"""
        return isinstance(self.dataset, JpegFileDataset) and self.dataset.learn and \
            isinstance(self.sampler, DistributedSampler) and dist.is_available() and dist.is_initialized() and \
            dist.get_world_size() > 1

    def __iter__(self):
        if self._shares_index():                                 # before the staging thread reads the index
            share_jpeg_index(self.dataset.index)
        with contextlib.closing(self._batches()) as batches:
            for t, raw in batches:
                if self.chain is None:
                    data = self.aug.augment_batch(raw, self.tail, seed=self.seed, first_index=self._drawn, parity=self.parity)
                elif self.chain_mode == "test":
                    data = self.chain.test(raw)
                else:
                    data = self.chain.train(raw, parity=self.parity, seed=self.seed, first_index=self._drawn)
                self._drawn += len(t)
                yield data, self.dataset.labels.index_select(0, t)

    def tta(self, replicas, policies=None):
        """The policy search's test-time augmentation (reference search.py:87-125, ``eval_tta``) from one loader: an
        iterator over one epoch of this loader's index stream yielding ``(data[replicas, B, ...], labels[B])``, replica r
        of batch k being what this loader's own ``__iter__`` would yield for it with the Philox keys of
        ``first_index = drawn + r * B`` (``drawn``: samples drawn before the batch).  Each batch is gathered, read or
        decoded once; the replicas come from ``augment_tta`` (no chain) or ``ImageNetChain.train_tta``.  The batch
        draws replicas * B keys, so no key repeats within or across batches or epochs, unlike replicas separate loaders
        built with one seed.  Raises ValueError for parity draws, a test-chain loader and what ``check_tta`` refuses.

        ``policies``: T candidate policies (what ``compile_policies`` takes: archive lists, ``CompiledPolicy``) scored in
        place of the loader's own.  Each batch then yields ``(data[T, replicas, B, ...], labels[B])`` from one read or
        decode, candidate t's block being what ``tta(replicas)`` of a loader with policy t would yield with the keys of
        ``first_index = drawn + t * replicas * B`` (``augment_tta_policies`` or ``ImageNetChain.train_tta_policies``),
        and ``drawn`` advances by T * replicas * B.  It also raises ValueError for what ``check_tta_policies``
        refuses."""
        if self.parity:
            raise ValueError("tta draws with Philox only: K reference loaders have no single parity draw order")
        if self.chain is not None and self.chain_mode != "train":
            raise ValueError("tta replicates the train chain: a %r chain loader draws nothing" % self.chain_mode)
        n = min(self.batch_size, self._n())
        if policies is not None:
            pols = compile_policies(policies)
            check_tta_policies(pols, n, replicas)
            return self._tta(int(replicas), pols)
        if self.chain is not None:
            self.chain.check_tta(n, replicas)
        else:
            check_tta(n, replicas)
            if self.aug.compiled.n_op > _lib.MAX_FUSED_OPS:
                raise ValueError("tta supports policies of at most %d ops per sub-policy (replicated launches)"
                                 % _lib.MAX_FUSED_OPS)
        return self._tta(int(replicas))

    def _tta(self, K, pols=None):
        with contextlib.closing(self._batches()) as batches:
            for t, raw in batches:
                if pols is not None and self.chain is None:
                    data = augment_tta_policies(pols, raw, self.tail, K, self.seed, self._drawn)
                elif pols is not None:
                    data = self.chain.train_tta_policies(raw, pols, K, seed=self.seed, first_index=self._drawn)
                elif self.chain is None:
                    data = augment_tta(self.aug.compiled, raw, self.tail, K, self.seed, self._drawn)
                else:
                    data = self.chain.train_tta(raw, K, seed=self.seed, first_index=self._drawn)
                self._drawn += (len(pols) if pols is not None else 1) * K * len(t)
                yield data, self.dataset.labels.index_select(0, t)


# ---------------------------------------------------------------------------------------------------
def _load_arrays(dataset, dataroot):
    """(train images, train targets, test images, test targets) as uint8 / int arrays.

    ``dataroot`` is the reference's dataset directory (torchvision layout, read with ``download=False`` - the
    build and GPU boxes have no network), or a directory holding ``<dataset>_train.npz`` / ``<dataset>_test.npz``
    (arrays ``data`` [N,H,W,3] uint8 and ``targets``), or - for in-memory injection (tests, synthetic benchmarks) -
    a mapping ``{"train": (images, targets), "test": (images, targets)}``.

    ImageNet sources may differ in size: a mapping whose images are a list of uint8 HWC arrays of different sizes, or
    an .npz whose ``data`` is the images' bytes packed back to back with their ``sizes`` [N, 2] (h, w).  Those images
    come back as a list of arrays.  ImageNet sources may also be JPEG files: a mapping whose images are a list of
    ``bytes``, or an .npz with ``jpeg`` (the files packed back to back), ``lengths`` and ``targets``; they come back as a
    list of ``bytes``, decoded on the device batch by batch.  Without a mapping or .npz, ``imagenet`` reads the
    reference's directory (``imagenet_index``: ``dataroot/imagenet-pytorch/{train,val}``): its images come back as
    ``FilePaths``, read from disk batch by batch."""
    base = dataset.replace("reduced_", "")
    ragged_ok = "imagenet" in dataset

    def images(x):
        if ragged_ok and isinstance(x, (list, tuple)) and len(x) and all(isinstance(a, (bytes, bytearray)) for a in x):
            return [bytes(a) for a in x]
        if ragged_ok and isinstance(x, (list, tuple)) and len({np.shape(a) for a in x}) > 1:
            return [np.asarray(a) for a in x]
        return np.asarray(x)

    def npz_images(z):
        if ragged_ok and "jpeg" in z.files:
            lengths = np.asarray(z["lengths"], np.int64).reshape(-1)
            flat = np.asarray(z["jpeg"], np.uint8).reshape(-1)
            if int(lengths.sum()) != flat.size:
                raise ValueError("packed jpeg bytes do not match lengths")
            ends = np.cumsum(lengths)
            return [flat[e - n:e].tobytes() for e, n in zip(ends, lengths)]
        if ragged_ok and "sizes" in z.files:
            sizes = np.asarray(z["sizes"], np.int64).reshape(-1, 2)
            ends = np.cumsum(sizes[:, 0] * sizes[:, 1] * 3)
            flat = np.asarray(z["data"], np.uint8).reshape(-1)
            if len(ends) and ends[-1] != flat.size:
                raise ValueError("packed data does not match sizes")
            return [p.reshape(h, w, 3) for p, (h, w) in zip(np.split(flat, ends[:-1]), sizes)]
        return z["data"]
    if isinstance(dataroot, dict):
        tr, te = dataroot["train"], dataroot.get("test", dataroot["train"])
        return images(tr[0]), list(tr[1]), images(te[0]), list(te[1])
    npz = [os.path.join(str(dataroot), "%s_%s.npz" % (base, s)) for s in ("train", "test")]
    if all(os.path.exists(p) for p in npz):
        a, b = np.load(npz[0]), np.load(npz[1])
        return npz_images(a), list(a["targets"]), npz_images(b), list(b["targets"])
    import torchvision
    if base in ("cifar10", "cifar100"):
        cls = torchvision.datasets.CIFAR10 if base == "cifar10" else torchvision.datasets.CIFAR100
        tr, te = cls(root=dataroot, train=True, download=False), cls(root=dataroot, train=False, download=False)
        return tr.data, list(tr.targets), te.data, list(te.targets)
    if base == "svhn":
        def hwc(d):
            return np.ascontiguousarray(np.transpose(d.data, (0, 2, 3, 1)))
        tr = torchvision.datasets.SVHN(root=dataroot, split="train", download=False)
        te = torchvision.datasets.SVHN(root=dataroot, split="test", download=False)
        if dataset == "svhn":                                   # data.py:132-135: train + extra
            ex = torchvision.datasets.SVHN(root=dataroot, split="extra", download=False)
            return (np.concatenate([hwc(tr), hwc(ex)]), list(tr.labels) + list(ex.labels), hwc(te), list(te.labels))
        return hwc(tr), list(tr.labels), hwc(te), list(te.labels)
    if dataset == "imagenet":                                   # data.py:146-150
        out = []
        for split in ("train", "val"):
            samples = imagenet_index(dataroot, split)
            paths = FilePaths(p for p, _ in samples)
            paths.split, paths.folder = split, imagenet_split_folder(dataroot, split)
            out += [paths, [t for _, t in samples]]
        return tuple(out)
    raise ValueError("invalid dataset name=%s" % dataset)


def imagenet_split_folder(dataroot, split):
    """``dataroot/imagenet-pytorch/<split>``: the folder ``imagenet_index``'s paths lie in"""
    return os.path.join(os.path.expanduser(os.path.join(str(dataroot), "imagenet-pytorch")), split)


def imagenet_index(dataroot, split):
    """[(path, class index)] of the reference's ``ImageNet(os.path.join(dataroot, 'imagenet-pytorch'), split)``
    (data.py:146-150, imagenet.py:52-90), in its order.  ``train`` with ``imagenet-pytorch/train_cls.txt``: the
    file's non-empty lines in order, classes the sorted first path components, path ``train/<line>.JPEG``.  Otherwise
    torchvision's own ``find_classes`` / ``make_dataset`` over the split folder, as ``ImageFolder`` walks it.  The
    class names of ``meta.bin`` are not needed for the targets and are not read."""
    root = os.path.expanduser(os.path.join(str(dataroot), "imagenet-pytorch"))
    folder = os.path.join(root, split)
    listfile = os.path.join(root, "train_cls.txt")
    if split == "train" and os.path.exists(listfile):
        with open(listfile, "r") as f:
            lines = [line.strip().split(" ")[0] for line in f.readlines() if line.strip()]
        classes = sorted(set(line.split("/")[0] for line in lines))
        to_idx = {c: i for i, c in enumerate(classes)}
        return [(os.path.join(folder, line + ".JPEG"), to_idx[line.split("/")[0]]) for line in lines]
    if not os.path.isdir(folder):
        raise FileNotFoundError("ImageNet %s folder not found: %s (the reference's layout is "
                                "<dataroot>/imagenet-pytorch/{train,val}/<class>/...)" % (split, folder))
    from torchvision.datasets.folder import IMG_EXTENSIONS, find_classes, make_dataset
    return make_dataset(folder, find_classes(folder)[1], IMG_EXTENSIONS)


def split_samplers(targets, split=0.15, split_idx=0, multinode=False, target_lb=-1):
    """(train sampler or None, valid sampler) of ``get_dataloaders`` over a train set with these targets
    (reference data.py:189-212)"""
    from sklearn.model_selection import StratifiedShuffleSplit
    import torch.distributed as dist

    train_sampler = None
    if split > 0.0:                                             # data.py:189-203
        sss = StratifiedShuffleSplit(n_splits=5, test_size=split, random_state=0)
        sss = sss.split(list(range(len(targets))), targets)
        for _ in range(split_idx + 1):
            train_idx, valid_idx = next(sss)
        if target_lb >= 0:
            train_idx = [i for i in train_idx if targets[i] == target_lb]
            valid_idx = [i for i in valid_idx if targets[i] == target_lb]
        train_sampler = SubsetRandomSampler(train_idx)
        valid_sampler = SubsetSampler(valid_idx)
        if multinode:
            train_sampler = torch.utils.data.distributed.DistributedSampler(
                torch.utils.data.Subset(range(len(targets)), train_idx),
                num_replicas=dist.get_world_size(), rank=dist.get_rank())
    else:
        valid_sampler = SubsetSampler([])
        if multinode:
            train_sampler = torch.utils.data.distributed.DistributedSampler(
                range(len(targets)), num_replicas=dist.get_world_size(), rank=dist.get_rank())
    return train_sampler, valid_sampler


def get_dataloaders(dataset, batch, dataroot, split=0.15, split_idx=0, multinode=False, target_lb=-1):
    """Drop-in for reference ``get_dataloaders`` (data.py:37-225): same signature, same conf keys
    (``C.get()['aug']``, ``['cutout']``), same stratified splits and sampler objects, same return tuple
    ``(train_sampler, trainloader, validloader, testloader)`` - but the three loaders are
    ``GpuAugmentedLoader`` s over device-resident uint8 datasets, so the per-sample PIL chain of the reference's
    DataLoader workers is replaced by one fused kernel launch per batch.

    Extra conf keys (optional): ``faa_out_dtype`` ('float32' default - what the reference yields -, 'float16',
    'bfloat16'), ``faa_parity`` (replay the reference's global RNG draws per sample; tests), ``faa_crop_resize``
    (ImageNet: the stored images are uncropped sources, of one size or of many, and the loaders run the reference's full chains,
    ``ImageNetChain``: train / valid = policy -> EfficientNetRandomCrop + bicubic Resize -> ColorJitter -> HFlip +
    Lighting + Normalize, test = EfficientNetCenterCrop + Resize + Normalize, at 224 or the EfficientNet size of
    ``conf['model']['type']``; without it ImageNet images must already have the network's size).

    ``imagenet`` with the reference's ``dataroot`` (``imagenet-pytorch/{train,val}``, ``imagenet_index``) keeps the
    files on disk (``JpegFileDataset``): the loaders read, stage and decode each batch's files one batch ahead.
    ``faa_jpeg_index``: a directory holding ``train.npz`` / ``val.npz`` written by ``python -m
    fast_autoaugment_b200.jpeg_index DATAROOT DIR``; the files they index are decoded on many threads each, with the
    same pixels.  ``faa_jpeg_index_learn``: the datasets start from that index, or from an empty one, and the loaders
    enter the scan index of every file they decode serially, so from the second epoch on the files the loaders have
    seen are decoded on many threads, with the same pixels; the train and valid loaders share what they learn
    (``trainloader.dataset.index.save(path)`` writes it as ``faa_jpeg_index`` reads it).  With ``multinode=True``
    the train loader's ranks exchange what they learned at the start of every epoch (``share_jpeg_index``), so each
    rank's index lists what any rank learned.  It costs host memory: 16 bytes a point, about 1.7 KB a file at
    ImageNet's mean file size.  ``faa_jpeg_progressive`` (default False): the
    train, valid, test and ``tta`` loaders decode progressive JPEG files on the device, bit-exact with Pillow, instead of
    with Pillow on the host; files whose progression is incomplete still go to Pillow.  They get no scan index.
    ``faa_jpeg_index_find`` (default False): the loaders find, on the device and in parallel, the scan index of every
    restart-free file that has none (``decode_jpeg(find=True)``), so even the first epoch and files no index lists
    decode on many threads, with the same pixels; with ``faa_jpeg_index_learn`` the index learns the found points, and
    the first epoch pays no serial decode.  A find that does not converge within its rounds still splits the file at
    the points it verified (DESIGN §4.8).  ``faa_jpeg_progressive_index`` (default False; needs
    ``faa_jpeg_progressive``): progressive files take a scan index too, so with ``faa_jpeg_index`` or
    ``faa_jpeg_index_learn`` their restart-free scans decode on many threads from points looked up or learned like any
    other file's, with the same pixels (``python -m fast_autoaugment_b200.jpeg_index --progressive`` writes them).
    ``faa_jpeg_resident`` (default False): the directory's splits are read, parsed and uploaded once, here, and held in
    device memory (``ResidentJpegDataset``; with ``multinode=True`` a collective, the ranks of each host sharing each
    split), so the loaders read no file; every file's scan index comes from ``faa_jpeg_index`` or is built on the device
    here, and ``faa_jpeg_index_learn`` / ``faa_jpeg_index_find`` are refused.  ``dataset.device_bytes`` is what a
    rank's shard takes, ``dataset.close()`` frees it."""
    from sklearn.model_selection import StratifiedShuffleSplit

    conf = C.get()
    out_dtype = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}[
        str(conf.get("faa_out_dtype", "float32"))]
    cutout = int(conf.get("cutout", 0) or 0)
    if "cifar" in dataset or "svhn" in dataset:                 # data.py:38-48
        tail = TailSpec((32, 32), 4, True, CIFAR_MEAN, CIFAR_STD, cutout, out_dtype)
        test_tail = TailSpec(None, 0, False, CIFAR_MEAN, CIFAR_STD, 0, out_dtype)
    elif "imagenet" in dataset:                                 # data.py:49-80 on already-sized images (SURVEY.md 3-D)
        tail = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, cutout, out_dtype)
        test_tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, out_dtype)
    else:
        raise ValueError("dataset=%s" % dataset)
    policies = policy_by_conf_name(conf["aug"])                 # data.py:85-109 (ValueError on an unknown name)

    tr_x, tr_y, te_x, te_y = _load_arrays(dataset, dataroot)
    ragged = isinstance(tr_x, list) or isinstance(te_x, list)
    if ragged and not conf.get("faa_crop_resize", False):
        raise ValueError("ImageNet images of different sizes (or JPEG files) need conf['faa_crop_resize']: without it the "
                         "images are augmented at one fixed size")

    index_dir = conf.get("faa_jpeg_index")
    learn = bool(conf.get("faa_jpeg_index_learn", False))
    progressive = bool(conf.get("faa_jpeg_progressive", False))
    find = bool(conf.get("faa_jpeg_index_find", False))
    progressive_index = bool(conf.get("faa_jpeg_progressive_index", False))
    if progressive_index and not progressive:
        raise ValueError("conf['faa_jpeg_progressive_index'] needs conf['faa_jpeg_progressive']")
    resident = bool(conf.get("faa_jpeg_resident", False))
    if resident and (learn or find):
        raise ValueError("conf['faa_jpeg_resident'] builds every file's scan index on the device when the store is made: "
                         "conf['faa_jpeg_index_learn'] and conf['faa_jpeg_index_find'] have nothing left to do")

    def saved_index(x):
        if not index_dir:
            return None
        path = os.path.join(os.fspath(index_dir), "%s.npz" % x.split)
        if not os.path.exists(path):
            raise FileNotFoundError("conf['faa_jpeg_index']: no index of the %s split at %s (write it with "
                                    "python -m fast_autoaugment_b200.jpeg_index)" % (x.split, path))
        return JpegIndex.load(path, x.folder)

    def device_dataset(x, y):
        if isinstance(x, FilePaths) and resident:
            return ResidentJpegDataset(x, y, index=saved_index(x), progressive=progressive,
                                       progressive_index=progressive_index, multinode=multinode)
        if isinstance(x, FilePaths):
            index = saved_index(x)
            if learn and index is None:
                index = JpegIndex.empty(x.folder)
            return JpegFileDataset(x, y, index=index, learn=learn, progressive=progressive, find=find,
                                   progressive_index=progressive_index)
        if isinstance(x, list) and len(x) and isinstance(x[0], bytes):
            return EncodedDeviceDataset(x, y, progressive=progressive, find=find, progressive_index=progressive_index)
        return RaggedDeviceDataset(x, y) if isinstance(x, list) else DeviceDataset(x, y)
    if dataset in ("cifar10", "cifar100", "svhn", "imagenet"):
        total_trainset, testset = device_dataset(tr_x, tr_y), device_dataset(te_x, te_y)
    elif dataset in ("reduced_cifar10", "reduced_svhn"):        # data.py:117-126, 136-146
        test_size = 46000 if dataset == "reduced_cifar10" else 73257 - 1000
        sss = StratifiedShuffleSplit(n_splits=1, test_size=test_size, random_state=0)
        train_idx, _ = next(sss.split(list(range(len(tr_y))), tr_y))
        total_trainset, testset = DeviceDataset(tr_x, tr_y).subset(train_idx), DeviceDataset(te_x, te_y)
    else:
        raise ValueError("invalid dataset name=%s" % dataset)

    train_sampler, valid_sampler = split_samplers(total_trainset.targets, split, split_idx, multinode, target_lb)
    parity = bool(conf.get("faa_parity", False))
    if "imagenet" in dataset and conf.get("faa_crop_resize", False):      # data.py:49-80, 217-224
        model_type = (conf.get("model") or {}).get("type", "")
        chain = ImageNetChain(policies, imagenet_input_size(model_type), out_dtype)
        trainloader = GpuAugmentedLoader(total_trainset, batch, policies, tail, sampler=train_sampler,
                                         shuffle=train_sampler is None, drop_last=True, parity=parity, chain=chain)
        validloader = GpuAugmentedLoader(total_trainset, batch, policies, tail, sampler=valid_sampler,
                                         shuffle=False, drop_last=False, parity=parity, chain=chain)
        testloader = GpuAugmentedLoader(testset, batch, None, test_tail, shuffle=False, drop_last=False,
                                        chain=chain, chain_mode="test")
        return train_sampler, trainloader, validloader, testloader
    trainloader = GpuAugmentedLoader(total_trainset, batch, policies, tail, sampler=train_sampler,
                                     shuffle=train_sampler is None, drop_last=True, parity=parity)       # data.py:214-216
    validloader = GpuAugmentedLoader(total_trainset, batch, policies, tail, sampler=valid_sampler,
                                     shuffle=False, drop_last=False, parity=parity)                      # data.py:217-219
    testloader = GpuAugmentedLoader(testset, batch, None, test_tail, shuffle=False, drop_last=False)     # data.py:221-224
    return train_sampler, trainloader, validloader, testloader
