#!/usr/bin/env python
"""Generate tests/golden/golden_resize.npz from the LIVE reference (the ImageNet chains' geometry).

    python tests/golden/make_golden_resize.py <checkout of kakaobrain/fast-autoaugment>

Imports the reference read-only like make_golden.py and writes only golden_resize.npz:

* ``boxes_<s>_<H>x<W>``: int32 [N][4] (x0, y0, w, h) that the reference's ``EfficientNetRandomCrop(s)`` cuts for
  ``random.seed(i)``, i < N.  The crop is read without patching the reference: the input's pixels encode their own
  (x, y), so the output's first pixel and its size give the box.
* ``test_<H>x<W>`` / ``train_<H>x<W>`` (+ ``in_<H>x<W>``, digests of the inputs ``chain_input`` regenerates): per-image sha256 digests (first 16 hex digits) of the fp32 output of
  the reference ``transform_test`` and ``transform_train`` with ``fa_resnet50_rimagenet`` (data.py:60-80, 94-95) on
  seeded inputs, under ``random.seed / np.random.seed / torch.manual_seed(3)``, one image after another.
* ``test_s<s>_<H>x<W>`` / ``train_s<s>_<H>x<W>`` (+ ``in_s<s>_<H>x<W>``): the same digests for the EfficientNet input
  sizes ``EFFNET_CHAIN_CASES`` (data.py:53-55): ``EfficientNetRandomCrop(s)`` / ``EfficientNetCenterCrop(s)`` and
  ``Resize((s, s))``, inputs from ``np.random.default_rng(s)``.

Environment that produced the committed file: Pillow 12.2.0, numpy 2.3.5, torch 2.11.0, torchvision 0.26.0.
"""
import hashlib
import os
import random
import sys

import numpy as np
import PIL.Image
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
BOX_CASES = ((224, 375, 500), (224, 256, 256), (224, 333, 500), (380, 500, 375), (224, 48, 64), (224, 1536, 2048),
             (224, 3, 4), (224, 2, 2))        # (tiny images: whole-image and failed-attempt fallbacks)
N_BOXES = 200
CHAIN_CASES = ((256, 256, 64), (375, 500, 32))
EFFNET_CHAIN_CASES = ((380, 375, 500, 8), (600, 375, 500, 8))      # (s, H, W, N)


def coord_image(h, w):
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([x & 255, y & 255, (x >> 8) | ((y >> 8) << 4)], -1).astype(np.uint8)


def chain_input(rng, i, h, w):
    """noise (odd i) or a ramp + noise (even i)"""
    if i % 2:
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return np.clip(np.linspace(30, 220, w)[None, :, None] + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)


def digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def effnet_chain_inputs(s, h, w, n):
    rng = np.random.default_rng(s)
    return np.stack([chain_input(rng, i, h, w) for i in range(n)])


def reference_transforms(aug, archive, data, s):
    """the reference's transform_train / transform_test at input size s, as data.py:60-80 and 94-95 build them"""
    from torchvision.transforms import transforms as T
    norm = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    train = T.Compose([
        data.EfficientNetRandomCrop(s), T.Resize((s, s), interpolation=PIL.Image.BICUBIC), T.RandomHorizontalFlip(),
        T.ColorJitter(brightness=0.4, contrast=0.4, saturation=0.4), T.ToTensor(),
        aug.Lighting(0.1, data._IMAGENET_PCA["eigval"], data._IMAGENET_PCA["eigvec"]), norm])
    train.transforms.insert(0, data.Augmentation(archive.fa_resnet50_rimagenet()))
    test = T.Compose([data.EfficientNetCenterCrop(s), T.Resize((s, s), interpolation=PIL.Image.BICUBIC), T.ToTensor(), norm])
    return {"train": train, "test": test}


def chain_digests(tf, batch):
    """digests of tf on each image, under the seeds of the committed digests, one image after another"""
    random.seed(3)
    np.random.seed(3)
    torch.manual_seed(3)
    return np.array([digest(tf(PIL.Image.fromarray(a)).numpy()) for a in batch])


def main(ref):
    sys.path.insert(0, HERE)
    from make_golden import import_reference
    aug, archive, _, data = import_reference(ref)
    from torchvision.transforms import transforms as T
    out = {}
    for s, h, w in BOX_CASES:
        img = PIL.Image.fromarray(coord_image(h, w))
        crop = data.EfficientNetRandomCrop(s)
        boxes = []
        for i in range(N_BOXES):
            random.seed(i)
            c = np.asarray(crop(img))
            x0 = int(c[0, 0, 0]) | ((int(c[0, 0, 2]) & 15) << 8)
            y0 = int(c[0, 0, 1]) | ((int(c[0, 0, 2]) >> 4) << 8)
            boxes.append((x0, y0, c.shape[1], c.shape[0]))
        out["boxes_%d_%dx%d" % (s, h, w)] = np.array(boxes, np.int32)
    norm = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    transform_test = T.Compose([data.EfficientNetCenterCrop(224), T.Resize((224, 224), interpolation=PIL.Image.BICUBIC),
                                T.ToTensor(), norm])
    transform_train = T.Compose([
        data.Augmentation(archive.fa_resnet50_rimagenet()),
        data.EfficientNetRandomCrop(224), T.Resize((224, 224), interpolation=PIL.Image.BICUBIC),
        T.RandomHorizontalFlip(), T.ColorJitter(brightness=0.4, contrast=0.4, saturation=0.4), T.ToTensor(),
        aug.Lighting(0.1, data._IMAGENET_PCA["eigval"], data._IMAGENET_PCA["eigvec"]), norm])
    rng = np.random.default_rng(2024)
    for h, w, n in CHAIN_CASES:
        tag = "%dx%d" % (h, w)
        batch = np.stack([chain_input(rng, i, h, w) for i in range(n)])
        out["in_" + tag] = np.array([digest(a) for a in batch])     # the inputs are regenerated from the seed
        for name, tf in (("test", transform_test), ("train", transform_train)):
            random.seed(3)
            np.random.seed(3)
            torch.manual_seed(3)
            out["%s_%s" % (name, tag)] = np.array([digest(tf(PIL.Image.fromarray(a)).numpy()) for a in batch])
    for s, h, w, n in EFFNET_CHAIN_CASES:
        tag = "s%d_%dx%d" % (s, h, w)
        batch = effnet_chain_inputs(s, h, w, n)
        out["in_" + tag] = np.array([digest(a) for a in batch])
        for name, tf in reference_transforms(aug, archive, data, s).items():
            out["%s_%s" % (name, tag)] = chain_digests(tf, batch)
    np.savez_compressed(os.path.join(HERE, "golden_resize.npz"), **out)
    print("wrote golden_resize.npz:", os.path.getsize(os.path.join(HERE, "golden_resize.npz")), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
