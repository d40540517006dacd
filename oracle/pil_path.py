"""Oracle layer 1: the reference's call sequence into Pillow / torchvision.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Every function restates one piece of the reference and cites it.  The
per-pixel arithmetic is *not* here - it is inside Pillow's C library, exactly as
for the reference - so this layer has the reference's CPU cost profile and is
what ``bench.py`` times as ``cpu_baseline`` (kind "port").  The RNG streams that
are consumed (Python ``random``, ``numpy.random`` legacy global state, torch's
CPU generator) and the order of the draws are the reference's.
"""
from __future__ import annotations

import random

import numpy as np
import PIL.Image
import PIL.ImageDraw
import PIL.ImageEnhance
import PIL.ImageOps
import torch

# --------------------------------------------------------------------------
# magnitude ranges: FastAutoAugment/augmentations.py:156-182 (augment_list)
# kind: 'mirror'  -> one random.random() draw, negate v if > 0.5
#                    (augmentations.py:15,22,29,37,59 with random_mirror=True :10,
#                     and unconditionally for the *Abs translates :45,52)
# --------------------------------------------------------------------------
RANGES = {
    "ShearX": (-0.3, 0.3), "ShearY": (-0.3, 0.3),
    "TranslateX": (-0.45, 0.45), "TranslateY": (-0.45, 0.45),
    "Rotate": (-30, 30),
    "AutoContrast": (0, 1), "Invert": (0, 1), "Equalize": (0, 1),
    "Solarize": (0, 256), "Posterize": (4, 8),
    "Contrast": (0.1, 1.9), "Color": (0.1, 1.9), "Brightness": (0.1, 1.9),
    "Sharpness": (0.1, 1.9),
    "Cutout": (0, 0.2),
    # the four AutoAugment-compat ops, augmentations.py:175-181
    "CutoutAbs": (0, 20), "Posterize2": (0, 4),
    "TranslateXAbs": (0, 10), "TranslateYAbs": (0, 10),
}
# asserted magnitude windows (augmentations.py:14,21,28,36,44,51,58,81,86,92,98,103,108,113,118);
# CutoutAbs' assert is commented out in the reference (:127).
ASSERT_WINDOW = dict(RANGES)
ASSERT_WINDOW["Solarize"] = (0, 256)
ASSERT_WINDOW["Cutout"] = (0.0, 0.2)
del ASSERT_WINDOW["CutoutAbs"]
for _n in ("AutoContrast", "Invert", "Equalize"):
    del ASSERT_WINDOW[_n]

CUTOUT_RGB = (125, 123, 114)          # augmentations.py:140


def magnitude(name: str, level: float) -> float:
    """``apply_augment``'s level -> magnitude map, augmentations.py:192-194."""
    low, high = RANGES[name]          # KeyError on unknown op, like augmentations.py:189
    return level * (high - low) + low


def _mirror_draw(v):
    return -v if random.random() > 0.5 else v


def _affine(img, coeffs):
    # no ``resample`` argument in the reference => Pillow's default, NEAREST
    return img.transform(img.size, PIL.Image.AFFINE, coeffs)


def _cutout_abs(img, v):
    """augmentations.py:126-144 (``np.random.uniform(w)`` is uniform(low=w, high=1.0))."""
    if v < 0:
        return img
    w, h = img.size
    cx = np.random.uniform(w)
    cy = np.random.uniform(h)
    left = int(max(0, cx - v / 2.0))
    top = int(max(0, cy - v / 2.0))
    right = min(w, left + v)
    bottom = min(h, top + v)
    out = img.copy()
    PIL.ImageDraw.Draw(out).rectangle((left, top, right, bottom), CUTOUT_RGB)
    return out


def run_op(img: PIL.Image.Image, name: str, v: float) -> PIL.Image.Image:
    """One op at magnitude ``v``: augmentations.py:13-144."""
    if name in ASSERT_WINDOW:
        lo, hi = ASSERT_WINDOW[name]
        assert lo <= v <= hi
    if name == "ShearX":                                   # :13-17
        v = _mirror_draw(v)
        return _affine(img, (1, v, 0, 0, 1, 0))
    if name == "ShearY":                                   # :20-24
        v = _mirror_draw(v)
        return _affine(img, (1, 0, 0, v, 1, 0))
    if name == "TranslateX":                               # :27-32
        v = _mirror_draw(v)
        return _affine(img, (1, 0, v * img.size[0], 0, 1, 0))
    if name == "TranslateY":                               # :35-40
        v = _mirror_draw(v)
        return _affine(img, (1, 0, 0, 0, 1, v * img.size[1]))
    if name == "TranslateXAbs":                            # :43-47
        return _affine(img, (1, 0, _mirror_draw(v), 0, 1, 0))
    if name == "TranslateYAbs":                            # :50-54
        return _affine(img, (1, 0, 0, 0, 1, _mirror_draw(v)))
    if name == "Rotate":                                   # :57-61
        return img.rotate(_mirror_draw(v))
    if name == "AutoContrast":                             # :64-65
        return PIL.ImageOps.autocontrast(img)
    if name == "Invert":                                   # :68-69
        return PIL.ImageOps.invert(img)
    if name == "Equalize":                                 # :72-73
        return PIL.ImageOps.equalize(img)
    if name == "Solarize":                                 # :80-82
        return PIL.ImageOps.solarize(img, v)
    if name in ("Posterize", "Posterize2"):                # :85-94
        return PIL.ImageOps.posterize(img, int(v))
    if name == "Contrast":                                 # :97-99
        return PIL.ImageEnhance.Contrast(img).enhance(v)
    if name == "Color":                                    # :102-104
        return PIL.ImageEnhance.Color(img).enhance(v)
    if name == "Brightness":                               # :107-109
        return PIL.ImageEnhance.Brightness(img).enhance(v)
    if name == "Sharpness":                                # :112-114
        return PIL.ImageEnhance.Sharpness(img).enhance(v)
    if name == "Cutout":                                   # :117-123
        if v <= 0.0:
            return img
        return _cutout_abs(img, v * img.size[0])
    if name == "CutoutAbs":
        return _cutout_abs(img, v)
    raise KeyError(name)


def apply_op(img: PIL.Image.Image, name: str, level: float) -> PIL.Image.Image:
    """``apply_augment``: copy, map level, dispatch (augmentations.py:192-194)."""
    return run_op(img.copy(), name, magnitude(name, level))


class PolicyTransform:
    """``Augmentation`` of data.py:253-264: one sub-policy per image, each op
    gated by ``random.random() > pr`` *before* any op-internal draw."""

    def __init__(self, policies):
        self.policies = policies

    def __call__(self, img):
        chosen = random.choice(self.policies)
        for name, pr, level in chosen:
            if random.random() > pr:
                continue
            img = apply_op(img, name, level)
        return img


class ZeroBoxCutout:
    """``CutoutDefault`` of data.py:228-250 (DARTS cutout on the normalised CHW
    tensor; y drawn before x; half-open clipped box; in place)."""

    def __init__(self, length):
        self.length = length

    def __call__(self, t):
        h, w = t.size(1), t.size(2)
        keep = np.ones((h, w), np.float32)
        cy = np.random.randint(h)
        cx = np.random.randint(w)
        half = self.length // 2
        ya, yb = np.clip(cy - half, 0, h), np.clip(cy + half, 0, h)
        xa, xb = np.clip(cx - half, 0, w), np.clip(cx + half, 0, w)
        keep[ya:yb, xa:xb] = 0.0
        t *= torch.from_numpy(keep).expand_as(t)
        return t


CIFAR_MEAN, CIFAR_STD = (0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010)     # data.py:34
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)      # data.py:72


def cifar_train_chain(policies, cutout_length=16):
    """``transform_train`` for cifar/svhn: data.py:39-44, policy inserted at
    index 0 (:85-105), CutoutDefault appended (:111-112)."""
    from torchvision.transforms import transforms as T
    steps = [T.RandomCrop(32, padding=4), T.RandomHorizontalFlip(), T.ToTensor(),
             T.Normalize(CIFAR_MEAN, CIFAR_STD)]
    if policies is not None:
        steps.insert(0, PolicyTransform(policies))
    if cutout_length > 0:
        steps.append(ZeroBoxCutout(cutout_length))
    return T.Compose(steps)


def fixed_shape_chain(policies, mean, std, hflip=True, cutout_length=0):
    """The fixed-shape (already cropped/resized) chain of SURVEY.md 8(d)
    configs 3-5: policy -> HFlip (data.py:64) -> ToTensor -> Normalize
    (data.py:70-72) [-> CutoutDefault (data.py:111-112)]."""
    from torchvision.transforms import transforms as T
    steps = []
    if policies is not None:
        steps.append(PolicyTransform(policies))
    if hflip:
        steps.append(T.RandomHorizontalFlip())
    steps += [T.ToTensor(), T.Normalize(mean, std)]
    if cutout_length > 0:
        steps.append(ZeroBoxCutout(cutout_length))
    return T.Compose(steps)


def mixup_pairs(data, targets, alpha):
    """``mixup`` of aug_mixup.py:13-23: randperm (torch CPU generator) first,
    then one Beta(alpha, alpha) draw from numpy's global state."""
    order = torch.randperm(data.size(0))
    partner = data[order]
    partner_targets = targets[order]
    lam = np.random.beta(alpha, alpha)
    lam = max(lam, 1.0 - lam)
    assert 0.0 <= lam <= 1.0, lam
    return data * lam + partner * (1 - lam), targets, partner_targets, lam


def run_chain_on_batch(chain, batch_u8_nhwc: np.ndarray) -> torch.Tensor:
    """Apply ``chain`` image by image in index order (== a num_workers=0
    DataLoader, SURVEY.md 8d) and stack like default_collate."""
    outs = [chain(PIL.Image.fromarray(a)) for a in batch_u8_nhwc]
    return torch.stack(outs, 0)


def seed_all(s: int):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
