"""fast_autoaugment_b200 - H100-native (sm_90a CUDA) implementation of Fast AutoAugment's
per-batch augmentation hot path, behind the reference's own Python surface.

Reference (kakaobrain/fast-autoaugment) module  ->  this package
    FastAutoAugment/archive.py        ->  archive        (policy lists, same functions)
    FastAutoAugment/augmentations.py  ->  augmentations  (apply_augment, augment_list, get_augment)
    FastAutoAugment/data.py           ->  data           (Augmentation, CutoutDefault, loaders)
    FastAutoAugment/aug_mixup.py      ->  aug_mixup      (mixup)

The pixel path exists only as CUDA kernels in ``libfaa_b200.so`` (C ABI:
``include/faa_b200.h``); importing this package without that library raises ImportError,
and calling it without a CUDA device raises - there is no CPU fallback.
"""
from . import _lib                      # noqa: F401  (fails loudly if the CUDA library is missing)
from . import archive                   # noqa: F401
from .engine import (CompiledPolicy, FusedAugmenter, TailSpec, augment_batch, augment_tta, make_rng,   # noqa: F401
                     CIFAR_MEAN, CIFAR_STD, IMAGENET_MEAN, IMAGENET_STD)
from .data import (Augmentation, ColorJitter, CutoutDefault, GpuAugmentedLoader, Lighting,   # noqa: F401
                   get_dataloaders)
from .aug_mixup import mixup                                                      # noqa: F401

__version__ = "0.1.0"
