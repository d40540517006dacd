#!/usr/bin/env python
"""Generate tests/golden/golden_ragged.npz from the LIVE reference: the ImageNet chains on a list of differently sized
images.

    python tests/golden/make_golden_ragged.py <checkout of kakaobrain/fast-autoaugment>

The reference transforms one PIL image at a time, whatever its size.  ``ragged_inputs`` regenerates a list of
``SIZES`` images from ``np.random.default_rng(SEED)`` (``chain_input`` of make_golden_resize.py); 3 x 4 exercises the
crop's center-crop fallback.  Keys, per input size s in ``INPUT_SIZES``:

* ``in``: sha256 digests (first 16 hex digits) of the inputs;
* ``train_s<s>`` / ``test_s<s>``: digests of the fp32 output of the reference ``transform_train`` (with
  ``fa_resnet50_rimagenet``) and ``transform_test`` at input size s (data.py:53-80, 94-95), one image after another
  under ``random.seed / np.random.seed / torch.manual_seed(3)``.

Environment that produced the committed file: Pillow 12.2.0, numpy 2.3.5, torch 2.11.0, torchvision 0.26.0.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_resize import chain_digests, chain_input, digest, reference_transforms  # noqa: E402

SIZES = ((375, 500), (500, 375), (333, 500), (256, 256), (375, 500), (48, 64), (3, 4), (500, 375), (333, 500),
         (375, 500))
INPUT_SIZES = (224, 380)
SEED = 77


def ragged_inputs():
    rng = np.random.default_rng(SEED)
    return [chain_input(rng, i, h, w) for i, (h, w) in enumerate(SIZES)]


def main(ref):
    from make_golden import import_reference
    aug, archive, _, data = import_reference(ref)
    batch = ragged_inputs()
    out = {"in": np.array([digest(a) for a in batch])}
    for s in INPUT_SIZES:
        for name, tf in reference_transforms(aug, archive, data, s).items():
            out["%s_s%d" % (name, s)] = chain_digests(tf, batch)
    path = os.path.join(HERE, "golden_ragged.npz")
    np.savez_compressed(path, **out)
    print("wrote golden_ragged.npz:", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
