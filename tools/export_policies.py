#!/usr/bin/env python
"""Export the reference's policy archive into compact data files.

``python tools/export_policies.py <checkout of kakaobrain/fast-autoaugment>``; the outputs
``fast_autoaugment_b200/policies/<name>.json`` are committed so the package has
the searched policies (the *data* the reference publishes - its README result
tables are produced with them) without importing the reference.

Layout of each file: {"source": "<reference file:line>", "ops": [op names],
"n_sub": S, "n_op": K, "table": [[op_index, prob, level], ...]}  (row-major,
S*K rows).  ``level`` is what ``Augmentation`` receives, i.e. AFTER the
``autoaug2arsaug`` re-scaling (archive.py:59-87) for the two AutoAugment sets.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "fast_autoaugment_b200", "policies")

SETS = {
    "fa_reduced_cifar10": "FastAutoAugment/archive.py:281",
    "fa_resnet50_rimagenet": "FastAutoAugment/archive.py:286",
    "fa_reduced_svhn": "FastAutoAugment/archive.py:291",
    "arsaug_policy": "FastAutoAugment/archive.py:11",
    "autoaug_paper_cifar10": "FastAutoAugment/archive.py:90-119",
    "autoaug_policy": "FastAutoAugment/archive.py:122-242",
}


def main(ref):
    sys.path.insert(0, ref)
    from FastAutoAugment import archive
    os.makedirs(OUT, exist_ok=True)
    for name, src in SETS.items():
        subs = getattr(archive, name)()
        ops = sorted({op for sub in subs for op, _, _ in sub})
        n_op = len(subs[0])
        assert all(len(s) == n_op for s in subs)
        table = [[ops.index(op), float(p), float(l)] for sub in subs for op, p, l in sub]
        with open(os.path.join(OUT, name + ".json"), "w") as f:
            json.dump({"source": src, "ops": ops, "n_sub": len(subs), "n_op": n_op,
                       "table": table}, f, separators=(",", ":"))
        print(name, len(subs), "sub-policies x", n_op, "ops")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
