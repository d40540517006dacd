#!/usr/bin/env python
"""Recipe for ``oracle/_ref``: the UNMODIFIED reference package, importable without the reference checkout.

TEST / BASELINE INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

The reference (kakaobrain/fast-autoaugment @ 2424224) is pure Python - there is nothing to
compile - so "building" it means placing its package where ``bench.py --impl reference`` can
import it on a machine that has no checkout of the reference:

    oracle/_ref/FastAutoAugment/   verbatim copy of <checkout>/FastAutoAugment (git-ignored:
                                   the reference's sources never enter this repository's history)
    oracle/_ref/theconf.py         import shim: ``theconf`` is not installed (reference data.py:16)
    oracle/_ref/torch_six_shim.py  import shim: ``torch._six`` no longer exists
                                   (reference networks/efficientnet_pytorch/condconv.py:4)
    oracle/_ref/MANIFEST.json      sha256 of every copied file + the commit they came from

``import_ref`` also installs an import shim for ``sklearn.model_selection`` when scikit-learn is not
installed (reference data.py:15 imports ``StratifiedShuffleSplit`` at module level; the augmentation path never
calls it).

The checkout is ``$FAA_REFERENCE_ROOT``, by default ``reference/`` next to this repository.
``python oracle/build_ref.py``; ``__graft_entry__.build()`` calls it and builds ``oracle/_ref`` whenever that
checkout exists.  Without it the tests compare against the fixtures under ``tests/golden/``, and
``bench.py --impl reference`` times the oracle's restatement (``kind: "port"``) and says so on stderr.
"""
from __future__ import annotations

import hashlib
import importlib.machinery
import json
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
# a checkout of kakaobrain/fast-autoaugment: $FAA_REFERENCE_ROOT, else reference/ next to this repository
REF_ROOT = os.environ.get("FAA_REFERENCE_ROOT") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
DST = os.path.join(HERE, "_ref")

THECONF = '''"""Import shim for the `theconf` package (not installed): the two names reference data.py /
train.py import.  `Config.get()` returns one process-wide dict, like theconf's singleton."""


class Config:
    _d = {}

    @classmethod
    def get(cls):
        return cls._d


class ConfigArgumentParser:  # only imported by train.py / search.py, never constructed here
    def __init__(self, *a, **k):
        raise RuntimeError("theconf shim: ConfigArgumentParser is not available")
'''

SIX = '''"""Import shim: `torch._six` was removed from torch; the reference only needs `container_abcs`."""
import collections.abc
import sys
import types


def install():
    if "torch._six" not in sys.modules:
        m = types.ModuleType("torch._six")
        m.container_abcs = collections.abc
        sys.modules["torch._six"] = m
'''


def install_sklearn_shim():
    """Import shim for ``sklearn.model_selection`` (reference data.py:15) when scikit-learn is not installed: the
    name imports, constructing it raises.  Nothing on the augmentation path uses it."""
    try:
        import sklearn.model_selection  # noqa: F401
        return
    except ImportError:
        pass

    class StratifiedShuffleSplit:
        def __init__(self, *a, **k):
            raise RuntimeError("sklearn shim: StratifiedShuffleSplit needs scikit-learn")
    sk, ms = types.ModuleType("sklearn"), types.ModuleType("sklearn.model_selection")
    sk.__spec__ = importlib.machinery.ModuleSpec("sklearn", None, is_package=True)     # (find_spec() callers)
    sk.__path__ = []
    ms.__spec__ = importlib.machinery.ModuleSpec("sklearn.model_selection", None)
    ms.StratifiedShuffleSplit = StratifiedShuffleSplit
    sk.model_selection = ms
    sys.modules["sklearn"], sys.modules["sklearn.model_selection"] = sk, ms


def build(force: bool = False) -> str | None:
    src = os.path.join(REF_ROOT, "FastAutoAugment")
    if not os.path.isdir(src):
        return DST if os.path.isdir(os.path.join(DST, "FastAutoAugment")) else None
    man_path = os.path.join(DST, "MANIFEST.json")
    files = {}
    for root, _, names in os.walk(src):
        for n in sorted(names):
            if n.endswith(".py"):
                p = os.path.join(root, n)
                with open(p, "rb") as f:
                    files[os.path.relpath(p, REF_ROOT)] = hashlib.sha256(f.read()).hexdigest()
    if not force and os.path.exists(man_path):
        try:
            with open(man_path) as f:
                if json.load(f).get("files") == files:
                    return DST
        except Exception:
            pass
    shutil.rmtree(DST, ignore_errors=True)
    os.makedirs(DST)
    shutil.copytree(src, os.path.join(DST, "FastAutoAugment"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    with open(os.path.join(DST, "theconf.py"), "w") as f:
        f.write(THECONF)
    with open(os.path.join(DST, "torch_six_shim.py"), "w") as f:
        f.write(SIX)
    commit = None
    try:
        with open(os.path.join(REF_ROOT, ".SUBMODULES.json")) as f:
            commit = json.load(f).get("commit")
    except Exception:
        pass
    with open(man_path, "w") as f:
        json.dump({"source": "kakaobrain/fast-autoaugment", "commit": commit, "files": files}, f, indent=1)
    return DST


def import_ref():
    """Import the vendored reference (``oracle/_ref``), or the live one when only that exists.
    Returns (augmentations, archive, aug_mixup, data) modules of the reference, or None."""
    root = None
    if os.path.isdir(os.path.join(DST, "FastAutoAugment")):
        root = DST
    elif os.path.isdir(os.path.join(REF_ROOT, "FastAutoAugment")):
        root = build() or None
    if root is None:
        return None
    if root not in sys.path:
        sys.path.insert(0, root)
    import torch_six_shim
    torch_six_shim.install()
    install_sklearn_shim()
    from FastAutoAugment import augmentations, archive, aug_mixup, data
    return augmentations, archive, aug_mixup, data


if __name__ == "__main__":
    out = build(force="--force" in sys.argv)
    print("oracle/_ref:", out)
