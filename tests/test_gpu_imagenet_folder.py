"""The ImageNet directory on the device: ``get_dataloaders('imagenet', ...)`` over a seeded tree in the reference's
layout (4:2:0 / 4:2:2 / 4:4:4, grayscale and restart-interval files at mixed sizes, a progressive JPEG, a CMYK JPEG, a
PNG named .JPEG and a text file) against the same loaders over Pillow's pixels and over the files' bytes; the refused
files' pixels; corrupt scans; device memory; the staging slots."""
import os
import re

import numpy as np
import pytest
import torch
from torch.utils.data.distributed import DistributedSampler

from helpers import seed_all
from imagenet_tree import baseline_file, cut_scan, pillow_pixels, refused_files, write, write_tree
from jpeg_cases import content, encode

from fast_autoaugment_b200 import data
from fast_autoaugment_b200.conf import Config as C_

pytestmark = pytest.mark.gpu

B = 8


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("imagenet")
    write_tree(root, 11, n_classes=3, per_class=10, n_val=4)
    return str(root)


class conf_set:
    def __init__(self, **kw):
        self.kw = {"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}, **kw}

    def __enter__(self):
        self.saved = dict(C_.get())
        C_.get().clear()
        C_.get().update(self.kw)

    def __exit__(self, *a):
        C_.get().clear()
        C_.get().update(self.saved)


def index(root):
    tr, te = data.imagenet_index(root, "train"), data.imagenet_index(root, "val")
    return [p for p, _ in tr], [t for _, t in tr], [p for p, _ in te], [t for _, t in te]


def run(loader, seed):
    seed_all(seed)
    return [(x.cpu(), y.cpu()) for x, y in loader]


def assert_same(got, want, what):
    assert len(got) == len(want) and len(got) > 0, what
    for k, ((xa, ya), (xw, yw)) in enumerate(zip(got, want)):
        assert torch.equal(ya, yw), (what, k)
        assert torch.equal(xa, xw), (what, k)


def extra_loaders(ds, parity):
    """a shuffled train loader and one over a DistributedSampler (rank 1 of 2) on the same dataset"""
    pol = data.policy_by_conf_name("fa_reduced_imagenet")
    tail = data.TailSpec(None, 0, True, data.IMAGENET_MEAN, data.IMAGENET_STD, 0, torch.float32)
    seed_all(5)
    shuf = data.GpuAugmentedLoader(ds, B, pol, tail, shuffle=True, drop_last=True, parity=parity,
                                   chain=data.ImageNetChain(pol, 224, torch.float32))
    samp = DistributedSampler(range(len(ds)), num_replicas=2, rank=1, shuffle=True, seed=9)
    dist = data.GpuAugmentedLoader(ds, B, pol, tail, sampler=samp, drop_last=False, parity=parity,
                                   chain=data.ImageNetChain(pol, 224, torch.float32))
    return shuf, dist


@pytest.mark.parametrize("parity", [False, True])
def test_directory_loaders_equal_loaders_over_pillow_pixels(tree, parity):
    trp, trt, tep, tet = index(tree)
    mapping = {"train": (pillow_pixels(trp), trt), "test": (pillow_pixels(tep), tet)}
    with conf_set(faa_parity=parity):
        seed_all(3)
        got = data.get_dataloaders("imagenet", B, tree, split=0.2)
        seed_all(3)
        want = data.get_dataloaders("imagenet", B, mapping, split=0.2)
    assert isinstance(got[1].dataset, data.JpegFileDataset) and isinstance(got[3].dataset, data.JpegFileDataset)
    assert isinstance(want[1].dataset, data.RaggedDeviceDataset)
    assert got[1].dataset.targets == trt and got[3].dataset.targets == tet
    assert list(got[0].indices) == list(want[0].indices)
    g_extra, w_extra = extra_loaders(got[1].dataset, parity), extra_loaders(want[1].dataset, parity)
    for epoch in range(2):
        g_extra[1].sampler.set_epoch(epoch)
        w_extra[1].sampler.set_epoch(epoch)
        for which, g, w in (("train", got[1], want[1]), ("valid", got[2], want[2]), ("test", got[3], want[3]),
                            ("shuffled", g_extra[0], w_extra[0]), ("distributed", g_extra[1], w_extra[1])):
            assert_same(run(g, 100 + epoch), run(w, 100 + epoch), (which, epoch))


@pytest.mark.parametrize("parity", [False, True])
def test_directory_loaders_equal_bytes_mapping_on_baseline_files(tmp_path, parity):
    write_tree(tmp_path, 12, n_classes=2, per_class=9, n_val=5, refused=False)
    trp, trt, tep, tet = index(str(tmp_path))
    read = lambda ps: [open(p, "rb").read() for p in ps]            # noqa: E731
    with conf_set(faa_parity=parity):
        seed_all(4)
        got = data.get_dataloaders("imagenet", B, str(tmp_path), split=0.0)
        seed_all(4)
        want = data.get_dataloaders("imagenet", B, {"train": (read(trp), trt), "test": (read(tep), tet)}, split=0.0)
    assert isinstance(want[1].dataset, data.EncodedDeviceDataset)
    for epoch in range(2):
        for which in (1, 3):
            assert_same(run(got[which], 7 + epoch), run(want[which], 7 + epoch), (which, epoch))


def test_refused_files_get_pillow_pixels_in_their_positions(tree):
    trp, _, _, _ = index(tree)
    names = set(refused_files(11))
    refused = [p for p in trp if os.path.basename(p) in names]
    assert len(refused) == 3
    others = [p for p in trp if p not in refused]
    batches = [[others[0], refused[0], others[1], refused[1], refused[2]], refused[::-1], others[2:9]]
    stream = data.FileBatchStream(workers=3)
    outs = list(stream(batches, "cuda"))
    torch.cuda.synchronize()
    for paths, out in zip(batches, outs):
        want = pillow_pixels(paths)
        assert [tuple(s) for s in out.sizes] == [w.shape[:2] for w in want]
        for i, w in enumerate(want):
            assert np.array_equal(out.image(i).cpu().numpy(), w), paths[i]


def corrupt_tree(root, pos):
    """a val split of 6 batches of 4 baseline files whose file ``pos`` (index order) is cut inside its scan"""
    write_tree(root, 13, n_classes=2, per_class=3, n_val=12, refused=False, text=False)
    _, _, tep, _ = index(str(root))
    with open(tep[pos], "rb") as f:
        b = f.read()
    write(tep[pos], cut_scan(b))
    return tep[pos], len(tep)


@pytest.mark.parametrize("pos", [5, 23])
def test_corrupt_scan_raises_naming_the_file(tmp_path, pos):
    bad, n = corrupt_tree(tmp_path, pos)
    with conf_set():
        _, _, _, test = data.get_dataloaders("imagenet", 4, str(tmp_path), split=0.0)
    seen = []
    with pytest.raises(OSError, match=re.escape(bad) + r": 0x[0-9a-f]+ \([^)]*scan truncated"):
        for x, _ in test:
            seen.append(x)
    assert len(seen) <= pos // 4 + 1                     # no later than the batch after the one that holds it
    if pos // 4 + 1 == n // 4:                           # the last batch: checked at the end of the epoch
        assert len(seen) == n // 4


def test_dataset_keeps_no_file_on_the_device(tmp_path):
    base = os.path.join(str(tmp_path), "imagenet-pytorch")
    big = encode(content("noise", 1024, 1024, 1), quality=95, subsampling=0)
    n = -(-64 * 2 ** 20 // len(big)) + 2
    for i in range(n):
        write(os.path.join(base, "train", "n%02d" % (i % 2), "f%03d.JPEG" % i), big)
    for i in range(2):
        write(os.path.join(base, "val", "n00", "v%d.JPEG" % i), baseline_file(i, 1))
    on_disk = sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(base) for f in fs)
    assert on_disk >= 64 * 2 ** 20
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    with conf_set():
        loaders = data.get_dataloaders("imagenet", 8, str(tmp_path), split=0.0)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - m0 < 2 ** 20
    assert len(loaders[1].dataset) == n


def test_loader_holds_at_most_two_staging_slots(tree):
    with conf_set():
        _, train, _, _ = data.get_dataloaders("imagenet", 4, tree, split=0.0)
    assert len(train) >= 6
    for epoch in range(2):
        for k, (x, _) in enumerate(train):
            st = train.staging
            live = [s for s in st.slots if s is not None]
            assert len(st.slots) == 2 and 1 <= len(live) <= 2 and all(s.is_pinned() for s in live)
        assert k + 1 == len(train)
    torch.cuda.synchronize()
