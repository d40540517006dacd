"""The ImageNet directory source without a device: ``data.imagenet_index`` against torchvision's ``ImageFolder`` and,
where ``oracle/_ref`` has been built, the reference's own ``ImageNet`` on trees with nested folders, mixed-case
extensions, skipped files, PNGs, a symlinked class and a ``train_cls.txt``; the samplers of ``get_dataloaders`` over
it; and the host half of batch staging (``read_jpeg_batch``) against ``EncodedImages.from_bytes``."""
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from imagenet_tree import baseline_file, pillow_pixels, refused_files, write, write_tree
from jpeg_cases import pillow

from fast_autoaugment_b200 import data
from fast_autoaugment_b200.engine import EncodedImages


def odd_tree(root):
    """val and train folders with nested subdirectories, .JPEG / .jpg / .Jpeg / .png files, files the extension filter
    skips, and a class that is a symlink to a directory elsewhere"""
    base = os.path.join(str(root), "imagenet-pytorch")
    k = 0
    for split in ("train", "val"):
        s = os.path.join(base, split)
        for rel in ("n01/a.JPEG", "n01/b.jpg", "n01/sub/c.Jpeg", "n01/sub/deeper/d.JPEG", "n01/e.png",
                    "n01/notes.txt", "n01/f.JPEG.bak", "n02/z.JPEG", "n02/A.JPEG", "n02/sub2/m.PNG", "n02/README",
                    "n00/x.jpeg"):
            write(os.path.join(s, rel), baseline_file(k, 1))
            k += 1
        elsewhere = os.path.join(str(root), "elsewhere_" + split)
        write(os.path.join(elsewhere, "q.JPEG"), baseline_file(k, 1))
        write(os.path.join(elsewhere, "inner", "r.jpg"), baseline_file(k + 1, 1))
        os.symlink(elsewhere, os.path.join(s, "n03"))
        write(os.path.join(s, "stray_file_at_top.JPEG"), baseline_file(k + 2, 1))
    return base


def image_folder_samples(folder):
    import torchvision
    return torchvision.datasets.ImageFolder(folder).samples


def reference_imagenet():
    from oracle import build_ref
    if build_ref.import_ref() is None:
        return None
    from FastAutoAugment.imagenet import ImageNet
    return ImageNet


def write_meta(base):
    """meta.bin of the reference's ImageNet (wnid -> class names, val wnids): it reads it for class names only"""
    wnids = set()
    for split in ("train", "val"):
        d = os.path.join(base, split)
        if os.path.isdir(d):
            wnids.update(n for n in os.listdir(d) if os.path.isdir(os.path.join(d, n)))
    lst = os.path.join(base, "train_cls.txt")
    if os.path.exists(lst):
        with open(lst) as f:
            wnids.update(line.strip().split(" ")[0].split("/")[0] for line in f if line.strip())
    torch.save(({w: (w,) for w in sorted(wnids)}, []), os.path.join(base, "meta.bin"))


@pytest.mark.parametrize("split", ["train", "val"])
def test_index_equals_image_folder(tmp_path, split):
    base = odd_tree(tmp_path)
    got = data.imagenet_index(str(tmp_path), split)
    want = image_folder_samples(os.path.join(base, split))
    assert got == want
    names = [os.path.relpath(p, os.path.join(base, split)) for p, _ in got]
    assert "n01/sub/deeper/d.JPEG" in names and "n01/e.png" in names and "n02/sub2/m.PNG" in names
    assert "n03/inner/r.jpg" in names                                  # walked through the symlink
    assert not any(n.endswith((".txt", ".bak", "README")) for n in names)
    assert sorted({t for _, t in got}) == [0, 1, 2, 3]


def test_empty_class_raises_like_image_folder(tmp_path):
    base = odd_tree(tmp_path)
    os.makedirs(os.path.join(base, "val", "n99_empty"))
    write(os.path.join(base, "val", "n99_empty", "only.txt"), b"x")
    with pytest.raises(FileNotFoundError) as want:
        image_folder_samples(os.path.join(base, "val"))
    with pytest.raises(FileNotFoundError) as got:
        data.imagenet_index(str(tmp_path), "val")
    assert str(got.value) == str(want.value)


def test_missing_folder_names_the_path(tmp_path):
    with pytest.raises(FileNotFoundError, match=re.escape(os.path.join(str(tmp_path), "imagenet-pytorch", "val"))):
        data.imagenet_index(str(tmp_path), "val")
    with pytest.raises(FileNotFoundError, match=re.escape(os.path.join(str(tmp_path), "imagenet-pytorch", "train"))):
        data._load_arrays("imagenet", str(tmp_path))


def test_reduced_imagenet_stays_refused(tmp_path):
    write_tree(tmp_path, 0, per_class=2, n_val=1)
    with pytest.raises(ValueError, match="invalid dataset name=reduced_imagenet"):
        data._load_arrays("reduced_imagenet", str(tmp_path))


LIST = ["n05/img_b", "n02/img_z", "", "n05/sub/img_a extra fields 7", "   ", "n02/img_a", "n09/img_0"]


def list_tree(root):
    base = os.path.join(str(root), "imagenet-pytorch")
    for line in LIST:
        if line.strip():
            write(os.path.join(base, "train", line.strip().split(" ")[0] + ".JPEG"), baseline_file(len(line), 2))
    for other in ("n05/not_listed.JPEG", "n02/also_not_listed.jpg", "n07/unlisted_class.JPEG"):   # ignored
        write(os.path.join(base, "train", other), baseline_file(3, 2))
    with open(os.path.join(base, "train_cls.txt"), "w") as f:
        f.write("\n".join(LIST) + "\n")
    write(os.path.join(base, "val", "n02", "v.JPEG"), baseline_file(4, 2))
    return base


def test_train_cls_list(tmp_path):
    base = list_tree(tmp_path)
    got = data.imagenet_index(str(tmp_path), "train")
    t = os.path.join(base, "train")
    want = [(os.path.join(t, "n05/img_b.JPEG"), 1), (os.path.join(t, "n02/img_z.JPEG"), 0),
            (os.path.join(t, "n05/sub/img_a.JPEG"), 1), (os.path.join(t, "n02/img_a.JPEG"), 0),
            (os.path.join(t, "n09/img_0.JPEG"), 2)]
    assert got == want
    assert data.imagenet_index(str(tmp_path), "val") == [(os.path.join(base, "val", "n02", "v.JPEG"), 0)]


def test_equals_reference_imagenet(tmp_path):
    ImageNet = reference_imagenet()
    if ImageNet is None:
        pytest.skip("oracle/_ref has not been built (no reference checkout)")
    for sub, make in (("odd", odd_tree), ("list", list_tree), ("seeded", lambda r: write_tree(r, 3, per_class=3, n_val=2))):
        root = tmp_path / sub
        base = make(root)
        write_meta(base)
        for split in ("train", "val"):
            ref = ImageNet(base, split=split)
            assert data.imagenet_index(str(root), split) == ref.samples, (sub, split)
            tr = data._load_arrays("imagenet", str(root))
            if split == "train":
                assert tr[1] == [lb for _, lb in ref.samples]           # data.py:150


@pytest.mark.parametrize("split_idx,target_lb", [(0, -1), (3, -1), (0, 1), (3, 2)])
def test_samplers_over_directory_equal_samplers_over_mapping(tmp_path, split_idx, target_lb):
    write_tree(tmp_path, 5, n_classes=3, per_class=8, n_val=2, refused=False, text=False)
    paths, targets, vpaths, vtargets = data._load_arrays("imagenet", str(tmp_path))
    assert isinstance(paths, data.FilePaths) and isinstance(vpaths, data.FilePaths)
    imgs = [np.zeros((2, 2, 3), np.uint8)] * len(targets)
    _, mtargets, _, _ = data._load_arrays("imagenet", {"train": (imgs, targets), "test": (imgs[:2], vtargets[:2])})
    assert targets == [t for _, t in image_folder_samples(os.path.join(str(tmp_path), "imagenet-pytorch", "train"))]
    torch.manual_seed(0)
    a = data.split_samplers(targets, 0.15, split_idx, False, target_lb)
    torch.manual_seed(0)
    b = data.split_samplers(mtargets, 0.15, split_idx, False, target_lb)
    assert list(a[0].indices) == list(b[0].indices) and list(a[1].indices) == list(b[1].indices)
    assert len(a[1].indices) > 0
    if target_lb >= 0:
        assert all(targets[i] == target_lb for i in list(a[0].indices) + list(a[1].indices))


def test_host_staging_equals_from_bytes(tmp_path):
    base = write_tree(tmp_path, 7, n_classes=2, per_class=6, n_val=1)
    paths = [p for p, _ in data.imagenet_index(str(tmp_path), "train")]
    rng = np.random.default_rng(0)
    batch = [paths[int(i)] for i in rng.permutation(len(paths))]
    files = [open(p, "rb").read() for p in batch]
    refused_names = set(refused_files(7))
    with ThreadPoolExecutor(4) as ex:
        hb = data.read_jpeg_batch(batch, ex.map)
    want_refused = [i for i, p in enumerate(batch) if os.path.basename(p) in refused_names]
    assert list(hb.refused) == want_refused and len(want_refused) == 3
    with pytest.raises(ValueError) as e:
        EncodedImages.from_bytes(files, device="cpu")
    named = [int(m) for m in re.findall(r"(?:take: |; )(\d+): ", str(e.value))]
    assert named == want_refused
    ok = [i for i in range(len(batch)) if i not in want_refused]
    assert list(hb.accepted) == ok
    enc = EncodedImages.from_bytes([files[i] for i in ok], device="cpu")
    assert hb.headers.tobytes() == enc.headers.tobytes()
    assert hb.pool.tobytes() == enc.pool.tobytes()
    for i, px in zip(hb.refused, hb.pixels):
        assert np.array_equal(px, pillow(files[i]))
    sizes = hb.sizes()
    assert [tuple(s) for s in sizes] == [pillow(f).shape[:2] for f in files]

    lay = data._Layout(hb)                                     # the staged bytes, as the device buffer receives them
    buf = np.full(lay.total, 0xA5, np.uint8)
    lay.pack(hb, buf)
    assert buf[:hb.headers.nbytes].tobytes() == hb.headers.tobytes()
    assert buf[lay.pool:lay.pool + hb.pool.nbytes].tobytes() == hb.pool.tobytes()
    for k, i in enumerate(ok):
        o = lay.files + int(hb.headers["offset"][k])
        assert buf[o:o + len(files[i])].tobytes() == files[i]
    for o, i in zip(lay.pixels, hb.refused):
        assert o % 16 == 0 and buf[o:o + int(np.prod(pillow(files[i]).shape))].tobytes() == pillow(files[i]).tobytes()
    assert pillow_pixels(batch[:1])[0].shape[2] == 3


def test_unreadable_file_names_its_path(tmp_path):
    p = os.path.join(str(tmp_path), "imagenet-pytorch", "val", "n01", "broken.JPEG")
    write(p, b"this is not an image")
    with pytest.raises(OSError, match=re.escape(p)):
        data.read_jpeg_batch([p])
