"""faa_crop_resize on the device (EfficientNet crops + Pillow bicubic Resize) and the ImageNet chains built on it,
bit for bit against the host build of the kernel's arithmetic, the NumPy model and the reference's own transforms."""
import hashlib
import os
import random
import sys

import numpy as np
import pytest
import torch

import resize_model as M
from helpers import ROOT
from test_crop_resize_host import emu_crop_resize, emu_philox_boxes, load_emu_resize

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, TailSpec

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_resize as G  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_resize.npz")


@pytest.fixture(scope="module")
def emu_rs():
    return load_emu_resize()


def norm_f32(u8_hwc):
    """ToTensor + Normalize in fp32 (torch's operation order) of uint8 [B,H,W,3] -> [B,3,H,W]"""
    x = torch.from_numpy(np.ascontiguousarray(u8_hwc)).permute(0, 3, 1, 2).float() / 255.0
    m = torch.tensor(IMAGENET_MEAN, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(IMAGENET_STD, dtype=torch.float32).view(1, 3, 1, 1)
    return (x - m) / s


def noise_batch(rng, n, h, w):
    b = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    b[::2] = np.clip(np.linspace(10, 240, w)[None, None, :, None] + rng.normal(0, 9, (len(b[::2]), h, w, 3)), 0, 255)
    return b


def random_boxes(rng, n, h, w):
    bx = np.zeros(n, _lib.CROP_BOX_DTYPE)
    for i in range(n):
        bw, bh = int(rng.integers(1, w + 1)), int(rng.integers(1, h + 1))
        if i % 5 == 0:
            bw, bh = w, h
        bx[i] = (int(rng.integers(0, w - bw + 1)), int(rng.integers(0, h - bh + 1)), bw, bh)
    return bx


CASES = [((256, 256), 224, 24), ((375, 500), 224, 24), ((333, 500), 380, 12), ((48, 64), 224, 12),
         ((301, 203), 224, 12), ((375, 500), 600, 6), ((1536, 2048), 224, 3)]


@pytest.mark.parametrize("src,size,n", CASES)
def test_given_boxes_bitexact_all_dtypes(emu_rs, src, size, n):
    h, w = src
    rng = np.random.default_rng(h * 7 + w + size)
    batch = noise_batch(rng, n, h, w)
    boxes = random_boxes(rng, n, h, w)
    want = np.stack([emu_crop_resize(emu_rs, batch[i], tuple(int(v) for v in boxes[i]), size, size) for i in range(n)])
    for i in (0, n - 1):
        assert np.array_equal(want[i], M.crop_resize(batch[i], boxes[i], size, size))
    x = torch.from_numpy(batch).cuda()
    got = engine.crop_resize(x, size, boxes=boxes)
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), want)
    f32 = norm_f32(want)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
        y = engine.crop_resize(x, size, boxes=torch.from_numpy(boxes.view(np.int32).reshape(n, 4)), tail=tail)
        torch.cuda.synchronize()
        assert torch.equal(y.cpu(), f32.to(dt)), dt                 # fp16 / bf16: the fp32 value rounded once


def test_normalised_output_equals_faa_augment(emu_rs):
    rng = np.random.default_rng(5)
    batch = noise_batch(rng, 16, 375, 500)
    x = torch.from_numpy(batch).cuda()
    boxes = random_boxes(rng, 16, 375, 500)
    u8 = engine.crop_resize(x, 224, boxes=boxes)
    ident = CompiledPolicy([[("Invert", -1.0, 0.0)]])
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
        a = engine.augment_batch(ident, u8, tail, rng=engine.make_rng(1, 0, tail))
        b = engine.crop_resize(x, 224, boxes=boxes, tail=tail)
        torch.cuda.synchronize()
        assert torch.equal(a, b), dt


@pytest.mark.parametrize("size,src", [(224, (375, 500)), (380, (500, 375)), (224, (256, 256)), (224, (1536, 2048))])
def test_philox_and_center_boxes_equal_host_build(emu_rs, size, src):
    h, w = src
    n = 40 if h < 1000 else 4
    rng = np.random.default_rng(size + h)
    batch = noise_batch(rng, n, h, w)
    x = torch.from_numpy(batch).cuda()
    cfg = engine.crop_cfg(size, seed=123, first_index=7000)
    boxes = emu_philox_boxes(emu_rs, cfg, n, h, w)
    got = engine.crop_resize(x, size, rng=cfg)
    via_boxes = engine.crop_resize(x, size, boxes=boxes)
    center = engine.crop_resize(x, size, rng=engine.crop_cfg(size, center=True))
    torch.cuda.synchronize()
    assert torch.equal(got, via_boxes)               # the device drew the host build's boxes
    for i in range(0, n, max(1, n // 8)):
        assert np.array_equal(got[i].cpu().numpy(), M.crop_resize(batch[i], boxes[i], size, size))
        assert np.array_equal(center[i].cpu().numpy(), M.crop_resize(batch[i], M.center_box(h, w, size), size, size))


@pytest.mark.parametrize("src", [(1801, 1801), (1800, 2400)])
def test_plans_near_48kb_of_shared_memory(emu_rs, src):
    """sources whose tile plan needs just under 48 KB of dynamic shared memory: with the kernel's static table the
    total is above the default limit, so the launch must raise it"""
    h, w = src
    rng = np.random.default_rng(h + w)
    batch = noise_batch(rng, 2, h, w)
    x = torch.from_numpy(batch).cuda()
    box = M.center_box(h, w, 224)
    want = np.stack([M.crop_resize(a, box, 224, 224) for a in batch])
    for dt in (torch.float32, torch.float16, torch.uint8):
        tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
        got = engine.crop_resize(x, 224, rng=engine.crop_cfg(224, center=True), tail=tail)
        torch.cuda.synchronize()
        if dt == torch.uint8:
            assert np.array_equal(got.cpu().numpy(), want)
        else:
            assert torch.equal(got.cpu(), norm_f32(want).to(dt)), dt
    cfg = engine.crop_cfg(224, seed=8)
    got = engine.crop_resize(x, 224, rng=cfg)
    torch.cuda.synchronize()
    boxes = emu_philox_boxes(emu_rs, cfg, 2, h, w)
    assert np.array_equal(got.cpu().numpy(), np.stack([M.crop_resize(a, b, 224, 224) for a, b in zip(batch, boxes)]))


def test_empty_center_crop_is_refused_in_both_modes():
    x = torch.zeros(1, 10, 12, 3, dtype=torch.uint8, device="cuda")
    for center in (True, False):
        with pytest.raises(ValueError):
            engine.crop_resize(x, 8, rng=engine.crop_cfg(1, center=center))


def test_bad_boxes_are_refused():
    x = torch.zeros(2, 40, 50, 3, dtype=torch.uint8, device="cuda")
    for bad in ([(0, 0, 50, 40), (1, 0, 50, 40)], [(0, 0, 0, 4), (0, 0, 5, 5)], [(0, 0, 5, 5), (-1, 0, 5, 5)],
                [(0, 36, 5, 5), (0, 0, 5, 5)]):
        with pytest.raises(ValueError):
            engine.crop_resize(x, 32, boxes=np.array(bad, np.int32))


def test_policy_then_crop_resize_needs_no_synchronize():
    """the crop-resize launch is stream-ordered behind the policy kernels that write its input"""
    pol = CompiledPolicy(archive.fa_resnet50_rimagenet())
    rng = np.random.default_rng(9)
    x = torch.from_numpy(noise_batch(rng, 256, 375, 500)).cuda()
    raw = TailSpec.raw_u8()
    cfg = engine.crop_cfg(224, seed=5, first_index=0)
    torch.cuda.synchronize()
    a = engine.augment_batch(pol, x, raw, rng=engine.make_rng(3, 0, raw))
    ya = engine.crop_resize(a, 224, rng=cfg)
    torch.cuda.synchronize()
    b = engine.augment_batch(pol, x, raw, rng=engine.make_rng(3, 0, raw))
    torch.cuda.synchronize()
    yb = engine.crop_resize(b, 224, rng=cfg)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(ya, yb)


def _chain_inputs():
    rng = np.random.default_rng(2024)
    out = {}
    for h, w, n in G.CHAIN_CASES:
        out[(h, w)] = np.stack([G.chain_input(rng, i, h, w) for i in range(n)])
    return out


def _reference_transforms():
    try:
        from oracle import build_ref
        mods = build_ref.import_ref()
    except Exception:
        mods = None
    if mods is None:
        return None
    aug, ref_archive, _, ref_data = mods
    import PIL.Image
    from torchvision.transforms import transforms as T
    norm = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    test = T.Compose([ref_data.EfficientNetCenterCrop(224), T.Resize((224, 224), interpolation=PIL.Image.BICUBIC),
                      T.ToTensor(), norm])
    train = T.Compose([
        ref_data.Augmentation(ref_archive.fa_resnet50_rimagenet()),
        ref_data.EfficientNetRandomCrop(224), T.Resize((224, 224), interpolation=PIL.Image.BICUBIC),
        T.RandomHorizontalFlip(), T.ColorJitter(brightness=0.4, contrast=0.4, saturation=0.4), T.ToTensor(),
        aug.Lighting(0.1, ref_data._IMAGENET_PCA["eigval"], ref_data._IMAGENET_PCA["eigvec"]), norm])
    return {"train": train, "test": test}


def test_full_reference_chains_parity():
    """transform_train (fa_resnet50_rimagenet) and transform_test (data.py:60-80) == the batched parity chains, fp32"""
    import PIL.Image
    g = np.load(GOLDEN)
    ref = _reference_transforms()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float32)
    for (h, w), batch in _chain_inputs().items():
        tag = "%dx%d" % (h, w)
        assert [G.digest(a) for a in batch] == list(g["in_" + tag])
        x = torch.from_numpy(batch).cuda()
        for name in ("test", "train"):
            random.seed(3)
            np.random.seed(3)
            torch.manual_seed(3)
            got = (chain.train(x, parity=True) if name == "train" else chain.test(x)).cpu().numpy()
            assert got.shape == (len(batch), 3, 224, 224)
            if ref is not None:
                random.seed(3)
                np.random.seed(3)
                torch.manual_seed(3)
                want = np.stack([ref[name](PIL.Image.fromarray(a)).numpy() for a in batch])
                assert float(np.abs(got - want).max()) == 0.0, (name, tag)
            assert [G.digest(a) for a in got] == list(g["%s_%s" % (name, tag)]), (name, tag)


def test_philox_train_chain_runs_and_is_keyed():
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float16)
    x = torch.from_numpy(noise_batch(np.random.default_rng(1), 64, 375, 500)).cuda()
    a = chain.train(x, seed=4, first_index=0)
    b = chain.train(x, seed=4, first_index=0)
    c = chain.train(x, seed=4, first_index=64)
    torch.cuda.synchronize()
    assert a.shape == (64, 3, 224, 224) and a.dtype == torch.float16
    assert torch.equal(a, b) and not torch.equal(a, c) and bool(torch.isfinite(a.float()).all())


@pytest.mark.parametrize("model_type,size", [("resnet50", 224), ("efficientnet-b1", 240)])
def test_loader_with_crop_resize(model_type, size):
    from fast_autoaugment_b200.conf import Config as C
    rng = np.random.default_rng(0)
    tr = noise_batch(rng, 40, 300, 400)
    te = noise_batch(rng, 12, 300, 400)
    root = {"train": (tr, [i % 4 for i in range(40)]), "test": (te, [i % 4 for i in range(12)])}
    conf = C.get()
    saved = dict(conf)
    try:
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": model_type}})
        _, train, valid, test = data.get_dataloaders("imagenet", 8, root, split=0.0)
        xb, yb = next(iter(train))
        assert tuple(xb.shape) == (8, 3, size, size) and xb.dtype == torch.float32 and yb.shape == (8,)
        got = torch.cat([xb for xb, _ in test])
        want = norm_f32(np.stack([M.crop_resize(a, M.center_box(300, 400, size), size, size) for a in te]))
        assert torch.equal(got.cpu(), want)
    finally:
        conf.clear()
        conf.update(saved)
