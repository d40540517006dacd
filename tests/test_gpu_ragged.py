"""The ImageNet chains on batches of differently sized sources (``RaggedImages``): the ragged crop-resize launch
against the host build of its arithmetic at each image's own size, the positional Philox sampler, the per-size policy
groups of ``ImageNetChain.train`` against a host reference assembled image by image, the parity chains against digests
of the reference's transforms, the loaders, and the launch counts."""
import ctypes as C
import os
import sys

import numpy as np
import PIL.Image
import pytest
import torch

import resize_model as M
from helpers import ROOT, emu_philox_records, philox_reference, reference_output, seed_all
from test_chain_records_host import jitter_oracle
from test_crop_resize_host import emu_crop_resize, emu_philox_boxes, load_emu_resize
from test_ragged_host import emu_philox_at, load_emu_ragged

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, RaggedImages, TailSpec

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_ragged as GR  # noqa: E402
import make_golden_resize as G  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_ragged.npz")
FLOATS = (torch.float32, torch.float16, torch.bfloat16)


@pytest.fixture(scope="module")
def emu_rs():
    return load_emu_resize()


@pytest.fixture(scope="module")
def emu_rg():
    return load_emu_ragged()


def norm_f32(u8_hwc):
    x = torch.from_numpy(np.ascontiguousarray(u8_hwc)).permute(0, 3, 1, 2).float() / 255.0
    m = torch.tensor(IMAGENET_MEAN, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(IMAGENET_STD, dtype=torch.float32).view(1, 3, 1, 1)
    return (x - m) / s


def launches():
    torch.cuda.synchronize()
    return _lib.lib.faa_launch_count()


def image(rng, i, h, w):
    if i % 2:
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return np.clip(np.linspace(10, 240, w)[None, :, None] + rng.normal(0, 9, (h, w, 3)), 0, 255).astype(np.uint8)


def images(sizes, seed):
    rng = np.random.default_rng(seed)
    return [image(rng, i, h, w) for i, (h, w) in enumerate(sizes)]


def random_box(rng, h, w, i):
    bw, bh = int(rng.integers(1, w + 1)), int(rng.integers(1, h + 1))
    if i % 5 == 0:
        bw, bh = w, h
    return int(rng.integers(0, w - bw + 1)), int(rng.integers(0, h - bh + 1)), bw, bh


def odd_offset_batch(imgs, order):
    """the images at odd byte offsets inside one larger storage (gaps between them), then descriptors in `order`"""
    offs, at = [], 0
    for a in imgs:
        at += 3 - at % 2                        # next offset odd, after a gap
        offs.append(at)
        at += a.size
    host = np.full(at + 7, 0xA5, np.uint8)
    for a, o in zip(imgs, offs):
        host[o:o + a.size] = a.reshape(-1)
    r = RaggedImages(torch.from_numpy(host).cuda(), offs, [a.shape[:2] for a in imgs])
    assert all(o % 2 == 1 for o in r.offsets)
    return r.select(order), [imgs[i] for i in order]


BATCHES = {
    "mixed_tall_and_wide": ([(375, 500), (500, 375), (333, 500), (48, 64), (3, 4), (256, 256)], (224, 380)),
    "8192x2_with_2x8192": ([(8192, 2), (2, 8192), (8192, 2)], (224,)),
    "1536x2048_among_small": ([(48, 64), (1536, 2048), (3, 4), (256, 256), (64, 48)], (224,)),
}


def _check(got, want_u8, dt, what):
    if dt == torch.uint8:
        bad = [i for i in range(len(want_u8)) if not np.array_equal(got[i].cpu().numpy(), want_u8[i])]
    else:
        f = norm_f32(np.stack(want_u8)).to(dt)
        bad = [i for i in range(len(want_u8)) if not torch.equal(got[i].cpu(), f[i])]
    assert not bad, (what, dt, bad)


@pytest.mark.parametrize("name", list(BATCHES) + ["odd_offsets_unsorted_repeated"])
def test_ragged_crop_resize_equals_host_build(emu_rs, name):
    if name == "odd_offsets_unsorted_repeated":
        sizes, outs = [(375, 500), (37, 41), (500, 375), (3, 4)], (224,)
        x, imgs = odd_offset_batch(images(sizes, 5), [2, 0, 2, 3, 1, 0])
    else:
        sizes, outs = BATCHES[name]
        imgs = images(sizes, len(sizes))
        x = RaggedImages.from_list(imgs)
    n = len(imgs)
    rng = np.random.default_rng(n)
    for s in outs:
        given = np.array([random_box(rng, a.shape[0], a.shape[1], i) for i, a in enumerate(imgs)], np.int32)
        cfg = engine.crop_cfg(s, seed=42, first_index=900)
        drawn = [emu_philox_boxes(emu_rs, engine.crop_cfg(s, seed=42, first_index=900 + i), 1, *a.shape[:2])[0]
                 for i, a in enumerate(imgs)]
        cases = [("given", dict(boxes=given), [tuple(b) for b in given]),
                 ("philox", dict(rng=cfg), [tuple(int(v) for v in b) for b in drawn]),
                 ("center", dict(rng=engine.crop_cfg(s, center=True)), [M.center_box(*a.shape[:2], s) for a in imgs])]
        for what, kw, boxes in cases:
            want = [emu_crop_resize(emu_rs, a, b, s, s) for a, b in zip(imgs, boxes)]
            for i in (0, n - 1):
                assert np.array_equal(want[i], M.crop_resize(imgs[i], boxes[i], s, s))
            for dt in (torch.uint8,) + FLOATS:
                tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
                _check(engine.crop_resize(x, s, tail=tail, **kw), want, dt, (name, s, what))


def test_ragged_boxes_are_checked_against_their_own_image():
    x = RaggedImages.from_list(images([(40, 50), (50, 40)], 1))
    engine.crop_resize(x, 32, boxes=np.array([(0, 0, 50, 40), (0, 0, 40, 50)], np.int32))
    c0 = launches()
    for bad in ([(0, 0, 50, 40), (0, 0, 50, 40)], [(0, 0, 40, 50), (0, 0, 40, 50)], [(0, 0, 5, 5), (36, 0, 5, 5)]):
        with pytest.raises(ValueError):
            engine.crop_resize(x, 32, boxes=np.array(bad, np.int32))
    assert launches() == c0


# ------------------------------------------------------------------------------------- same size == uniform --
def test_same_size_ragged_batch_equals_the_uniform_launch():
    n = 16
    batch = np.stack(images([(375, 500)] * n, 7))
    x = torch.from_numpy(batch).cuda()
    r = RaggedImages.from_list(list(x))
    for kw in (dict(rng=engine.crop_cfg(224, seed=9, first_index=33)), dict(rng=engine.crop_cfg(224, center=True))):
        for dt in (torch.uint8,) + FLOATS:
            tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
            assert torch.equal(engine.crop_resize(r, 224, tail=tail, **kw), engine.crop_resize(x, 224, tail=tail, **kw))
    policies = archive.fa_resnet50_rimagenet()
    for dt in (torch.float32, torch.float16):
        chain = data.ImageNetChain(policies, 224, dt)
        a = chain.train(x, seed=5, first_index=4000)
        b = chain.train(r, seed=5, first_index=4000)
        assert torch.equal(a, b), dt


def test_sample_philox_at_equals_sample_philox(emu, emu_rg):
    pol = CompiledPolicy(archive.fa_resnet50_rimagenet())
    raw = TailSpec.raw_u8()
    n, h, w = 300, 375, 500
    rng = engine.make_rng(17, 123, raw)
    d_s = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    d_b = torch.empty(n * pol.n_op * 8, dtype=torch.uint8, device="cuda")
    t = raw.c_struct(h, w)
    _lib.check(_lib.lib.faa_sample_philox(pol.handle, n, h, w, C.byref(t), C.byref(rng), d_s.data_ptr(), d_b.data_ptr(),
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    s_at, b_at = engine.sample_philox_at(pol, np.arange(n), h, w, raw, engine.make_rng(17, 123, raw), torch.device("cuda"))
    assert torch.equal(s_at, d_s) and torch.equal(b_at, d_b)
    pos = np.array([5, 299, 0, 5, 100000, 77], np.int64)
    s_at, b_at = engine.sample_philox_at(pol, pos, h, w, raw, engine.make_rng(17, 123, raw), torch.device("cuda"))
    ws, wb = emu_philox_at(emu_rg, pol, pos, h, w, raw, 17, 123)
    assert s_at.cpu().numpy().tobytes() == ws.tobytes() and b_at.cpu().numpy().tobytes() == wb.tobytes()
    assert s_at[:16].cpu().numpy().tobytes() == d_s[5 * 16:6 * 16].cpu().numpy().tobytes()


# ----------------------------------------------------------------------------------- Philox train chain, mixed --
MIXED = [(375, 500), (37, 41), (500, 375), (333, 500), (375, 500), (256, 256), (500, 375), (48, 64), (375, 500),
         (3, 4), (333, 500)]           # (37 x 41: an odd byte count in front of groups whose rows are whole words)


@pytest.mark.parametrize("s", [224, 600])
def test_philox_train_chain_on_a_mixed_batch(emu, emu_rs, s):
    """each image == its own host reference: the policy's decisions of sample first + i at its size, its crop box
    at its size, resize, the batch's jitter record, flip and Lighting"""
    n = len(MIXED)
    seed, first = 2000 + s, 91 * s
    policies = archive.fa_resnet50_rimagenet()
    pol = CompiledPolicy(policies)
    imgs = images(MIXED, s)
    chain = data.ImageNetChain(policies, s, torch.float32)
    cropped = []
    for i, a in enumerate(imgs):
        h, w = a.shape[:2]
        u8 = philox_reference(emu, pol, a[None], TailSpec.raw_u8(), seed, first + i).numpy()[0]
        box = emu_philox_boxes(emu_rs, chain.crop.cfg(seed, first + i), 1, h, w)[0]
        cropped.append(M.crop_resize(u8, box, s, s))
    recs, rgb = chain._device_records(n, torch.device("cuda"), seed, first)
    jit = recs.cpu().numpy().view(_lib.JITTER_DTYPE).reshape(n)
    jittered = np.stack([jitter_oracle(cropped[i], jit[i]) for i in range(n)])
    flips, fb = emu_philox_records(emu, chain.flip_policy, n, s, s, chain.tail, seed, first)
    want = reference_output(emu, chain.flip_policy, jittered, chain.tail, flips, fb, lighting_rgb=rgb.cpu())
    x = RaggedImages.from_list(imgs)
    for dt in (torch.float32, torch.float16):
        got = data.ImageNetChain(policies, s, dt).train(x, seed=seed, first_index=first).cpu()
        assert got.shape == (n, 3, s, s) and got.dtype == dt
        bad = [i for i in range(n) if not torch.equal(got[i], want[i].to(dt))]
        assert not bad, (s, dt, bad)


# ------------------------------------------------------------------------------------------- parity chains --
@pytest.mark.parametrize("s", GR.INPUT_SIZES)
def test_ragged_parity_chains_equal_the_reference(s):
    g = np.load(GOLDEN)
    batch = GR.ragged_inputs()
    assert [G.digest(a) for a in batch] == list(g["in"])
    try:
        from oracle import build_ref
        mods = build_ref.import_ref()
    except Exception:
        mods = None
    ref = G.reference_transforms(*mods[:2], mods[3], s) if mods is not None else None
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), s, torch.float32)
    x = RaggedImages.from_list(batch)
    for name in ("test", "train"):
        seed_all(3)
        got = (chain.train(x, parity=True) if name == "train" else chain.test(x)).cpu().numpy()
        assert got.shape == (len(batch), 3, s, s)
        if ref is not None:
            seed_all(3)
            want = np.stack([ref[name](PIL.Image.fromarray(a)).numpy() for a in batch])
            assert float(np.abs(got - want).max()) == 0.0, (name, s)
        assert [G.digest(a) for a in got] == list(g["%s_s%d" % (name, s)]), (name, s)


# ------------------------------------------------------------------------------------------------- loaders --
def test_loaders_yield_the_chains_of_the_selected_images():
    from fast_autoaugment_b200.conf import Config as C_
    n, b = 12, 4
    tr = images([MIXED[i % len(MIXED)] for i in range(n)], 8)
    te = images([MIXED[(i + 3) % len(MIXED)] for i in range(6)], 9)
    root = {"train": (tr, list(range(n))), "test": (te, list(range(6)))}        # labels = dataset indices
    conf = C_.get()
    saved = dict(conf)
    try:
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}})
        _, train, _, test = data.get_dataloaders("imagenet", b, root, split=0.0)
        assert isinstance(train.dataset, data.RaggedDeviceDataset)
        k = -1
        for k, (xb, yb) in enumerate(train):
            want = train.chain.train(train.dataset.images.select(yb.tolist()), seed=train.seed, first_index=k * b)
            assert xb.shape == (b, 3, 224, 224) and torch.equal(xb, want), k
        assert k == n // b - 1
        got = torch.cat([xb for xb, _ in test])
        assert torch.equal(got, test.chain.test(RaggedImages.from_list(te)))
        conf.pop("faa_crop_resize")
        with pytest.raises(ValueError, match="faa_crop_resize"):
            data.get_dataloaders("imagenet", b, root, split=0.0)
    finally:
        conf.clear()
        conf.update(saved)


# ------------------------------------------------------------------------------------------------ launches --
def test_launch_counts():
    """a test batch is one launch; a train batch is, per source size, the positional sampler and the policy
    launches on the gathered images, then the crop-resize, the jitter and the flip + Lighting + Normalize launches"""
    policies = archive.fa_resnet50_rimagenet()
    chain = data.ImageNetChain(policies, 224, torch.float16)
    imgs = images(MIXED, 3)
    x = RaggedImages.from_list(imgs)
    chain.train(x, seed=1)                                          # (tables of every size exist)
    c0 = launches()
    chain.test(x)
    assert launches() - c0 == 1
    raw = TailSpec.raw_u8()
    per_group = 0
    groups = x.groups()
    assert len(groups) == len(set(MIXED))
    for (h, w), pos in groups:
        xs = torch.stack([x.image(int(i)) for i in pos])
        smp, bx = engine.sample_philox_at(chain.aug.compiled, pos, h, w, raw, engine.make_rng(1, 0, raw), xs.device)
        c = launches()
        engine.augment_batch(chain.aug.compiled, xs, raw, smp, bx)
        per_group += 1 + (launches() - c)
    y = torch.zeros(len(MIXED), 224, 224, 3, dtype=torch.uint8, device="cuda")
    recs, rgb = chain._device_records(len(MIXED), y.device, 1, 0)
    c = launches()
    engine.augment_batch(chain.flip_policy, y, chain.tail, rng=engine.make_rng(1, 0, chain.tail), lighting_rgb=rgb)
    tail = launches() - c
    c0 = launches()
    chain.train(x, seed=1)
    assert launches() - c0 == per_group + 2 + tail
    n_tab, nbytes = engine.cached_tables(chain.aug.compiled)
    assert n_tab == len(groups) and nbytes == n_tab * chain.aug.compiled.n_sub * chain.aug.compiled.n_op * 2 * 32
