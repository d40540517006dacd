"""The policy over a batch of differently sized images in one launch group (``faa_augment_ragged``, ``augment_batch`` on
``RaggedImages``): every image against the host build at its own size (Philox and resolved records), against the oracle,
against the per-size launch groups of ``ImageNetChain._policy_ragged`` and the uniform launch, the parity train chain
against the golden digests, layouts, launch counts, cached tables and the parity draws."""
import os
import random
import sys

import numpy as np
import PIL.Image
import pytest
import torch

from helpers import ROOT, philox_reference, reference_output, seed_all
from test_gpu_geometries import _reduced
from test_gpu_ragged import BATCHES, MIXED, images, odd_offset_batch

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import CompiledPolicy, RaggedImages, TailSpec
from oracle import pil_path

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_ragged as GR  # noqa: E402
import make_golden_resize as G  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_ragged.npz")
RAW = TailSpec.raw_u8()


def many_sizes(seed, n):
    """a mixture of n images, at least 40 distinct sizes: the photo shapes and random sizes in [1, 700]^2"""
    rng = np.random.default_rng(seed)
    sizes = [(375, 500), (500, 375), (333, 500), (480, 640), (1, 1), (3, 4), (2, 64), (64, 2)]
    while len(set(sizes)) < 40 or len(sizes) < n:
        sizes.append((int(rng.integers(1, 701)), int(rng.integers(1, 701))))
    rng.shuffle(sizes)
    return [tuple(s) for s in sizes]


MANY = many_sizes(0, 48)
POLICIES = {
    "fa_resnet50_rimagenet": archive.fa_resnet50_rimagenet(),
    "every_class": _reduced(),
    "three_ops": [[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)],
                  [("Color", 1.0, 0.3), ("Cutout", 1.0, 0.4), ("TranslateY", 1.0, 0.8)],
                  [("AutoContrast", 1.0, 0.5), ("Sharpness", 1.0, 0.2), ("Rotate", 1.0, 0.9)],
                  [("Contrast", 1.0, 0.6), ("Posterize", 1.0, 0.5), ("Solarize", 0.5, 0.4)]],
}
MIXES = {name: sizes for name, (sizes, _) in BATCHES.items()}
MIXES["MIXED"] = MIXED
MIXES["many_sizes"] = MANY


def launches():
    torch.cuda.synchronize()
    return int(_lib.lib.faa_launch_count())


def host_philox(emu, pol, imgs, seed, first):
    """image i: the host build of a uniform launch of it alone, decisions of global sample first + i at its size"""
    return [philox_reference(emu, pol, a[None], RAW, seed, first + i).numpy()[0] for i, a in enumerate(imgs)]


def host_records(emu, pol, imgs, samples, boxes):
    return [reference_output(emu, pol, a[None], RAW, samples[i:i + 1], boxes[i:i + 1]).numpy()[0]
            for i, a in enumerate(imgs)]


def parity_records(pol, sizes, seed):
    seed_all(seed)
    recs = [pol.sample_parity(1, h, w, RAW) for h, w in sizes]
    return np.concatenate([s for s, _ in recs]), np.concatenate([b for _, b in recs])


def bad_images(got: RaggedImages, want):
    assert isinstance(got, RaggedImages) and len(got) == len(want)
    return [i for i, a in enumerate(want) if not np.array_equal(got.image(i).cpu().numpy(), a)]


@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("mix", list(MIXES))
def test_philox_equals_host_build(emu, policy, mix):
    sizes = MIXES[mix]
    pol = CompiledPolicy(POLICIES[policy])
    imgs = images(sizes, len(sizes))
    seed, first = 17 + len(sizes), 1000
    got = engine.augment_batch(pol, RaggedImages.from_list(imgs), RAW, rng=engine.make_rng(seed, first, RAW))
    assert not bad_images(got, host_philox(emu, pol, imgs, seed, first)), (policy, mix)
    # a fresh output starts every image on a 16-byte boundary
    assert all((got.storage.data_ptr() + int(o)) % 16 == 0 for o in got.offsets)


@pytest.mark.parametrize("policy", list(POLICIES))
def test_resolved_records_equal_host_build_and_oracle(emu, policy):
    pols = POLICIES[policy]
    pol = CompiledPolicy(pols)
    sizes = MIXED + [(1, 1), (2, 64), (64, 2), (3, 4)]
    imgs = images(sizes, 7)
    samples, boxes = parity_records(pol, sizes, 5)
    got = engine.augment_batch(pol, RaggedImages.from_list(imgs), RAW, samples, boxes)
    assert not bad_images(got, host_records(emu, pol, imgs, samples, boxes)), policy
    # the oracle (the reference's PIL path) on a sample of images, with the same draws
    seed_all(5)
    for i, a in enumerate(imgs):
        want = np.asarray(pil_path.PolicyTransform(pols)(PIL.Image.fromarray(a)))
        if i % 3 == 0 or a.shape[0] * a.shape[1] < 4096:
            assert np.array_equal(got.image(i).cpu().numpy(), want), (policy, i, a.shape)


@pytest.mark.parametrize("mode", ["philox", "records"])
def test_equals_the_per_size_launch_groups_of_the_chain(mode):
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float32)
    pol = chain.aug.compiled
    for sizes in (MIXED, MANY):
        x = RaggedImages.from_list(images(sizes, 11))
        if mode == "philox":
            want = chain._policy_ragged(x, None, 5, 300)
            got = engine.augment_batch(pol, x, RAW, rng=engine.make_rng(5, 300, RAW))
        else:
            recs = parity_records(pol, sizes, 9)
            want = chain._policy_ragged(x, recs, 0, 0)
            got = engine.augment_batch(pol, x, RAW, *recs)
        assert not bad_images(got, [want.image(i).cpu().numpy() for i in range(len(sizes))]), mode


@pytest.mark.parametrize("s", GR.INPUT_SIZES)
def test_parity_train_chain_from_the_ragged_launch_matches_the_digests(s):
    g = np.load(GOLDEN)
    batch = GR.ragged_inputs()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), s, torch.float32)
    x = RaggedImages.from_list(batch)
    seed_all(3)
    samples, boxes, crops, flips, jit, rgb = chain.sample_parity(len(batch), sizes=x.sizes)
    inter = engine.augment_batch(chain.aug.compiled, x, RAW, samples, boxes)
    y = engine.crop_resize(inter, s, boxes=crops)
    chain.jitter.jitter_batch(y, jit, out=y)
    zb = np.zeros((len(batch), 1), dtype=_lib.BOX_DTYPE)
    got = engine.augment_batch(chain.flip_policy, y, chain.tail, flips, zb, lighting_rgb=rgb).cpu().numpy()
    assert [G.digest(a) for a in got] == list(g["train_s%d" % s]), s


def test_same_size_batch_equals_the_uniform_launch():
    for (h, w), policy in (((375, 500), "fa_resnet50_rimagenet"), ((480, 640), "every_class"), ((224, 224), "three_ops")):
        pol = CompiledPolicy(POLICIES[policy])
        b = 24
        x = torch.from_numpy(np.stack(images([(h, w)] * b, 3))).cuda()
        r = RaggedImages(x.view(-1), np.arange(b, dtype=np.int64) * h * w * 3, [(h, w)] * b)
        rng = engine.make_rng(8, 40, RAW)
        want = engine.augment_batch(pol, x, RAW, rng=rng)
        got = engine.augment_batch(pol, r, RAW, rng=rng)
        assert not bad_images(got, list(want.cpu().numpy())), (h, w)
        recs = parity_records(pol, [(h, w)] * b, 2)
        want = engine.augment_batch(pol, x, RAW, *recs)
        got = engine.augment_batch(pol, r, RAW, *recs)
        assert not bad_images(got, list(want.cpu().numpy())), (h, w)


def test_layouts(emu):
    """odd byte offsets (the library re-aligns W % 4 == 0 inputs), unsorted and repeated descriptors, an output given as
    a RaggedImages at odd offsets, batch sizes 0 and 1"""
    pol = CompiledPolicy(_reduced())
    sizes = [(375, 500), (37, 41), (500, 375), (3, 4), (64, 64), (2, 8)]
    order = [2, 0, 2, 3, 1, 0, 4, 5, 4]
    x, imgs = odd_offset_batch(images(sizes, 5), order)
    seed, first = 3, 77
    want = host_philox(emu, pol, imgs, seed, first)
    got = engine.augment_batch(pol, x, RAW, rng=engine.make_rng(seed, first, RAW))
    assert not bad_images(got, want)
    # the given output: W % 4 == 0 images on 4-byte boundaries, the others anywhere
    offs, at = [], 0
    for a in imgs:
        at += 1 if a.shape[1] % 4 else (-at) % 4 + 4
        offs.append(at)
        at += a.size
    out = RaggedImages(torch.zeros(at + 5, dtype=torch.uint8, device="cuda"), offs, [a.shape[:2] for a in imgs])
    res = engine.augment_batch(pol, x, RAW, rng=engine.make_rng(seed, first, RAW), out=out)
    assert res is out and not bad_images(out, want)
    with pytest.raises(ValueError):
        engine.augment_batch(pol, x, RAW, rng=engine.make_rng(seed, first, RAW), out=RaggedImages.empty(sizes))
    empty = RaggedImages(torch.zeros(0, dtype=torch.uint8, device="cuda"), [], np.zeros((0, 2)))
    assert len(engine.augment_batch(pol, empty, RAW, rng=engine.make_rng(1, 0, RAW))) == 0
    one = RaggedImages.from_list(imgs[:1])
    assert not bad_images(engine.augment_batch(pol, one, RAW, rng=engine.make_rng(seed, first, RAW)), want[:1])


def test_launch_count_and_cached_tables():
    """the 40-size mixture: one resolve launch and one pixel launch per cluster size present, per two-op window; one
    more (the re-aligning copy) when some W % 4 == 0 image starts off a 4-byte boundary; one table per new size"""
    imgs = images(MANY, 1)
    x = RaggedImages.empty([a.shape[:2] for a in imgs])
    for i, a in enumerate(imgs):
        x.image(i).copy_(torch.from_numpy(a))
    n_sizes = len(set(MANY))
    assert n_sizes >= 40
    for name, n_win in (("fa_resnet50_rimagenet", 1), ("three_ops", 2)):
        pol = CompiledPolicy(POLICIES[name])
        bands = {engine_bands(h, w) for h, w in MANY}
        n0 = launches()
        engine.augment_batch(pol, x, RAW, rng=engine.make_rng(1, 0, RAW))
        n1 = launches()
        assert n1 - n0 == n_win * (1 + len(bands)) and len(bands) <= 4, (name, n1 - n0, bands)
        assert engine.cached_tables(pol)[0] == n_sizes
        engine.augment_batch(pol, x, RAW, rng=engine.make_rng(2, 0, RAW))
        assert engine.cached_tables(pol)[0] == n_sizes
        new = RaggedImages.from_list(images([(71, 73), (71, 73), (2, 3)], 2))
        engine.augment_batch(pol, new, RAW, rng=engine.make_rng(2, 0, RAW))
        assert engine.cached_tables(pol)[0] == n_sizes + 2
    # odd offsets: W % 4 == 0 images are copied first, in one more launch
    pol = CompiledPolicy(POLICIES["fa_resnet50_rimagenet"])
    y, _ = odd_offset_batch(imgs, list(range(len(imgs))))
    n0 = launches()
    engine.augment_batch(pol, y, RAW, rng=engine.make_rng(1, 0, RAW))
    assert launches() - n0 == 2 + len({engine_bands(h, w) for h, w in MANY})


def engine_bands(h, w):
    """CTAs per image of the cluster kernel (faa_core.cuh pick_bands for an output of the image's size)"""
    quads = h * ((w + 3) // 4)
    b = 1
    while b < 8 and quads // (b * 2) >= 1024 and b * 2 <= h:
        b *= 2
    return b


def test_parity_draws_consume_like_the_per_image_loop():
    aug = data.Augmentation(archive.fa_resnet50_rimagenet())
    sizes = MIXED
    imgs = images(sizes, 4)
    seed_all(6)
    want = [np.asarray(aug(PIL.Image.fromarray(a))) for a in imgs]
    after = (random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2])
    seed_all(6)
    got = aug.augment_batch(RaggedImages.from_list(imgs), parity=True)
    assert (random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2]) == after
    assert not bad_images(got, want)
    # Philox mode through the same entry
    r = aug.augment_batch(RaggedImages.from_list(imgs), seed=4, first_index=10)
    want = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)._policy_ragged(RaggedImages.from_list(imgs), None, 4, 10)
    assert not bad_images(r, [want.image(i).cpu().numpy() for i in range(len(imgs))])
