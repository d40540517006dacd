"""The ImageNet train chain's test-time-augmentation replicas (``ImageNetChain.train_tta``, ``augment_tta`` on a
``RaggedImages`` batch, ``GpuAugmentedLoader.tta``): every replica bit for bit against ``train`` with the shifted first
index, on a uniform 375x500 batch, a ragged batch of DESIGN.md 4.7's size mixture packed back to back (so some images
start off a 4-byte boundary) and a batch of JPEG files; at 224 and an EfficientNet size, fp32 and fp16, with and without
a policy, K = 1, 2, 5.  Also: the launch count of a call, the loader over a JPEG directory (one read per file per
epoch, no Philox key twice), and the refusals before any launch."""
import os

import numpy as np
import pytest
import torch

from imagenet_tree import baseline_file, pillow_pixels, write_tree
from test_gpu_ragged import images, odd_offset_batch

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import EncodedImages, RaggedImages, TailSpec, decode_jpeg

pytestmark = pytest.mark.gpu

RAW = TailSpec.raw_u8()
KS = (1, 2, 5)


def launches():
    torch.cuda.synchronize()
    return int(_lib.lib.faa_launch_count())


def mixture_sizes(seed, n=64, distinct=40):
    """DESIGN.md 4.7's photo shapes (375x500, 500x375, 333x500) and random sizes in [64, 1024]^2, at least
    ``distinct`` sizes in all"""
    rng = np.random.default_rng(seed)
    sizes = [(375, 500)] * 10 + [(500, 375)] * 6 + [(333, 500)] * 5
    while len(set(sizes)) < distinct or len(sizes) < n:
        sizes.append((int(rng.integers(64, 1025)), int(rng.integers(64, 1025))))
    rng.shuffle(sizes)
    return [tuple(s) for s in sizes]


def make_input(kind):
    if kind == "uniform":
        return torch.from_numpy(np.stack(images([(375, 500)] * 6, 1))).cuda()
    if kind == "ragged":
        x = RaggedImages.from_list(images(mixture_sizes(2), 3))       # back to back: no padding between images
        unaligned = [i for i, (h, w) in enumerate(x.sizes) if w % 4 == 0 and (x.storage.data_ptr() + x.offsets[i]) % 4]
        assert len(set(map(tuple, x.sizes))) >= 40 and unaligned
        return x
    files = [baseline_file(i, 3) for i in range(10)]               # 4:4:4 / 4:2:2 / 4:2:0, grayscale, restart intervals
    return EncodedImages.from_bytes(files)


@pytest.mark.parametrize("with_policy", [True, False])
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("s", [224, 260])
@pytest.mark.parametrize("kind", ["uniform", "ragged", "encoded"])
def test_replicas_equal_train_with_shifted_first_index(kind, s, dt, with_policy):
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet() if with_policy else None, s, dt)
    x = make_input(kind)
    B = len(x) if not isinstance(x, torch.Tensor) else x.shape[0]
    seed, first = 13, 1000
    want = [chain.train(x, seed=seed, first_index=first + r * B).cpu() for r in range(max(KS))]
    for K in KS:
        chain.last_status = None
        got = chain.train_tta(x, K, seed=seed, first_index=first)
        assert got.shape == (K, B, 3, s, s) and got.dtype == dt
        got = got.cpu()
        for r in range(K):
            bad = [i for i in range(B) if not torch.equal(got[r, i], want[r][i])]
            assert not bad, (kind, s, dt, with_policy, K, r, bad)
        if kind == "encoded":
            assert chain.last_status is not None and chain.last_status.cpu().tolist() == [0] * B


def test_ragged_augment_tta_equals_one_launch_per_replica():
    """repeated descriptors at odd offsets (the realigned copies are shared by the replicas) into a given output"""
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    sizes = [(375, 500), (37, 41), (500, 376), (3, 4), (64, 64), (2, 8)]
    x, imgs = odd_offset_batch(images(sizes, 5), [2, 0, 2, 3, 1, 0, 4, 5, 4])
    B, K, seed, first = len(x), 3, 4, 50
    out = RaggedImages.empty(np.tile(x.sizes, (K, 1)))
    got = engine.augment_tta(pol, x, RAW, K, seed, first, out=out)
    assert got is out and len(got) == K * B
    for r in range(K):
        want = engine.augment_batch(pol, x, RAW, rng=engine.make_rng(seed, first + r * B, RAW))
        for i in range(B):
            assert torch.equal(got.image(r * B + i), want.image(i)), (r, i)


def test_launch_count_depends_on_neither_replicas_nor_sizes():
    """an encoded batch: decode 2, the policy window's resolve + at most 4 pixel launches + at most 1 re-aligning copy,
    crop-resize 1, jitter 1, then the final flip + Lighting + Normalize call (the same call ``train`` makes, over K * B
    images; K * B * 224^2 stays under the planner's split threshold here, so it is one schedule for every K)"""
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float16)
    enc = make_input("encoded")
    B = len(enc)
    chain.train_tta(enc, 5, seed=1)                                 # every size's table exists
    counts = []
    for k, K in enumerate(KS):                                      # distinct seeds: no resolve-ahead hit
        c0 = launches()
        chain.train_tta(enc, K, seed=10 + k)
        counts.append(launches() - c0)
    assert len(set(counts)) == 1, counts
    c0 = launches()
    x, _ = decode_jpeg(enc)
    n_dec = launches() - c0
    c0 = launches()
    engine.augment_tta(chain.aug.compiled, x, RAW, 5, 30, 0)
    n_pol = launches() - c0
    y = torch.zeros(5 * B, 224, 224, 3, dtype=torch.uint8, device="cuda")
    _, rgb = chain._device_records_tta(B, y.device, 31, 0, 5)
    c0 = launches()
    engine.augment_batch(chain.flip_policy, y, chain.tail, rng=engine.make_rng(31, 0, chain.tail), lighting_rgb=rgb)
    n_final = launches() - c0
    assert n_dec == 2 and 2 <= n_pol <= 1 + 4 + 1
    assert counts[0] == n_dec + n_pol + 1 + 1 + n_final, (counts, n_dec, n_pol, n_final)
    # forty-odd sizes: still one resolve, at most four pixel launches and one copy
    many = make_input("ragged")
    engine.augment_tta(chain.aug.compiled, many, RAW, 5, 1, 0)
    for K in KS:
        c0 = launches()
        engine.augment_tta(chain.aug.compiled, many, RAW, K, 40 + K, 0)
        assert 2 <= launches() - c0 <= 1 + 4 + 1


def test_refusals_raise_before_any_launch():
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)
    long_chain = data.ImageNetChain([[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)]], 224)
    u = torch.zeros(4, 16, 16, 3, dtype=torch.uint8, device="cuda")
    huge = torch.zeros(65535 // 5 + 1, 1, 1, 3, dtype=torch.uint8, device="cuda")
    enc = make_input("encoded")
    for c, x, kw in ((chain, u, dict(replicas=2, parity=True)), (chain, u, dict(replicas=0)),
                     (chain, huge, dict(replicas=5)), (long_chain, u, dict(replicas=2)),
                     (chain, enc, dict(replicas=2, parity=True)), (chain, enc, dict(replicas=0))):
        c.last_status = None
        c0 = launches()
        with pytest.raises(ValueError):
            c.train_tta(x, **kw)
        assert launches() == c0 and c.last_status is None


def test_loader_over_a_jpeg_directory(tmp_path, monkeypatch):
    """refused files among the batches; a scan index learned in the first epoch; each file read once per epoch; replica
    r of every batch equal to ``train`` of Pillow's pixels of the batch at ``drawn + r * B``; no key drawn twice"""
    write_tree(tmp_path, 11, n_classes=3, per_class=6, n_val=1)
    samples = data.imagenet_index(str(tmp_path), "train")
    paths, targets = [p for p, _ in samples], [t for _, t in samples]
    index = data.JpegIndex.empty(data.imagenet_split_folder(str(tmp_path), "train"))
    ds = data.JpegFileDataset(paths, targets, index=index, learn=True)
    pol = archive.fa_resnet50_rimagenet()
    chain = data.ImageNetChain(pol, 224, torch.float16)
    order = list(np.random.default_rng(4).permutation(len(paths)))
    B, K, seed = 8, 3, 21
    ld = data.GpuAugmentedLoader(ds, B, pol, TailSpec.imagenet(), sampler=data.SubsetSampler(order), seed=seed,
                                 chain=chain)
    reads = []
    read = data._read_file
    monkeypatch.setattr(data, "_read_file", lambda p: reads.append(p) or read(p))
    ref = data.ImageNetChain(pol, 224, torch.float16)
    keys = []
    for epoch in range(2):
        reads.clear()
        drawn = ld._drawn
        n = 0
        for x, y in ld.tta(K):
            idx = order[n:n + B]
            n += len(idx)
            assert x.shape == (K, len(idx), 3, 224, 224) and y.cpu().tolist() == [targets[i] for i in idx]
            pix = RaggedImages.from_list(pillow_pixels([paths[i] for i in idx]))
            for r in range(K):
                assert torch.equal(x[r].cpu(), ref.train(pix, seed=seed, first_index=drawn + r * len(idx)).cpu()), \
                    (epoch, n, r)
            keys += list(range(drawn, drawn + K * len(idx)))
            drawn += K * len(idx)
        assert n == len(paths) and ld._drawn == drawn
        assert sorted(reads) == sorted(paths), epoch                  # every file once
    assert len(keys) == len(set(keys)) == 2 * K * len(paths)
    refused = {"progressive.JPEG", "cmyk.JPEG", "png_named.JPEG"}
    assert refused <= {os.path.basename(p) for p in paths}


def test_loader_without_a_chain_yields_its_own_batches_at_shifted_keys():
    """a uniform CIFAR loader (RandomCrop, flip, Cutout tail): replica r of batch k is what ``__iter__`` augments for
    batch k with first index drawn_k + r * B_k"""
    rng = np.random.default_rng(0)
    x = rng.integers(0, 256, (20, 32, 32, 3), dtype=np.uint8)
    ds = data.DeviceDataset(x, list(range(20)))
    pol = archive.fa_reduced_cifar10()
    tail = TailSpec.cifar(cutout=16, out_dtype=torch.float16)
    ld = data.GpuAugmentedLoader(ds, 8, pol, tail, seed=3)
    K, drawn = 2, 0
    for k, (xb, yb) in enumerate(ld.tta(K)):
        idx = list(range(8 * k, min(8 * k + 8, 20)))
        assert xb.shape == (K, len(idx), 3, 32, 32) and yb.cpu().tolist() == idx
        raw = ds.images[idx[0]:idx[-1] + 1]
        for r in range(K):
            want = ld.aug.augment_batch(raw, tail, seed=3, first_index=drawn + r * len(idx))
            assert torch.equal(xb[r], want), (k, r)
        drawn += K * len(idx)
    assert k == 2 and ld._drawn == drawn
