"""Multi-policy test-time augmentation (``augment_tta_policies``, ``ImageNetChain.train_tta_policies``,
``GpuAugmentedLoader.tta(K, policies=...)``): candidate t's block bit for bit against the single-policy call at
``first_index + t * K * B``, on uniform batches with CIFAR and ImageNet tails in every output type, one candidate,
candidates of different n_sub and two built from one policy list, ragged and encoded batches, and the loader over a JPEG
tree with and without a scan index.  Also the launch counts: one resolve launch and the pixel launches of one replicated
launch per policy stage, and one launch per later chain stage, whatever the number of candidates."""
import numpy as np
import pytest
import torch

from imagenet_tree import pillow_pixels, write_tree
from test_gpu_ragged import images, odd_offset_batch
from test_gpu_tta_chain import make_input, mixture_sizes

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import CompiledPolicy, RaggedImages, TailSpec

pytestmark = pytest.mark.gpu

RAW = TailSpec.raw_u8()
DTYPES = (torch.float32, torch.float16, torch.bfloat16, torch.uint8)


def launches():
    torch.cuda.synchronize()
    return int(_lib.lib.faa_launch_count())


def candidates(source=archive.fa_reduced_cifar10):
    """n_sub 7, the whole list and 3, and a fourth handle built from the first one's list"""
    return [CompiledPolicy(source()[:7]), CompiledPolicy(source()), CompiledPolicy(archive.arsaug_policy()[:3]),
            CompiledPolicy(source()[:7])]


def uniform_batch(n, h, w, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    x[::2] = (np.linspace(30, 220, w)[None, None, :, None] + rng.normal(0, 6, (len(x[::2]), h, w, 3))).clip(0, 255)
    return torch.from_numpy(x).cuda()


def check_blocks(got, pols, single, K, B):
    for t, pol in enumerate(pols):
        want = single(pol, t)
        assert torch.equal(got[t], want), t


@pytest.mark.parametrize("dt", DTYPES, ids=str)
@pytest.mark.parametrize("kind", ["cifar", "imagenet", "imagenet_split"])
def test_uniform_blocks_equal_single_policy_calls(kind, dt, monkeypatch):
    if kind == "cifar":
        tail = TailSpec.cifar(cutout=16, out_dtype=dt) if dt != torch.uint8 else \
            TailSpec((32, 32), 4, True, engine.CIFAR_MEAN, engine.CIFAR_STD, 16, dt)
        x, pols = uniform_batch(24, 32, 32, 1), candidates()
    else:
        tail = TailSpec.imagenet(out_dtype=dt)
        x, pols = uniform_batch(6, 64, 64, 2), candidates(archive.fa_resnet50_rimagenet)
        if kind == "imagenet_split":                                # the split schedule (mid + light kernels)
            monkeypatch.setenv("FAA_SPLIT_MIN", "0")
    B, K, seed, first = x.shape[0], 3, 9, 500
    got = engine.augment_tta_policies(pols, x, tail, K, seed, first)
    assert got.shape[:3] == (len(pols), K, B) and got.dtype == dt
    check_blocks(got, pols, lambda p, t: engine.augment_tta(p, x, tail, K, seed, first + t * K * B), K, B)
    # candidates 0 and 3 share a policy list, not keys
    assert not torch.equal(got[0], got[3])


def test_one_candidate_is_augment_tta():
    tail = TailSpec.cifar(cutout=16)
    x, pol = uniform_batch(16, 32, 32, 3), CompiledPolicy(archive.fa_reduced_cifar10())
    K, seed = 4, 5
    c0 = launches()
    want = engine.augment_tta(pol, x, tail, K, seed, 100)
    n_single = launches() - c0
    c0 = launches()
    got = engine.augment_tta_policies([pol], x, tail, K, seed + 1, 100)
    n_multi = launches() - c0
    assert n_multi == n_single
    assert torch.equal(engine.augment_tta_policies([pol], x, tail, K, seed, 100)[0], want)
    assert got.shape == (1,) + tuple(want.shape)


@pytest.mark.parametrize("split", [False, True])
def test_uniform_launch_count_does_not_depend_on_candidates(split, monkeypatch):
    """one resolve launch and the pixel launches of one replicated launch: resolve + cluster kernel for CIFAR images
    (where T single-policy calls make T self-resolving launches), resolve + two or three pixel kernels split"""
    if split:
        monkeypatch.setenv("FAA_SPLIT_MIN", "0")
    tail = TailSpec.imagenet() if split else TailSpec.cifar(cutout=16)
    src = archive.fa_resnet50_rimagenet if split else archive.fa_reduced_cifar10
    x = uniform_batch(4, 64, 64, 4) if split else uniform_batch(8, 32, 32, 4)
    counts = []
    for T in (2, 4, 8):
        pols = [CompiledPolicy(src()[:5 + t]) for t in range(T)]
        engine.augment_tta_policies(pols, x, tail, 2, 1, 0)         # every table exists
        c0 = launches()
        engine.augment_tta_policies(pols, x, tail, 2, 2, 0)
        counts.append(launches() - c0)
    assert len(set(counts)) == 1, counts
    assert counts[0] in ((3, 4) if split else (2,)), counts


def test_ragged_blocks_equal_single_policy_calls():
    """repeated descriptors at odd offsets (the realigned copies are shared by the entries), ~40 sizes; the launches
    are those of one faa_augment_ragged group"""
    pols = candidates(archive.fa_resnet50_rimagenet)
    sizes = [(375, 500), (37, 41), (500, 376), (3, 4), (64, 64), (2, 8)]
    x, _ = odd_offset_batch(images(sizes, 5), [2, 0, 2, 3, 1, 0, 4, 5, 4])
    B, K, seed, first = len(x), 2, 4, 50
    got = engine.augment_tta_policies(pols, x, RAW, K, seed, first)
    assert isinstance(got, RaggedImages) and len(got) == len(pols) * K * B
    for t, pol in enumerate(pols):
        want = engine.augment_tta(pol, x, RAW, K, seed, first + t * K * B)
        for v in range(K * B):
            assert torch.equal(got.image(t * K * B + v), want.image(v)), (t, v)
    many = make_input("ragged")
    engine.augment_tta_policies(pols, many, RAW, 2, 1, 0)
    for T in (2, 4):
        c0 = launches()
        engine.augment_tta_policies(pols[:T], many, RAW, 2, 7 + T, 0)
        assert 2 <= launches() - c0 <= 1 + 4 + 1


@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("kind", ["uniform", "ragged", "encoded"])
def test_chain_blocks_equal_single_policy_train_tta(kind, dt):
    lists = [archive.fa_resnet50_rimagenet()[:9], archive.fa_resnet50_rimagenet(), archive.fa_resnet50_rimagenet()[:9]]
    chain = data.ImageNetChain(None, 224, dt)
    x = make_input(kind)
    B = len(x) if not isinstance(x, torch.Tensor) else x.shape[0]
    K, seed, first = 2, 13, 1000
    got = chain.train_tta_policies(x, lists, K, seed=seed, first_index=first)
    assert got.shape == (len(lists), K, B, 3, 224, 224) and got.dtype == dt
    if kind == "encoded":
        assert chain.last_status is not None and chain.last_status.cpu().tolist() == [0] * B
    for t, pol in enumerate(lists):
        want = data.ImageNetChain(pol, 224, dt).train_tta(x, K, seed=seed, first_index=first + t * K * B)
        assert torch.equal(got[t], want), t


def test_chain_launch_count_does_not_depend_on_candidates():
    """decode 2, the policy window's resolve + at most 4 pixel launches + at most 1 re-aligning copy, crop-resize 1,
    jitter 1, then the final flip + Lighting + Normalize call over T * K * B images"""
    chain = data.ImageNetChain(None, 224, torch.float16)
    enc = make_input("encoded")
    B, K = len(enc), 2
    lists = [archive.fa_resnet50_rimagenet()[:5 + t] for t in range(4)]
    pols = engine.compile_policies(lists)
    chain.train_tta_policies(enc, pols, K, seed=1)                  # every size's table exists
    x, _ = engine.decode_jpeg(enc)
    for T in (2, 4):
        c0 = launches()
        chain.train_tta_policies(enc, pols[:T], K, seed=10 + T)
        total = launches() - c0
        c0 = launches()
        engine.decode_jpeg(enc)
        n_dec = launches() - c0
        c0 = launches()
        engine.augment_tta_policies(pols[:T], x, RAW, K, 30 + T, 0)
        n_pol = launches() - c0
        y = torch.zeros(T * K * B, 224, 224, 3, dtype=torch.uint8, device="cuda")
        _, rgb = chain._device_records_tta(B, y.device, 31, 0, T * K)
        c0 = launches()
        engine.augment_batch(chain.flip_policy, y, chain.tail, rng=engine.make_rng(31 + T, 0, chain.tail), lighting_rgb=rgb)
        n_final = launches() - c0
        assert n_dec == 2 and 2 <= n_pol <= 1 + 4 + 1
        assert total == n_dec + n_pol + 1 + 1 + n_final, (T, total, n_dec, n_pol, n_final)


def test_refusals_raise_before_any_launch():
    chain = data.ImageNetChain(None, 224)
    a, b = CompiledPolicy(archive.fa_reduced_cifar10()), CompiledPolicy(archive.arsaug_policy())
    three = [[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)]]
    u = torch.zeros(4, 16, 16, 3, dtype=torch.uint8, device="cuda")
    enc = make_input("encoded")
    for x, pols, K in ((u, [a, a], 2), (u, [a, [[("Invert", 0.5, 0.0)]]], 2), (u, [three, three], 2), (u, [], 2),
                       (u, [a, b], 0), (u, [a, b], 65535 // 8 + 1), (enc, [a, a], 2)):
        chain.last_status = None
        c0 = launches()
        with pytest.raises(ValueError):
            chain.train_tta_policies(x, pols, K)
        with pytest.raises(ValueError):
            engine.augment_tta_policies(pols, u, RAW, K, 0)
        assert launches() == c0 and chain.last_status is None


@pytest.mark.parametrize("indexed", [False, True])
def test_loader_over_a_jpeg_directory(tmp_path, indexed):
    """one epoch: candidate t's block of every batch equal to ``train_tta`` of Pillow's pixels with policy t at
    ``drawn + t * K * B``; ``drawn`` advances by T * K * B; no key drawn twice"""
    write_tree(tmp_path, 11, n_classes=3, per_class=6, n_val=1)
    samples = data.imagenet_index(str(tmp_path), "train")
    paths, targets = [p for p, _ in samples], [t for _, t in samples]
    index = data.JpegIndex.empty(data.imagenet_split_folder(str(tmp_path), "train")) if indexed else None
    ds = data.JpegFileDataset(paths, targets, index=index, learn=indexed)
    lists = [archive.fa_resnet50_rimagenet()[:6], archive.fa_resnet50_rimagenet(), archive.fa_resnet50_rimagenet()[:6]]
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float16)
    order = list(np.random.default_rng(4).permutation(len(paths)))
    B, K, seed, T = 8, 2, 21, len(lists)
    ld = data.GpuAugmentedLoader(ds, B, archive.fa_resnet50_rimagenet(), TailSpec.imagenet(),
                                 sampler=data.SubsetSampler(order), seed=seed, chain=chain)
    refs = [data.ImageNetChain(p, 224, torch.float16) for p in lists]
    keys, n, drawn = [], 0, 0
    for x, y in ld.tta(K, policies=lists):
        idx = order[n:n + B]
        n += len(idx)
        assert x.shape == (T, K, len(idx), 3, 224, 224) and y.cpu().tolist() == [targets[i] for i in idx]
        pix = RaggedImages.from_list(pillow_pixels([paths[i] for i in idx]))
        for t in range(T):
            want = refs[t].train_tta(pix, K, seed=seed, first_index=drawn + t * K * len(idx))
            assert torch.equal(x[t], want), (n, t)
        keys += list(range(drawn, drawn + T * K * len(idx)))
        drawn += T * K * len(idx)
    assert n == len(paths) and ld._drawn == drawn
    assert len(keys) == len(set(keys)) == T * K * len(paths)


def test_loader_without_a_chain():
    """a uniform CIFAR loader (RandomCrop, flip, Cutout tail): candidate t of batch k is ``augment_tta`` of policy t at
    drawn_k + t * K * B_k"""
    rng = np.random.default_rng(0)
    x = rng.integers(0, 256, (20, 32, 32, 3), dtype=np.uint8)
    ds = data.DeviceDataset(x, list(range(20)))
    tail = TailSpec.cifar(cutout=16, out_dtype=torch.float16)
    ld = data.GpuAugmentedLoader(ds, 8, archive.fa_reduced_cifar10(), tail, seed=3)
    pols = candidates()
    T, K, drawn = len(pols), 2, 0
    for k, (xb, yb) in enumerate(ld.tta(K, policies=pols)):
        idx = list(range(8 * k, min(8 * k + 8, 20)))
        assert xb.shape == (T, K, len(idx), 3, 32, 32) and yb.cpu().tolist() == idx
        raw = ds.images[idx[0]:idx[-1] + 1]
        for t, pol in enumerate(pols):
            assert torch.equal(xb[t], engine.augment_tta(pol, raw, tail, K, 3, drawn + t * K * len(idx))), (k, t)
        drawn += T * K * len(idx)
    assert k == 2 and ld._drawn == drawn
