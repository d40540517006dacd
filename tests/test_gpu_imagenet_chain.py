"""The kernels behind the crop in the ImageNet train step, at every EfficientNet input size, against plain references:

* ``faa_color_jitter`` (ColorJitter) against ``jitter_oracle`` (torchvision's PIL path, pinned to
  ``transforms.ColorJitter`` in test_chain_records_host.py), out of place and in place, bit for bit;
* Lighting through the pixel kernels (per-image normalisation tables) against the host build's uint8 result followed
  by torch's fp32 ``((u / 255 + rgb) - mean) / std``;
* the Philox train chain ``ImageNetChain.train`` end to end against a host reference assembled from those pieces, and
  the loader that runs it;
* the parity chains at 380 and 600 against digests of the reference's own transforms;
* the standalone Mixup kernels (``mixup_resolved``, ``faa_mix_u8``) against torch's fp32 expression.
fp16 / bf16 outputs must equal the fp32 reference rounded once."""
import itertools
import os
import sys

import numpy as np
import PIL.Image
import pytest
import torch

import resize_model as M
from helpers import ROOT, emu_philox_records, philox_reference, reference_output, seed_all, synth, synth_batch
from test_chain_records_host import jitter_oracle
from test_crop_resize_host import emu_philox_boxes, load_emu_resize

from fast_autoaugment_b200 import _lib, archive, data
from fast_autoaugment_b200.aug_mixup import mixup_resolved
from fast_autoaugment_b200.distributed import mix_augmented
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, TailSpec, augment_batch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_resize as G  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_resize.npz")
EFFNET = (224, 240, 260, 300, 380, 456, 528, 600)
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
SPLITS = (None, "0", "1000000000000")          # planner default, two-kernel split, cluster kernel alone


@pytest.fixture(scope="module")
def emu_rs():
    return load_emu_resize()


def norm_f32(u8_hwc):
    """ToTensor + Normalize in torch fp32 of uint8 [B,H,W,3] -> [B,3,H,W]"""
    x = torch.from_numpy(np.ascontiguousarray(u8_hwc)).permute(0, 3, 1, 2).float() / 255.0
    m = torch.tensor(IMAGENET_MEAN, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(IMAGENET_STD, dtype=torch.float32).view(1, 3, 1, 1)
    return (x - m) / s


def launches():
    torch.cuda.synchronize()
    return _lib.lib.faa_launch_count()


# ------------------------------------------------------------------------------------------------- ColorJitter --
def _rec(order, alpha):
    r = np.zeros((), _lib.JITTER_DTYPE)
    r["order"] = order
    r["alpha"] = np.asarray(alpha, np.float32)
    return r


EDGE_FACTORS = (0.0, 0.6, 1.0, 1.4, float(np.nextafter(np.float32(1), np.float32(0))),
                float(np.nextafter(np.float32(1), np.float32(2))), 2.0)


def jitter_records():
    """every order of torch.randperm(4); every factor edge for each op alone and inside a full order; absent ops"""
    rng = np.random.default_rng(5)
    recs = [_rec(p, rng.uniform(0.6, 1.4, 3)) for p in itertools.permutations(range(4))]
    for i in range(3):
        for f in EDGE_FACTORS:
            a = rng.uniform(0.6, 1.4, 3)
            a[i] = f
            recs.append(_rec((i, 3, 3, 3), a))
            recs.append(_rec((i, (i + 1) % 3, 3, (i + 2) % 3), a))
    for order in ((0, 3, 3, 2), (3, 1, 0, 3), (3, 3, 2, 3), (1, 3, 2, 3), (3, 3, 3, 1), (2, 0, 3, 3)):
        recs.append(_rec(order, rng.uniform(0.6, 1.4, 3)))
    recs += [_rec((3, 3, 3, 3), (0.5, 1.5, 0.0)), _rec((3, 3, 3, 3), (1.0, 1.0, 1.0))]
    return np.stack(recs)


def half_gray(h, w, k, shift):
    """gray k on the first npx // 2 + shift pixels (raster order), k + 1 on the rest: mean luma k + 1/2 exactly
    (shift 0, even npx) or within 1/npx of it"""
    n = h * w
    v = np.full(n, k + 1, np.uint8)
    v[:max(0, min(n, n // 2 + shift))] = k
    return np.repeat(v, 3).reshape(h, w, 3)


def jitter_images(recs, h, w, seed):
    """a synth image per record; records that start with contrast get the half-gray images, whose contrast mean is
    a tie (or one pixel off it)"""
    rng = np.random.default_rng(seed)
    out = []
    for i, r in enumerate(recs):
        if r["order"][0] == 1:
            out.append(half_gray(h, w, int(rng.integers(0, 255)), (0, -1, 1)[i % 3]))
        else:
            out.append(synth((h, w), i % 3, rng))
    return np.stack(out)


@pytest.mark.parametrize("shape", [(s, s) for s in EFFNET] + [(1, 1), (3, 5), (333, 500), (375, 500)])
def test_color_jitter_equals_pil_oracle(shape):
    h, w = shape
    recs = jitter_records()
    batch = jitter_images(recs, h, w, seed=h * 1000 + w)
    want = np.stack([jitter_oracle(a, r) for a, r in zip(batch, recs)])
    cj = data.ColorJitter()
    x = torch.from_numpy(batch).cuda()
    got = cj.jitter_batch(x, recs).cpu().numpy()
    bad = [i for i in range(len(recs)) if not np.array_equal(got[i], want[i])]
    assert not bad, (shape, "out of place", recs[bad[:4]])
    y = x.clone()
    cj.jitter_batch(y, recs, out=y)                     # in place, as the train chain calls it
    got = y.cpu().numpy()
    bad = [i for i in range(len(recs)) if not np.array_equal(got[i], want[i])]
    assert not bad, (shape, "in place", recs[bad[:4]])
    assert torch.equal(x.cpu(), torch.from_numpy(batch))     # out of place left the input alone


def test_color_jitter_contrast_mean_above_32_bits():
    """an 8192 x 8192 ramp: its luma sum is above 2^32, so the contrast mean needs the 64-bit reduction"""
    s = 8192
    ramp = ((np.arange(s)[:, None] + np.arange(s)[None, :]) * 255 // (2 * s - 2)).astype(np.uint8)
    img = np.ascontiguousarray(np.stack([ramp, ramp[::-1], ramp.T], -1))
    assert int(img.astype(np.int64).sum()) > 2 ** 33
    recs = np.stack([_rec((1, 0, 2, 3), (1.3, 0.7, 1.2)), _rec((0, 2, 3, 1), (0.8, 1.35, 0.65))])
    x = torch.from_numpy(img[None]).cuda()
    for r in recs:
        got = data.ColorJitter().jitter_batch(x, r[None]).cpu().numpy()[0]
        assert np.array_equal(got, jitter_oracle(img, r)), r
    del x
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- Lighting --
@pytest.mark.parametrize("s", EFFNET)
def test_lighting_through_the_pixel_kernels(emu, s):
    n = 8
    batch = synth_batch(n, (s, s), seed=s + 1)
    torch.manual_seed(s)
    rgb = data.Lighting(0.1).sample_rgb(n)
    rgb[0], rgb[1], rgb[2] = torch.tensor([1.0, 1.0, 1.0]), torch.tensor([-1.0, -1.0, -1.0]), torch.tensor([1.0, -1.0, 0.5])
    tail32 = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, 0, torch.float32)
    ident = data.ImageNetChain(None, s).flip_policy
    flips = np.zeros(n, _lib.SAMPLE_DTYPE)
    flips["flip"] = np.arange(n) & 1
    rimagenet = CompiledPolicy(archive.fa_resnet50_rimagenet())
    seed_all(s)
    smp, bx = rimagenet.sample_parity(n, s, s, tail32)
    x = torch.from_numpy(batch).cuda()
    old = os.environ.get("FAA_SPLIT_MIN")
    try:
        for name, pol, samples, boxes in (("identity", ident, flips, np.zeros((n, 1), _lib.BOX_DTYPE)),
                                          ("fa_resnet50_rimagenet", rimagenet, smp, bx)):
            want = reference_output(emu, pol, batch, tail32, samples, boxes, lighting_rgb=rgb)
            for split in SPLITS:
                if split is None:
                    os.environ.pop("FAA_SPLIT_MIN", None)
                else:
                    os.environ["FAA_SPLIT_MIN"] = split
                for dt in DTYPES:
                    tail = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
                    got = augment_batch(pol, x, tail, samples, boxes, lighting_rgb=rgb).cpu()
                    bad = [i for i in range(n) if not torch.equal(got[i], want[i].to(dt))]
                    assert not bad, (name, split, dt, bad)
    finally:
        if old is None:
            os.environ.pop("FAA_SPLIT_MIN", None)
        else:
            os.environ["FAA_SPLIT_MIN"] = old


def test_lighting_rows_must_match_the_batch():
    n = 4
    x = torch.from_numpy(synth_batch(n, (32, 32), seed=1)).cuda()
    pol = data.ImageNetChain(None, 32).flip_policy
    tail = TailSpec.imagenet(0, torch.float32)
    flips = np.zeros(n, _lib.SAMPLE_DTYPE)
    boxes = np.zeros((n, 1), _lib.BOX_DTYPE)
    augment_batch(pol, x, tail, flips, boxes, lighting_rgb=torch.zeros(n, 3))       # (the policy's tables exist)
    c0 = launches()
    for rows in (n - 1, n + 1):
        with pytest.raises(ValueError):
            augment_batch(pol, x, tail, flips, boxes, lighting_rgb=torch.zeros(rows, 3))
    # the C entry refuses too when the offsets were set for another number of images
    rgb = torch.zeros(n + 1, 3, device="cuda")
    _lib.check(_lib.lib.faa_policy_set_lighting(pol.handle, rgb.data_ptr(), n + 1))
    try:
        with pytest.raises(ValueError):
            augment_batch(pol, x, tail, flips, boxes)
    finally:
        _lib.check(_lib.lib.faa_policy_set_lighting(pol.handle, None, 0))
    assert launches() == c0


# ---------------------------------------------------------------------------------------- Philox train chain --
CHAIN_BATCH = {224: 64, 240: 48, 260: 48, 300: 32, 380: 32, 456: 24, 528: 16, 600: 16}


@pytest.mark.parametrize("s,src", [(s, (375, 500)) for s in EFFNET] + [(224, (480, 640)), (600, (480, 640))])
def test_philox_train_chain_equals_host_reference(emu, emu_rs, s, src):
    h, w = src
    n = CHAIN_BATCH[s]
    seed, first = 1000 + s, 37 * s + h
    policies = archive.fa_resnet50_rimagenet()
    batch = synth_batch(n, src, seed=s + h)
    ref_chain = data.ImageNetChain(policies, s, torch.float32)
    u8 = philox_reference(emu, CompiledPolicy(policies), batch, TailSpec.raw_u8(), seed, first).numpy()
    boxes = emu_philox_boxes(emu_rs, ref_chain.crop.cfg(seed, first), n, h, w)
    cropped = [M.crop_resize(u8[i], boxes[i], s, s) for i in range(n)]
    recs, rgb = ref_chain._device_records(n, torch.device("cuda"), seed, first)
    jit = recs.cpu().numpy().view(_lib.JITTER_DTYPE).reshape(n)
    g = torch.Generator(device="cuda")
    g.manual_seed((seed * 1000003 + first) & 0x7FFFFFFFFFFFFFFF)
    order = np.argsort(torch.rand(n, 4, device="cuda", generator=g).cpu().numpy(), axis=1, kind="stable")
    assert np.array_equal(jit["order"], order)               # the records' first draw, packed in torch.randperm's order
    jittered = np.stack([jitter_oracle(cropped[i], jit[i]) for i in range(n)])
    flips, fb = emu_philox_records(emu, ref_chain.flip_policy, n, s, s, ref_chain.tail, seed, first)
    assert 0 < int(flips["flip"].sum()) < n
    want = reference_output(emu, ref_chain.flip_policy, jittered, ref_chain.tail, flips, fb, lighting_rgb=rgb.cpu())
    x = torch.from_numpy(batch).cuda()
    for dt in (torch.float32, torch.float16):
        got = data.ImageNetChain(policies, s, dt).train(x, seed=seed, first_index=first).cpu()
        assert got.shape == (n, 3, s, s) and got.dtype == dt
        bad = [i for i in range(n) if not torch.equal(got[i], want[i].to(dt))]
        assert not bad, (s, src, dt, bad)


def test_loader_yields_the_train_chain_of_the_gathered_batch():
    """get_dataloaders(faa_crop_resize, efficientnet-b7): each batch == ImageNetChain.train of the gathered images
    with the loader's seed and the batch's first sample index"""
    from fast_autoaugment_b200.conf import Config as C
    n, b = 12, 4
    tr = synth_batch(n, (375, 500), seed=3)
    root = {"train": (tr, list(range(n))), "test": (tr[:4], list(range(4)))}       # labels = dataset indices
    conf = C.get()
    saved = dict(conf)
    try:
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "efficientnet-b7"}})
        _, train, _, _ = data.get_dataloaders("imagenet", b, root, split=0.0)
        assert train.chain.input_size == 600
        for k, (xb, yb) in enumerate(train):
            want = train.chain.train(train.dataset.images.index_select(0, yb), seed=train.seed, first_index=k * b)
            assert xb.shape == (b, 3, 600, 600) and torch.equal(xb, want), k
        assert k == n // b - 1
    finally:
        conf.clear()
        conf.update(saved)


# ------------------------------------------------------------------------------------ parity chains, 380 / 600 --
@pytest.mark.parametrize("s,h,w,n", G.EFFNET_CHAIN_CASES)
def test_parity_chains_at_efficientnet_sizes(s, h, w, n):
    """ImageNetChain(s).train(parity=True) / .test == the reference's transform_train / transform_test at input size s"""
    g = np.load(GOLDEN)
    tag = "s%d_%dx%d" % (s, h, w)
    batch = G.effnet_chain_inputs(s, h, w, n)
    assert [G.digest(a) for a in batch] == list(g["in_" + tag])
    try:
        from oracle import build_ref
        mods = build_ref.import_ref()
    except Exception:
        mods = None
    ref = G.reference_transforms(*mods[:2], mods[3], s) if mods is not None else None
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), s, torch.float32)
    x = torch.from_numpy(batch).cuda()
    for name in ("test", "train"):
        seed_all(3)
        got = (chain.train(x, parity=True) if name == "train" else chain.test(x)).cpu().numpy()
        assert got.shape == (n, 3, s, s)
        if ref is not None:
            seed_all(3)
            want = np.stack([ref[name](PIL.Image.fromarray(a)).numpy() for a in batch])
            assert float(np.abs(got - want).max()) == 0.0, (name, tag)
        assert [G.digest(a) for a in got] == list(g["%s_%s" % (name, tag)]), (name, tag)


# ------------------------------------------------------------------------------------------------------- Mixup --
def mix_reference(x, perm, lam):
    """aug_mixup.py:21 in torch fp32 on the CPU, rounded once to x's dtype"""
    xf = x.cpu().float()
    return (xf * lam + xf[perm.cpu()] * (1 - lam)).to(x.dtype)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("s", EFFNET)
def test_mixup_at_chain_shapes(s, dt):
    g = torch.Generator().manual_seed(s)
    x = torch.randn(6, 3, s, s, generator=g).mul(2.5).to(dt).cuda()
    perm = torch.randperm(6, generator=g)
    for p, lam in ((perm, 0.7311), (perm, 1.0), (perm, 0.5), (torch.arange(6), 0.6180339887)):
        assert torch.equal(mixup_resolved(x, p, lam).cpu(), mix_reference(x, p, lam)), (p, lam)
    one = x[:1].clone()
    assert torch.equal(mixup_resolved(one, torch.zeros(1, dtype=torch.int64), 0.83).cpu(),
                       mix_reference(one, torch.zeros(1, dtype=torch.int64), 0.83))


@pytest.mark.parametrize("shape,dt,offset", [((4, 3, 375, 500), torch.float16, 0),     # n_per % 8 == 4
                                             ((5, 3, 31, 33), torch.float32, 0),       # n_per % 4 == 1
                                             ((4, 3, 64, 64), torch.float16, 1),       # output 2 bytes past 16
                                             ((3, 3, 31, 33), torch.bfloat16, 0)])
def test_mixup_scalar_path(shape, dt, offset):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(*shape, generator=g).to(dt).cuda()
    b, numel = shape[0], x.numel()
    buf = torch.empty(numel + 8, dtype=dt, device="cuda")
    out = buf[offset:offset + numel].view(shape)
    assert (out.data_ptr() % 16 != 0) == bool(offset)
    perm = torch.randperm(b, generator=g)
    for lam in (0.7311, 0.5, 1.0):
        mixup_resolved(x, perm, lam, out=out)
        assert torch.equal(out.cpu(), mix_reference(x, perm, lam)), lam
    assert torch.equal(mixup_resolved(x, torch.arange(b), 0.25).cpu(), mix_reference(x, torch.arange(b), 0.25))


@pytest.mark.parametrize("s", [260, 380, 600])
def test_mix_u8_local_pool(s):
    """faa_mix_u8 with a local partner pool and each source's CutoutDefault box (clipped at the border, or empty)"""
    rng = np.random.default_rng(s)
    n, n_pool = 6, 9
    a = synth_batch(n, (s, s), seed=s)
    pool = synth_batch(n_pool, (s, s), seed=s + 1)
    part = rng.integers(0, n_pool, n).astype(np.int32)
    h = s // 6

    def boxes(k):
        out = []
        for i in range(k):
            cy, cx = int(rng.integers(0, s)), int(rng.integers(0, s))
            if i % 3 == 1:
                cy, cx = (0, s - 1) if i % 2 else (s - 2, 3)            # clipped at the border
            y0, y1, x0, x1 = max(0, cy - h), min(s, cy + h), max(0, cx - h), min(s, cx + h)
            if i % 3 == 2:
                y1 = y0                                                 # empty
            out.append((y0, y1, x0, x1))
        return np.array(out, np.int16)
    za, zp = boxes(n), boxes(n_pool)
    na, npool = norm_f32(a), norm_f32(pool)
    for i, (y0, y1, x0, x1) in enumerate(za):
        na[i, :, y0:y1, x0:x1] = 0
    for i, (y0, y1, x0, x1) in enumerate(zp):
        npool[i, :, y0:y1, x0:x1] = 0
    pol = data.ImageNetChain(None, s).flip_policy
    d_a, d_pool = torch.from_numpy(a).cuda(), torch.from_numpy(pool).cuda()
    d_part = torch.from_numpy(part).cuda()
    for dt in DTYPES:
        for lam in (0.7311, 0.5):
            tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, dt)
            got = mix_augmented(pol, d_a, d_pool, d_part, tail, lam, torch.from_numpy(za).cuda(),
                                torch.from_numpy(zp).cuda()).cpu()
            want = (na * lam + npool[torch.from_numpy(part).long()] * (1 - lam)).to(dt)
            assert torch.equal(got, want), (dt, lam)


def test_mixup_refuses_overlapping_out_and_huge_batches():
    """refused before anything is launched; the racing in-place launch itself is never run"""
    x = torch.randn(8, 3, 4, 4, device="cuda")
    perm = torch.randperm(8)
    buf = torch.randn(9 * 48, device="cuda")
    c0 = launches()
    with pytest.raises(ValueError):
        mixup_resolved(x, perm, 0.7, out=x)
    with pytest.raises(ValueError):                          # shifted by one sample: partial overlap
        mixup_resolved(buf[:8 * 48].view(8, 3, 4, 4), perm, 0.7, out=buf[48:].view(8, 3, 4, 4))
    with pytest.raises(ValueError):                          # the last element of out is the first of data
        mixup_resolved(buf[48:96].view(1, 3, 4, 4), torch.zeros(1, dtype=torch.int64), 0.7, out=buf[1:49].view(1, 3, 4, 4))
    with pytest.raises(_lib.FaaRuntimeError):
        mixup_resolved(torch.zeros(65536, 2, device="cuda"), torch.arange(65536), 0.5)
    assert launches() == c0
    # touching but disjoint buffers still mix
    data_, out = buf[:4 * 48].view(4, 3, 4, 4), buf[4 * 48:8 * 48].view(4, 3, 4, 4)
    p4 = torch.randperm(4)
    want = mix_reference(data_, p4, 0.7)
    mixup_resolved(data_, p4, 0.7, out=out)
    assert torch.equal(out.cpu(), want)
