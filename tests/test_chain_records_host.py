"""The ImageNet train chain's ColorJitter and Lighting records on a CPU-only box.

``jitter_oracle`` applies a jitter record (``faa_jitter_t``: three factors and an order) with torchvision's PIL
functions, which call ``ImageEnhance``; it is pinned here to ``torchvision.transforms.ColorJitter`` itself, so the GPU
tests can compare ``faa_color_jitter`` with it on any record.  The device-drawn records of the Philox chain
(``ImageNetChain._device_records``) are checked with a CPU generator: their packing, their ranges and their
distributions."""
import itertools

import numpy as np
import PIL.Image
import pytest
import torch
from scipy import stats

from helpers import synth

from fast_autoaugment_b200 import _lib, data


def jitter_oracle(img_u8, rec):
    """uint8 [H,W,3] -> uint8 [H,W,3]: the ops of ``rec["order"]`` (0 brightness, 1 contrast, 2 saturation; ids of 3
    and above are absent) with the factors ``rec["alpha"]``, through torchvision's PIL path"""
    import torchvision.transforms.functional as F
    fns = (F.adjust_brightness, F.adjust_contrast, F.adjust_saturation)
    img = PIL.Image.fromarray(np.ascontiguousarray(img_u8))
    for i in rec["order"]:
        if i < 3:
            img = fns[int(i)](img, float(rec["alpha"][int(i)]))
    return np.asarray(img)


@pytest.mark.parametrize("b,c,s", [(0.4, 0.4, 0.4), (0.4, 0.0, 0.4), (1.0, 1.0, 1.0)])
def test_jitter_oracle_equals_torchvision_colorjitter(b, c, s):
    from torchvision import transforms
    tv = transforms.ColorJitter(brightness=b, contrast=c, saturation=s)
    cj = data.ColorJitter(b, c, s)
    rng = np.random.default_rng(int(10 * (b + 3 * c + 9 * s)))
    orders = set()
    for k in range(240):
        img = synth((13 + k % 5, 17 + k % 7), k % 3, rng)
        torch.manual_seed(k)
        perm = tuple(torch.randperm(4).tolist())
        torch.manual_seed(k)
        want = np.asarray(tv(PIL.Image.fromarray(img)))
        torch.manual_seed(k)
        rec = cj.sample_parity(1)[0]
        orders.add(perm)
        assert [o if o < 3 and cj.ranges[o] is not None else 3 for o in perm] == list(rec["order"]), k
        assert np.array_equal(jitter_oracle(img, rec), want), (k, rec)
    assert len(orders) == 24
    if c == 0.0:
        assert cj.ranges[1] is None


def _rebuilt_records(chain, n, seed, first_index):
    """the draws of ``_device_records`` repeated with an independent generator, packed field by field"""
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1000003 + first_index) & 0x7FFFFFFFFFFFFFFF)
    u = torch.rand(n, 4, generator=g).numpy()
    alpha = np.ones((n, 3), np.float32)
    for j, r in enumerate(chain.jitter.ranges):
        if r is not None:
            alpha[:, j] = torch.empty(n).uniform_(r[0], r[1], generator=g).numpy()
    normals = torch.randn(n, 3, generator=g)
    recs = np.zeros(n, dtype=_lib.JITTER_DTYPE)
    order = np.argsort(u, axis=1, kind="stable")
    absent = np.array([r is None for r in chain.jitter.ranges] + [True])
    recs["order"] = np.where(absent[order], 3, order)
    recs["alpha"] = alpha
    return recs, normals * float(chain.lighting.alphastd)


def _reference_lighting_rgb(alpha):
    """reference Lighting (augmentations.py:197-215) on one image's three normals: eigvec * alpha * eigval, summed"""
    eigval = torch.tensor(data._IMAGENET_PCA["eigval"])
    eigvec = torch.tensor(data._IMAGENET_PCA["eigvec"])
    return eigvec.type_as(alpha).clone().mul(alpha.view(1, 3).expand(3, 3)).mul(eigval.view(1, 3).expand(3, 3)).sum(1).squeeze()


@pytest.mark.parametrize("jitter", [(0.4, 0.4, 0.4), (0.4, 0.0, 0.4), (0.0, 0.0, 0.0)])
@pytest.mark.parametrize("seed,first_index", [(0, 0), (7, 4096), (2 ** 40 + 3, 123)])
def test_device_records_pack_the_draws(jitter, seed, first_index):
    chain = data.ImageNetChain(None, 224)
    chain.jitter = data.ColorJitter(*jitter)
    n = 300
    recs, rgb = chain._device_records(n, "cpu", seed, first_index)
    assert recs.dtype == torch.int32 and tuple(recs.shape) == (n, 4) and recs.is_contiguous()
    got = recs.numpy().view(_lib.JITTER_DTYPE).reshape(n)
    want, alpha = _rebuilt_records(chain, n, seed, first_index)
    assert got.tobytes() == want.tobytes()
    present = [r is not None for r in chain.jitter.ranges]
    for r in got:
        o = list(r["order"])
        assert sorted(o[k] for k in range(4) if o[k] != 3) == [i for i in range(3) if present[i]], o
        for i in range(3):
            if not present[i]:
                assert r["alpha"][i] == np.float32(1.0)
    for j, rg in enumerate(chain.jitter.ranges):
        if rg is not None:
            assert got["alpha"][:, j].min() >= np.float32(rg[0]) and got["alpha"][:, j].max() <= np.float32(rg[1])
    assert rgb.dtype == torch.float32 and tuple(rgb.shape) == (n, 3)
    ref = torch.stack([_reference_lighting_rgb(alpha[i]) for i in range(n)])
    assert torch.equal(rgb, ref)


def test_device_records_are_distributed_like_torchvision():
    """uniform over the 24 orders (chi-square) and factors uniform on [0.6, 1.4] (Kolmogorov-Smirnov); the seed is
    fixed, so the p-value thresholds cannot flake"""
    chain = data.ImageNetChain(None, 224)
    n = 48000
    recs, rgb = chain._device_records(n, "cpu", 11, 0)
    r = recs.numpy().view(_lib.JITTER_DTYPE).reshape(n)
    index = {p: i for i, p in enumerate(itertools.permutations(range(4)))}
    counts = np.bincount([index[tuple(int(v) for v in o)] for o in r["order"]], minlength=24)
    assert counts.min() > 0
    assert stats.chisquare(counts).pvalue > 1e-3
    a = r["alpha"].astype(np.float64)
    assert a.min() >= 0.6 - 1e-7 and a.max() <= 1.4 + 1e-7
    for j in range(3):
        assert stats.kstest(a[:, j], "uniform", args=(0.6, 0.8)).pvalue > 1e-3
    # Lighting: eigvec . (alpha * eigval), alpha ~ N(0, 0.1): the offsets' covariance
    ev = np.array(data._IMAGENET_PCA["eigvec"], np.float64)
    lam = np.array(data._IMAGENET_PCA["eigval"], np.float64)
    cov = ev @ np.diag((0.1 * lam) ** 2) @ ev.T
    emp = np.cov(rgb.numpy().astype(np.float64).T)
    assert np.allclose(emp, cov, rtol=0.05, atol=2e-6)
