"""Ragged ImageNet batches on a CPU-only box: the packing and grouping bookkeeping of ``RaggedImages``, the C ABI's
refusals before any device work, the positional Philox sampler through the host build (tests/emu/faa_emu_ragged.cpp),
and the ragged parity sampler's consumption of the global generators against the reference's per-image transforms."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import PIL.Image
import pytest
import torch

from helpers import ROOT, emu_philox_records, seed_all

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import RaggedImages, TailSpec

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_ragged as GR  # noqa: E402
import make_golden_resize as G  # noqa: E402


def load_emu_ragged():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_ragged.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_ragged.cpp")
    core = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i = C.c_void_p, C.c_int
    lib.faa_emu_philox_at.argtypes = [vp, vp, i, i, vp, i, i, i, i, i, vp, vp, vp]
    return lib


def emu_philox_at(lib, pol, pos, h, w, tail, seed, first_index, n=None):
    """records of global samples first_index + pos[k] for h x w images, as faa_sample_philox_at draws them (pos None:
    0..n-1)"""
    oh, ow = tail.out_size if tail.out_size is not None else (h, w)
    table = np.ascontiguousarray(pol.compiled_table(h, w))
    probs = np.ascontiguousarray(pol.probs, dtype=np.float64)
    rng = engine.make_rng(seed, first_index, tail)
    n = len(pos) if pos is not None else n
    samples = np.zeros(n, dtype=_lib.SAMPLE_DTYPE)
    boxes = np.zeros((n, pol.n_op), dtype=_lib.BOX_DTYPE)
    p = None if pos is None else np.ascontiguousarray(pos, dtype=np.int32)
    assert lib.faa_emu_philox_at(table.ctypes.data, probs.ctypes.data, pol.n_sub, pol.n_op, C.addressof(rng), n, h, w,
                                 oh, ow, None if p is None else p.ctypes.data, samples.ctypes.data,
                                 boxes.ctypes.data) == 0
    return samples, boxes


@pytest.fixture(scope="module")
def emu_rg():
    return load_emu_ragged()


def rand_images(sizes, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]


# ------------------------------------------------------------------------------------------------- bookkeeping --
def test_from_list_packs_back_to_back():
    sizes = [(5, 7), (1, 1), (3, 2), (5, 7), (2, 9)]
    imgs = rand_images(sizes)
    r = RaggedImages.from_list(imgs, device="cpu")
    assert r.storage.numel() == sum(h * w * 3 for h, w in sizes)
    assert r.offsets.tolist() == [0, 105, 108, 126, 231] and r.sizes.tolist() == [list(s) for s in sizes]
    for i, a in enumerate(imgs):
        assert np.array_equal(r.image(i).numpy(), a)
    # tensors pack the same bytes
    t = RaggedImages.from_list([torch.from_numpy(a) for a in imgs], device="cpu")
    assert torch.equal(t.storage, r.storage) and np.array_equal(t.offsets, r.offsets)


def test_select_shares_the_storage():
    sizes = [(4, 6), (3, 3), (8, 2), (4, 6)]
    imgs = rand_images(sizes, 1)
    r = RaggedImages.from_list(imgs, device="cpu")
    s = r.select([3, 1, 1, 0])                       # unsorted and repeated
    assert s.storage is r.storage and len(s) == 4
    assert s.sizes.tolist() == [[4, 6], [3, 3], [3, 3], [4, 6]]
    for k, i in enumerate([3, 1, 1, 0]):
        v = s.image(k)
        assert np.array_equal(v.numpy(), imgs[i])
        assert v.data_ptr() == r.storage.data_ptr() + int(r.offsets[i])          # a view, no copy
    h, d = s.descriptors()
    assert h.dtype == _lib.IMAGE_DTYPE and h["data"].tolist() == [r.storage.data_ptr() + int(r.offsets[i])
                                                                 for i in (3, 1, 1, 0)]
    assert h["h"].tolist() == [4, 3, 3, 4] and h["w"].tolist() == [6, 3, 3, 6]
    assert np.array_equal(d.numpy().view(_lib.IMAGE_DTYPE), h)


def test_descriptors_outside_the_storage_are_refused():
    st = torch.zeros(100, dtype=torch.uint8)
    RaggedImages(st, [1], [(3, 11)])                                   # 99 bytes at offset 1: ends exactly at 100
    for off, size in (([2], [(3, 11)]), ([-1], [(1, 1)]), ([0], [(0, 4)]), ([0, 0], [(1, 1)])):
        with pytest.raises(ValueError):
            RaggedImages(st, off, size)


def test_groups_keep_batch_order():
    sizes = [(375, 500), (500, 375), (375, 500), (3, 4), (500, 375), (375, 500)]
    r = RaggedImages(torch.zeros(3, dtype=torch.uint8), np.zeros(6, np.int64), [(1, 1)] * 6)
    r.sizes = np.array(sizes, np.int32)                 # (bookkeeping only: no pixel is read)
    g = r.groups()
    assert [k for k, _ in g] == [(375, 500), (500, 375), (3, 4)]
    assert [p.tolist() for _, p in g] == [[0, 2, 5], [1, 4], [3]]
    assert sorted(np.concatenate([p for _, p in g]).tolist()) == list(range(6))


# -------------------------------------------------------------------------------------------------- C ABI --
def _ragged_call(images, batch=None, boxes=None, cfg=None, tail=None):
    h = np.zeros(max(1, len(images)), _lib.IMAGE_DTYPE)
    for i, (ptr, hh, ww) in enumerate(images):
        h[i] = (ptr, hh, ww)
    t = tail or TailSpec.raw_u8().c_struct(1, 1)
    if tail is None:
        t.out_h = t.out_w = 224
    cfg = cfg or engine.crop_cfg(224)
    return _lib.lib.faa_crop_resize_ragged(h.ctypes.data, h.ctypes.data, len(images) if batch is None else batch,
                                           C.c_void_p(64), C.byref(t), boxes, C.byref(cfg), None)


def test_abi_refusals_before_device_work():
    ok = (4096, 375, 500)
    assert _ragged_call([ok, (8192, 0, 8)]) == _lib.ERR_VALUE           # a size out of range
    assert _ragged_call([ok, (8192, 8193, 8)]) == _lib.ERR_VALUE
    assert _ragged_call([ok, (0, 20, 20)]) == _lib.ERR_VALUE            # no data
    assert _ragged_call([ok], batch=-1) == _lib.ERR_VALUE
    assert _ragged_call([ok], batch=65536) == _lib.ERR_UNSUPPORTED
    # a center crop that is empty for one image only (img_size small against its short side), in both modes
    for center in (True, False):
        cfg = engine.crop_cfg(1, center=center)
        assert _ragged_call([ok, (8192, 10, 12)], cfg=cfg) == _lib.ERR_VALUE
        assert b"image 1" in _lib.lib.faa_last_error()
    bad_std = TailSpec(None, 0, False, (0.5,) * 3, (1.0, 0.0, 1.0), 0, torch.float32).c_struct(224, 224)
    assert _ragged_call([ok], tail=bad_std) == _lib.ERR_VALUE
    h = np.zeros(1, _lib.IMAGE_DTYPE)
    t = TailSpec.raw_u8().c_struct(224, 224)
    assert _lib.lib.faa_crop_resize_ragged(None, h.ctypes.data, 1, C.c_void_p(64), C.byref(t), None,
                                           C.byref(engine.crop_cfg(224)), None) == _lib.ERR_VALUE
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    rng = engine.make_rng(1)
    assert _lib.lib.faa_sample_philox_at(pol.handle, 4, 32, 32, C.byref(t), C.byref(rng), None, None, None,
                                         None) == _lib.ERR_VALUE
    n, b = C.c_int(-1), C.c_uint64(1)
    _lib.check(_lib.lib.faa_policy_cached_tables(pol.handle, C.byref(n), C.byref(b)))
    assert (n.value, b.value) == (0, 0)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the refusal of a machine without a device")
def test_valid_ragged_call_needs_a_device():
    assert _ragged_call([(4096, 375, 500), (8192, 500, 375)]) == _lib.ERR_NO_DEVICE


# ------------------------------------------------------------------------------------ positional sampler --
@pytest.mark.parametrize("hw", [(375, 500), (3, 4), (224, 224)])
def test_positional_sampler_equals_contiguous_and_per_image(emu, emu_rg, hw):
    h, w = hw
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    raw = TailSpec.raw_u8()
    n, seed, first = 64, 11, 1000
    want = emu_philox_records(emu, pol, n, h, w, raw, seed, first)
    for got in (emu_philox_at(emu_rg, pol, np.arange(n), h, w, raw, seed, first),
                emu_philox_at(emu_rg, pol, None, h, w, raw, seed, first, n=n)):
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    pos = np.array([37, 2, 2, 900, 0, 63, 5, 4096], np.int64)
    s, b = emu_philox_at(emu_rg, pol, pos, h, w, raw, seed, first)
    for k, p in enumerate(pos):
        s1, b1 = emu_philox_records(emu, pol, 1, h, w, raw, seed, first + int(p))
        assert s[k].tobytes() == s1[0].tobytes() and b[k].tobytes() == b1[0].tobytes(), (k, p)
    assert s[1].tobytes() == s[2].tobytes()
    assert s[0].tobytes() == want[0][37].tobytes()


# ---------------------------------------------------------------------------------- ragged parity sampler --
def _ref_mods():
    try:
        from oracle import build_ref
        return build_ref.import_ref()
    except Exception:
        return None


def _states():
    return (random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2], torch.get_rng_state())


@pytest.mark.parametrize("s", GR.INPUT_SIZES)
def test_ragged_parity_sampler_consumes_like_the_reference(s):
    """ImageNetChain.sample_parity(sizes=...) leaves random / numpy.random / torch exactly where the reference's
    transform_train leaves them after the same images, one after another; every crop box lies in its own image"""
    mods = _ref_mods()
    if mods is None:
        pytest.skip("oracle/_ref is not built")
    batch = GR.ragged_inputs()
    sizes = [a.shape[:2] for a in batch]
    ref = G.reference_transforms(*mods[:2], mods[3], s)["train"]
    seed_all(3)
    for a in batch:
        ref(PIL.Image.fromarray(a))
    want = _states()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), s, torch.float32)
    seed_all(3)
    recs = chain.sample_parity(len(batch), sizes=sizes)
    got = _states()
    assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2] and torch.equal(got[3], want[3])
    for (h, w), c in zip(sizes, recs[2]):
        assert 0 <= c["x0"] <= w - c["w"] and 0 <= c["y0"] <= h - c["h"] and c["w"] > 0 and c["h"] > 0
    # a size list of one repeated size draws what the uniform call draws
    seed_all(3)
    u = chain.sample_parity(4, 375, 500)
    seed_all(3)
    r = chain.sample_parity(4, sizes=[(375, 500)] * 4)
    assert all(np.array_equal(x, y) if isinstance(x, np.ndarray) else torch.equal(x, y) for x, y in zip(u, r))


# --------------------------------------------------------------------------------------------- dataset input --
def test_imagenet_arrays_of_many_sizes(tmp_path):
    sizes = [(5, 7), (2, 3), (5, 7), (9, 1)]
    imgs = rand_images(sizes, 4)
    tr, trl, te, tel = data._load_arrays("imagenet", {"train": (imgs, [0, 1, 2, 3]), "test": (imgs[:2], [5, 6])})
    assert isinstance(tr, list) and all(np.array_equal(a, b) for a, b in zip(tr, imgs)) and trl == [0, 1, 2, 3]
    assert isinstance(te, list) and all(np.array_equal(a, b) for a, b in zip(te, imgs[:2])) and tel == [5, 6]
    packed = np.concatenate([a.reshape(-1) for a in imgs])
    for split in ("train", "test"):
        np.savez(tmp_path / ("imagenet_%s.npz" % split), data=packed, sizes=np.array(sizes), targets=np.arange(4))
    tr, trl, te, tel = data._load_arrays("imagenet", str(tmp_path))
    assert [a.shape[:2] for a in tr] == sizes and all(np.array_equal(a, b) for a, b in zip(tr, imgs))
    assert trl == [0, 1, 2, 3]
    # one size: the uniform arrays as before
    same = rand_images([(4, 4)] * 3, 5)
    tr, _, _, _ = data._load_arrays("imagenet", {"train": (same, [0, 1, 2])})
    assert isinstance(tr, np.ndarray) and tr.shape == (3, 4, 4, 3)


def test_many_sizes_without_crop_resize_are_refused():
    from fast_autoaugment_b200.conf import Config as C_
    imgs = rand_images([(5, 7), (2, 3)], 6)
    conf = C_.get()
    saved = dict(conf)
    try:
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet"})
        with pytest.raises(ValueError, match="faa_crop_resize"):
            data.get_dataloaders("imagenet", 2, {"train": (imgs, [0, 1])}, split=0.0)
    finally:
        conf.clear()
        conf.update(saved)
