"""Multi-policy test-time augmentation on a CPU-only box: the refusals of ``faa_augment_tta_policies`` /
``faa_augment_ragged_policies`` and of their Python callers before any device work, the mapping from schedule entry to
(candidate, replica, image), the host build of the multi-policy resolve step against the single-policy one, and the
loader's Philox key layout with T candidates (the launches replaced by recorders)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from test_ragged_host import emu_philox_at, load_emu_ragged

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import CompiledPolicy, RaggedImages, TailSpec

THREE_OPS = [[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)]]
ONE_OP = [[("Invert", 0.5, 0.0)], [("Rotate", 0.9, 0.3)]]
NO_DEVICE = not torch.cuda.is_available()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_rg():
    return load_emu_ragged()


@pytest.fixture(scope="module")
def emu_tp():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_tta_policies.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_tta_policies.cpp")
    core = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i = C.c_void_p, C.c_int
    lib.faa_emu_philox_policies.argtypes = [vp, vp, vp, i, i, i, vp, i, i, i, i, i, vp, vp]
    return lib


def candidates():
    """four candidates: n_sub 5, 25 and 3, two built from the same list"""
    return [CompiledPolicy(archive.fa_reduced_cifar10()[:5]), CompiledPolicy(archive.fa_reduced_cifar10()),
            CompiledPolicy(archive.arsaug_policy()[:3]), CompiledPolicy(archive.fa_reduced_cifar10()[:5])]


def handles(pols):
    return (C.c_void_p * max(len(pols), 1))(*[p.handle.value for p in pols])


def uniform_call(pols, batch=4, replicas=3, n=None, h=8, w=8):
    buf = np.zeros((max(batch, 1), h, w, 3), np.uint8)
    out = np.zeros(len(pols or [0]) * replicas * max(batch, 1) * h * w * 3 * 4 + 64, np.uint8)
    t = TailSpec.raw_u8().c_struct(h, w)
    r = engine.make_rng(1, 0, TailSpec.raw_u8())
    return _lib.lib.faa_augment_tta_policies(handles(pols) if pols is not None else None,
                                             len(pols) if n is None else n, buf.ctypes.data, out.ctypes.data, batch,
                                             replicas, h, w, C.byref(t), C.byref(r), None)


def ragged_call(pols, cand, n=None):
    B = len(cand)
    desc = np.zeros(max(B, 1), _lib.IMAGE_DTYPE)
    desc["data"], desc["h"], desc["w"] = 4096, 8, 8
    c = np.ascontiguousarray(cand, dtype=np.int32)
    r = engine.make_rng(1, 0, TailSpec.raw_u8())
    return _lib.lib.faa_augment_ragged_policies(handles(pols), len(pols) if n is None else n, desc.ctypes.data,
                                                desc.ctypes.data, c.ctypes.data, B, desc.ctypes.data, desc.ctypes.data,
                                                C.byref(r), None)


def test_abi_refusals_before_device_work():
    a, b = CompiledPolicy(archive.fa_reduced_cifar10()), CompiledPolicy(archive.arsaug_policy())
    one = CompiledPolicy(ONE_OP)
    three, three2 = CompiledPolicy(THREE_OPS), CompiledPolicy(THREE_OPS)
    big = [CompiledPolicy(archive.fa_reduced_cifar10()) for _ in range(3)]
    for call, want in (
            (lambda: uniform_call(None, n=2), _lib.ERR_VALUE),                         # null list
            (lambda: uniform_call([a], n=0), _lib.ERR_VALUE),                          # empty list
            (lambda: uniform_call([a, b, a]), _lib.ERR_VALUE),                         # repeated handle
            (lambda: uniform_call([a, one]), _lib.ERR_VALUE),                          # n_op differ
            (lambda: uniform_call([a, b], replicas=0), _lib.ERR_VALUE),
            (lambda: uniform_call([three, three2]), _lib.ERR_UNSUPPORTED),             # n_op > FAA_MAX_FUSED_OPS
            (lambda: uniform_call([three]), _lib.ERR_UNSUPPORTED),
            (lambda: uniform_call(big, batch=65535 // 15 + 1, replicas=5, h=1, w=1), _lib.ERR_UNSUPPORTED),
            (lambda: ragged_call([a, a], [0, 1]), _lib.ERR_VALUE),
            (lambda: ragged_call([a, one], [0, 1]), _lib.ERR_VALUE),
            (lambda: ragged_call([three, three2], [0, 1]), _lib.ERR_UNSUPPORTED),
            (lambda: ragged_call([a, b], [0, 2]), _lib.ERR_VALUE),                     # candidate out of range
            (lambda: ragged_call([a, b], [-1, 0]), _lib.ERR_VALUE),
            (lambda: ragged_call([a], [0, 1]), _lib.ERR_VALUE)):
        assert call() == want, _lib.lib.faa_last_error()
    # the largest call passes the checks (and reaches the device)
    if NO_DEVICE:
        assert uniform_call(big, batch=65535 // 15, replicas=5, h=1, w=1) == _lib.ERR_NO_DEVICE
        assert uniform_call([a, b]) == _lib.ERR_NO_DEVICE
        assert ragged_call([a, b], [0, 1, 1, 0]) == _lib.ERR_NO_DEVICE


@pytest.mark.parametrize("T, B, K", [(1, 1, 1), (1, 5, 3), (4, 128, 5), (8, 7, 2), (3, 1, 4)])
def test_entry_mapping(T, B, K):
    t, r, i = engine.tta_policy_entries(T, B, K)
    v = np.arange(T * K * B)
    assert t.shape == r.shape == i.shape == v.shape
    assert np.array_equal((t * K + r) * B + i, v)
    assert t.min() >= 0 and t.max() == T - 1 and r.max() == K - 1 and i.max() == B - 1
    # the image each entry reads is the one tta_select / tta_positions give for T * K replicas
    assert np.array_equal(i, engine.tta_positions(B, T * K))
    # candidate t's entries are one contiguous block of K * B, in augment_tta's own order
    for c in range(T):
        blk = slice(c * K * B, (c + 1) * K * B)
        assert (t[blk] == c).all() and np.array_equal(r[blk] * B + i[blk], np.arange(K * B))


@pytest.mark.parametrize("tail", [TailSpec.cifar(cutout=16), TailSpec.imagenet(), TailSpec.raw_u8()],
                         ids=["cifar", "imagenet", "raw"])
def test_host_resolve_equals_single_policy_resolve_per_candidate(emu_rg, emu_tp, tail):
    pols = candidates()
    T, B, K, seed, first = len(pols), 6, 3, 77, 1234
    h, w = (32, 32) if tail.out_size is not None else (40, 48)
    oh, ow = tail.out_size if tail.out_size is not None else (h, w)
    tables = [np.ascontiguousarray(p.compiled_table(h, w)) for p in pols]
    probs = [np.ascontiguousarray(p.probs, dtype=np.float64) for p in pols]
    ops_arr = (C.c_void_p * T)(*[t.ctypes.data for t in tables])
    probs_arr = (C.c_void_p * T)(*[p.ctypes.data for p in probs])
    n_sub = np.array([p.n_sub for p in pols], np.int32)
    n = T * K * B
    samples = np.zeros(n, _lib.SAMPLE_DTYPE)
    boxes = np.zeros((n, 2), _lib.BOX_DTYPE)
    rng = engine.make_rng(seed, first, tail)
    assert emu_tp.faa_emu_philox_policies(ops_arr, probs_arr, n_sub.ctypes.data, T, K * B, 2, C.addressof(rng), n, h, w,
                                          oh, ow, samples.ctypes.data, boxes.ctypes.data) == 0
    for t, pol in enumerate(pols):
        want_s, want_b = emu_philox_at(emu_rg, pol, None, h, w, tail, seed, first + t * K * B, n=K * B)
        blk = slice(t * K * B, (t + 1) * K * B)
        assert samples[blk].tobytes() == want_s.tobytes(), t
        assert boxes[blk].tobytes() == want_b.tobytes(), t
        assert samples[blk]["sub"].max() < pol.n_sub
    # candidates 0 and 3 share a policy list but not keys: their blocks differ
    assert samples[:K * B].tobytes() != samples[3 * K * B:].tobytes()


def test_python_refusals_before_device_work():
    a, b = CompiledPolicy(archive.fa_reduced_cifar10()), CompiledPolicy(archive.arsaug_policy())
    x = torch.zeros(4, 8, 8, 3, dtype=torch.uint8)                  # a CPU tensor: any device work would fail differently
    ragged = RaggedImages(torch.zeros(4 * 192, dtype=torch.uint8), np.arange(4) * 192, [(8, 8)] * 4)
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)
    for pols, K, what in (([], 2, "at least one"), ([a, a], 2, "twice"), ([a, ONE_OP], 2, "same number"),
                          ([THREE_OPS, THREE_OPS], 2, "at most 2 ops"), ([a, b], 0, "positive"),
                          ([a, b, archive.arsaug_policy()], 65535 // 12 + 1, "65535")):
        with pytest.raises(ValueError, match=what):
            engine.augment_tta_policies(pols, x, TailSpec.raw_u8(), K, 0)
        with pytest.raises(ValueError, match=what):
            engine.augment_tta_policies(pols, ragged, TailSpec.raw_u8(), K, 0)
        for batch in (x, ragged):
            with pytest.raises(ValueError, match=what):
                chain.train_tta_policies(batch, pols, K)
    with pytest.raises(ValueError, match="parity"):
        chain.train_tta_policies(x, [a, b], 2, parity=True)
    with pytest.raises(ValueError, match="raw_u8"):
        engine.augment_tta_policies([a, b], ragged, TailSpec.imagenet(), 2, 0)


def test_compile_policies_takes_lists_augmentations_and_handles():
    a = CompiledPolicy(archive.fa_reduced_cifar10())
    aug = data.Augmentation(archive.arsaug_policy())
    got = engine.compile_policies([a, aug, archive.fa_reduced_svhn()])
    assert got[0] is a and got[1] is aug.compiled
    assert isinstance(got[2], CompiledPolicy) and got[2].n_sub == len(archive.fa_reduced_svhn())


class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, raw, n_pol, replicas, first_index):
        self.calls.append((int(raw.shape[0]), n_pol, int(replicas), int(first_index)))
        return torch.zeros(n_pol, replicas, raw.shape[0], 1)


def _loader(monkeypatch, n=10, batch=4, chain=None, **kw):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    ds = data.DeviceDataset(np.zeros((n, 8, 8, 3), np.uint8), list(range(n)), device="cpu")
    return data.GpuAugmentedLoader(ds, batch, archive.fa_resnet50_rimagenet(), TailSpec.imagenet(), chain=chain, **kw)


@pytest.mark.parametrize("with_chain", [False, True])
def test_loader_key_layout_with_candidates(monkeypatch, with_chain):
    rec = _Recorder()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224) if with_chain else None
    ld = _loader(monkeypatch, n=10, batch=4, chain=chain, seed=5)
    seen = []
    if with_chain:
        def fake(raw, pols, K, seed, first_index):
            seen.append(pols)
            return rec(raw, len(pols), K, first_index)
        monkeypatch.setattr(chain, "train_tta_policies", fake)
    else:
        def fake(pols, raw, tail, K, seed, first_index):
            seen.append(pols)
            return rec(raw, len(pols), K, first_index)
        monkeypatch.setattr(data, "augment_tta_policies", fake)
    T, K = 3, 2
    pols = [archive.fa_reduced_cifar10(), CompiledPolicy(archive.arsaug_policy()), archive.fa_reduced_cifar10()]
    labels = []
    for _ in range(2):
        for x, y in ld.tta(K, policies=pols):
            assert x.shape[:3] == (T, K, y.shape[0])
            labels.append(y.tolist())
    assert labels == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]] * 2
    assert rec.calls == [(4, 3, 2, 0), (4, 3, 2, 24), (2, 3, 2, 48), (4, 3, 2, 60), (4, 3, 2, 84), (2, 3, 2, 108)]
    assert ld._drawn == 2 * T * K * 10
    keys = [f + v for b, t, k, f in rec.calls for v in range(t * k * b)]
    assert len(keys) == len(set(keys)) == ld._drawn
    # the candidates are compiled once per tta call, the given handle kept
    assert all(len(p) == T and p[1] is pols[1] for p in seen)
    assert all(p is seen[0] for p in seen[:3])


@pytest.mark.parametrize("kw, replicas, pols, what", [
    (dict(parity=True), 2, None, "parity"),
    (dict(chain_mode="test"), 2, None, "test"),
    (dict(), 0, None, "positive"),
    (dict(), 2, [], "at least one"),
    (dict(), 2, [archive.fa_reduced_cifar10(), ONE_OP], "same number"),
    (dict(), 2, [THREE_OPS, THREE_OPS], "at most 2 ops"),
    (dict(batch=8000, n=8000), 3, None, "65535"),
])
def test_loader_refusals_with_candidates(monkeypatch, kw, replicas, pols, what):
    chain_mode = kw.pop("chain_mode", None)
    n, batch = kw.pop("n", 10), kw.pop("batch", 4)
    pols = pols if pols is not None else [archive.fa_reduced_cifar10(), archive.arsaug_policy(),
                                          archive.fa_reduced_svhn()]
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)
    for c in ([chain] if chain_mode else [None, chain]):
        ld = _loader(monkeypatch, n=n, batch=batch, chain=c, **({"chain_mode": chain_mode} if chain_mode else {}), **kw)
        with pytest.raises(ValueError, match=what):
            ld.tta(replicas, policies=pols)
        assert ld._drawn == 0
