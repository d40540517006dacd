"""Test-time-augmentation batching on a CPU-only box: the replicated schedule and descriptors, the replica-major jitter
and Lighting records, the refusals of ``ImageNetChain.train_tta`` and ``GpuAugmentedLoader.tta`` before any device
work, and the loader's Philox key layout across batches and epochs (the replica launches replaced by recorders)."""
import numpy as np
import pytest
import torch

from fast_autoaugment_b200 import _lib, archive, data, engine
from fast_autoaugment_b200.engine import RaggedImages, TailSpec

THREE_OPS = [[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)]]


def test_schedule_entry_v_reads_image_v_mod_b():
    for B, K in ((1, 1), (5, 1), (3, 4), (128, 5)):
        pos = engine.tta_positions(B, K)
        assert pos.dtype == np.int64 and pos.shape == (K * B,)
        v = np.arange(K * B)
        assert np.array_equal(pos, v % B)


def test_replicated_descriptors_share_the_storage():
    sizes = [(3, 5), (7, 4), (2, 2), (7, 4)]
    n = [h * w * 3 for h, w in sizes]
    offsets = np.cumsum([0] + n[:-1]) + 1                        # packed back to back from an odd byte
    storage = torch.zeros(sum(n) + 1, dtype=torch.uint8)
    batch = RaggedImages(storage, offsets, sizes)
    rep = engine.tta_select(batch, 3)
    assert rep.storage is storage
    assert np.array_equal(rep.offsets, np.tile(offsets, 3))
    assert np.array_equal(rep.sizes, np.tile(np.array(sizes, np.int32), (3, 1)))
    for r in range(3):
        for i in range(len(sizes)):
            assert rep.image(r * len(sizes) + i).data_ptr() == batch.image(i).data_ptr()


def test_replica_records_are_those_of_the_shifted_train_calls():
    chain = data.ImageNetChain(None, 224)
    B, K, seed, first = 6, 4, 11, 300
    recs, rgb = chain._device_records_tta(B, "cpu", seed, first, K)
    assert recs.shape == (K * B, 4) and rgb.shape == (K * B, 3)
    for r in range(K):
        want_recs, want_rgb = chain._device_records(B, "cpu", seed, first + r * B)
        assert torch.equal(recs[r * B:(r + 1) * B], want_recs)
        assert torch.equal(rgb[r * B:(r + 1) * B], want_rgb)
    # replica r is not replica 0 shifted: the records differ between replicas
    assert not torch.equal(recs[:B], recs[B:2 * B])


@pytest.mark.parametrize("kw, what", [
    (dict(replicas=2, parity=True), "parity"),
    (dict(replicas=0), "positive"),
    (dict(replicas=-1), "positive"),
    (dict(replicas=1.5), "positive"),
    (dict(replicas=65536 // 4 + 1), "65535"),
])
def test_chain_refusals(kw, what):
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)
    # a CPU tensor: any device work would fail differently
    with pytest.raises(ValueError, match=what):
        chain.train_tta(torch.zeros(4, 8, 8, 3, dtype=torch.uint8), **kw)
    ragged = RaggedImages(torch.zeros(4 * 8 * 8 * 3, dtype=torch.uint8), np.arange(4) * 192, [(8, 8)] * 4)
    with pytest.raises(ValueError, match=what):
        chain.train_tta(ragged, **kw)


def test_chain_refuses_policies_longer_than_one_window():
    chain = data.ImageNetChain(THREE_OPS, 224)
    with pytest.raises(ValueError, match="at most %d ops" % _lib.MAX_FUSED_OPS):
        chain.train_tta(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), 2)
    data.ImageNetChain([THREE_OPS[0][:2]], 224).check_tta(2, 2)           # two ops pass


def test_largest_launch_passes():
    engine.check_tta(65535 // 5, 5)
    engine.check_tta(65535, 1)
    with pytest.raises(ValueError):
        engine.check_tta(65535 // 5 + 1, 5)


class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, raw, replicas, first_index):
        self.calls.append((int(raw.shape[0]), int(replicas), int(first_index)))
        return torch.zeros(replicas, raw.shape[0], 1)


def _loader(monkeypatch, n=10, batch=4, chain=None, **kw):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    ds = data.DeviceDataset(np.zeros((n, 8, 8, 3), np.uint8), list(range(n)), device="cpu")
    return data.GpuAugmentedLoader(ds, batch, archive.fa_resnet50_rimagenet(), TailSpec.imagenet(), chain=chain, **kw)


@pytest.mark.parametrize("with_chain", [False, True])
def test_loader_key_layout_across_batches_and_epochs(monkeypatch, with_chain):
    rec = _Recorder()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224) if with_chain else None
    ld = _loader(monkeypatch, n=10, batch=4, chain=chain, seed=5)
    if with_chain:
        monkeypatch.setattr(chain, "train_tta", lambda raw, K, seed, first_index: rec(raw, K, first_index))
    else:
        monkeypatch.setattr(data, "augment_tta", lambda pol, raw, tail, K, seed, first_index: rec(raw, K, first_index))
    K = 3
    labels = []
    for _ in range(2):
        for x, y in ld.tta(K):
            assert x.shape[:2] == (K, y.shape[0])
            labels.append(y.tolist())
    assert labels == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]] * 2
    assert rec.calls == [(4, 3, 0), (4, 3, 12), (2, 3, 24), (4, 3, 30), (4, 3, 42), (2, 3, 54)]
    assert ld._drawn == 2 * K * 10
    keys = [f + v for b, k, f in rec.calls for v in range(k * b)]
    assert len(keys) == len(set(keys)) == ld._drawn
    # an ordinary epoch afterwards starts past every key the replicas drew
    if with_chain:
        monkeypatch.setattr(chain, "train", lambda raw, parity, seed, first_index: rec(raw, 1, first_index)[0])
    else:
        monkeypatch.setattr(ld.aug, "augment_batch", lambda raw, tail, seed, first_index, parity: rec(raw, 1, first_index)[0])
    next(iter(ld))
    assert rec.calls[-1] == (4, 1, 60)


@pytest.mark.parametrize("kw, replicas, what", [
    (dict(parity=True), 2, "parity"),
    (dict(chain_mode="test"), 2, "test"),
    (dict(), 0, "positive"),
    (dict(batch=20000, n=20000), 4, "65535"),
])
def test_loader_refusals(monkeypatch, kw, replicas, what):
    chain_mode = kw.pop("chain_mode", None)
    n, batch = kw.pop("n", 10), kw.pop("batch", 4)
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224)
    for c in ([chain] if chain_mode else [None, chain]):
        ld = _loader(monkeypatch, n=n, batch=batch, chain=c, **({"chain_mode": chain_mode} if chain_mode else {}), **kw)
        with pytest.raises(ValueError, match=what):
            ld.tta(replicas)
        assert ld._drawn == 0


def test_loader_refuses_long_policies(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    ds = data.DeviceDataset(np.zeros((4, 8, 8, 3), np.uint8), [0] * 4, device="cpu")
    for chain in (None, data.ImageNetChain(THREE_OPS, 224)):
        ld = data.GpuAugmentedLoader(ds, 2, THREE_OPS, TailSpec.imagenet(), chain=chain)
        with pytest.raises(ValueError, match="at most %d ops" % _lib.MAX_FUSED_OPS):
            ld.tta(2)
