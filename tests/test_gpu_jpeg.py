"""The JPEG decoder on the device (``EncodedImages`` / ``decode_jpeg``, C ABI ``faa_jpeg_decode``): the whole file grid
of tests/jpeg_cases.py decoded as ragged batches that mix sizes, subsamplings, grayscale and restart intervals, against
Pillow and the host build, into sentinel-filled storage at every offset mod 16; a b512 batch of photo-sized files; a
truncated file among valid ones; the launch count, with progressive files too; and the ImageNet loaders and chains
over JPEG bytes against the same over Pillow-decoded pixels."""
import numpy as np
import pytest
import torch

import jpeg_progressive_cases as jp
from helpers import seed_all
from jpeg_cases import GRID, content, emu_decode, encode, load_emu_jpeg, make, pillow

from fast_autoaugment_b200 import _lib, archive, data
from fast_autoaugment_b200.engine import EncodedImages, RaggedImages, decode_jpeg

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


def launches():
    torch.cuda.synchronize()
    return _lib.lib.faa_launch_count()


def sentinel_out(sizes, device="cuda"):
    """RaggedImages whose image i starts at byte offset i mod 16 of a sentinel-filled storage, with gaps between them"""
    offs, at = [], 0
    for i, (h, w) in enumerate(sizes):
        at = (at + 15) // 16 * 16 + 16 + i % 16
        offs.append(at)
        at += int(h) * int(w) * 3
    storage = torch.full((at + 32,), SENTINEL, dtype=torch.uint8, device=device)
    return RaggedImages(storage, np.array(offs, np.int64), np.asarray(sizes, np.int32).reshape(-1, 2))


def untouched_outside(out):
    host = out.storage.cpu().numpy()
    mask = np.ones(host.size, bool)
    for o, n in zip(out.offsets, out.nbytes()):
        mask[o:o + n] = False
    return bool((host[mask] == SENTINEL).all())


def _batches(n_per=48):
    rng = np.random.default_rng(5)
    order = rng.permutation(len(GRID))
    return [[GRID[int(i)] for i in order[k:k + n_per]] for k in range(0, len(order), n_per)]


BATCHES = _batches()


@pytest.fixture(scope="module")
def emu_jpeg():
    return load_emu_jpeg()


@pytest.mark.parametrize("k", range(len(BATCHES)))
def test_grid_in_ragged_batches_equals_pillow_and_host(emu_jpeg, k):
    cases = BATCHES[k]
    files, wants = zip(*[make(c) for c in cases])
    enc = EncodedImages.from_bytes(files)
    out = sentinel_out(enc.sizes)
    got, status = decode_jpeg(enc, out)
    assert got is out
    assert status.cpu().tolist() == [0] * len(cases)
    for i, (c, f, want) in enumerate(zip(cases, files, wants)):
        img = out.image(i).cpu().numpy()
        assert np.array_equal(img, want), c[0]
        if c[1] * c[2] <= 640 * 480:
            assert np.array_equal(img, emu_decode(emu_jpeg, f)[2]), c[0]
    assert untouched_outside(out)


def test_b512_photo_batch_equals_pillow():
    files = [encode(content("photo", 375, 500, i), quality=90, subsampling=2) for i in range(512)]
    enc = EncodedImages.from_bytes(files)
    out, status = decode_jpeg(enc)
    assert int(status.abs().sum()) == 0
    host = out.storage.cpu().numpy()
    for i, f in enumerate(files):
        o = int(out.offsets[i])
        assert np.array_equal(host[o:o + 375 * 500 * 3].reshape(375, 500, 3), pillow(f)), i


def test_truncated_scan_among_valid_images():
    files = [encode(content("photo", 120 + 8 * i, 90 + 4 * i, i), quality=85, subsampling=i % 3) for i in range(6)]
    enc_ok = EncodedImages.from_bytes(files)
    hdr = enc_ok.headers[3]
    cut = int(hdr["scan_off"]) + int(hdr["scan_len"]) // 2
    bad = list(files)
    bad[3] = files[3][:cut]
    enc = EncodedImages.from_bytes(bad)
    out = sentinel_out(enc.sizes)
    _, status = decode_jpeg(enc, out)
    st = status.cpu().tolist()
    assert st[3] & _lib.JPEG_TRUNCATED and [s for i, s in enumerate(st) if i != 3] == [0] * 5
    for i, f in enumerate(files):
        if i != 3:
            assert np.array_equal(out.image(i).cpu().numpy(), pillow(f)), i
    assert untouched_outside(out)


def test_each_call_is_two_launches():
    files = [encode(content("photo", 64 + 16 * i, 48 + 8 * i, i), quality=80, subsampling=2, restart_marker_blocks=i)
             for i in range(4)]
    enc = EncodedImages.from_bytes(files)
    out = RaggedImages.empty(enc.sizes)
    decode_jpeg(enc, out)
    c0 = launches()
    decode_jpeg(enc, out)
    assert launches() - c0 == 2
    c0 = launches()
    decode_jpeg(enc.select([2, 0]))
    assert launches() - c0 == 2
    # progressive files: two launches for a batch of them, three for one that mixes them with baseline files
    prog = [jp.encode(content("photo", 64 + 16 * i, 48 + 8 * i, i), progressive=True, quality=80, subsampling=2)
            for i in range(3)]
    for batch, n in ((prog, 2), (files[:2] + prog + files[2:], 3)):
        e = EncodedImages.from_bytes(batch, progressive=True)
        out = RaggedImages.empty(e.sizes)
        decode_jpeg(e, out)
        c0 = launches()
        decode_jpeg(e, out)
        assert launches() - c0 == n


def test_from_bytes_names_every_refused_file():
    import io
    import PIL.Image
    good = encode(content("photo", 32, 32, 0), quality=80)
    prog = encode(content("photo", 32, 32, 1), quality=80, progressive=True)
    bio = io.BytesIO()
    PIL.Image.fromarray(content("photo", 32, 32, 2)).convert("CMYK").save(bio, "JPEG")
    with pytest.raises(ValueError, match=r"1: unsupported JPEG: progressive.*3: unsupported JPEG: 4 components"):
        EncodedImages.from_bytes([good, prog, good, bio.getvalue()])


MIXED = [(180, 240), (240, 180), (256, 256), (150, 333), (333, 150)]


def _dataset(n, seed, q):
    imgs = [content("photo", *MIXED[(i + seed) % len(MIXED)], seed * 100 + i) for i in range(n)]
    files = [encode(a, quality=q, subsampling=i % 3) if i % 4 else encode(a, quality=q, gray=True) for i, a in enumerate(imgs)]
    return files, [pillow(f) for f in files]


def test_loaders_over_jpeg_bytes_equal_loaders_over_decoded_pixels():
    from fast_autoaugment_b200.conf import Config as C_
    n, b = 12, 4
    tr_f, tr_px = _dataset(n, 1, 88)
    te_f, te_px = _dataset(6, 2, 75)
    conf = C_.get()
    saved = dict(conf)
    try:
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "faa_parity": True,
                     "model": {"type": "resnet50"}})
        got = data.get_dataloaders("imagenet", b, {"train": (tr_f, list(range(n))), "test": (te_f, list(range(6)))},
                                   split=0.0)
        want = data.get_dataloaders("imagenet", b, {"train": (tr_px, list(range(n))), "test": (te_px, list(range(6)))},
                                    split=0.0)
        assert isinstance(got[1].dataset, data.EncodedDeviceDataset)
        for which in (1, 3):                                   # train, test
            seed_all(11)
            a = [(x.cpu(), y.cpu()) for x, y in got[which]]
            seed_all(11)
            w = [(x.cpu(), y.cpu()) for x, y in want[which]]
            assert len(a) == len(w) and len(a) > 0
            for (xa, ya), (xw, yw) in zip(a, w):
                assert torch.equal(ya, yw) and torch.equal(xa, xw), which
    finally:
        conf.clear()
        conf.update(saved)


def test_chain_test_on_encoded_images():
    files, px = _dataset(7, 3, 90)
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float32)
    enc = EncodedImages.from_bytes(files)
    got = chain.test(enc)
    assert chain.last_status.cpu().tolist() == [0] * 7
    assert torch.equal(got, chain.test(RaggedImages.from_list(px)))
    sel = enc.select([4, 1, 1])
    assert torch.equal(chain.test(sel), chain.test(RaggedImages.from_list([px[4], px[1], px[1]])))
