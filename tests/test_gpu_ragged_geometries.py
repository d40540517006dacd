"""The ragged policy launch (``faa_augment_ragged``) at every per-image geometry its planner can choose.

tests/geometry_cases.py holds RAGGED_CASES, one image per regime of `plan_ragged` (CTAs per image, TMA staging or why
not, the octet paths, the materialisation chunk, the scratch image), and RAGGED_MIXES, the calls that put them together
so that one launch holds staged, unstaged, chunk-less and copied images and its shared memory may come from an image
other than its first.  Each image sits at its case's input and output byte offsets mod 16 inside one storage per call;
the output storage is filled with a sentinel byte first, so that an image or band no launch wrote shows up as wrong
bytes, and the bytes between images must keep it.

References (no GPU result is its own reference): every image equals the host build of the kernels at its own size
(tests/emu), and every image up to 640 px plus a sample above that equals oracle.pil_path.PolicyTransform with the same
draws.  As a check of the header contract, each image also equals a uniform uint8 launch of that image alone.  The
launch count of every call is the planner's: per two-op window, the resolve kernel, one pixel launch per cluster size
present and one re-aligning copy if some W % 4 == 0 input starts off a 4-byte boundary.
"""
import random

import numpy as np
import PIL.Image
import pytest
import torch

import geometry_cases as G
from helpers import philox_reference, reference_output, seed_all, synth
from test_gpu_fastpaths import GEO, _policies
from test_gpu_geometries import _reduced
from test_gpu_ragged import images

from fast_autoaugment_b200 import _lib, archive, engine
from fast_autoaugment_b200.engine import CompiledPolicy, RaggedImages, TailSpec
from oracle import pil_path

pytestmark = pytest.mark.gpu

RAW = TailSpec.raw_u8()
SENTINEL = 0xA5
THREE_OPS = [[("Sharpness", 1.0, 0.7), ("ShearX", 0.8, 0.6), ("Equalize", 0.9, 0.5)],
             [("Color", 1.0, 0.3), ("Cutout", 1.0, 0.4), ("TranslateY", 1.0, 0.8)],
             [("AutoContrast", 1.0, 0.5), ("Sharpness", 1.0, 0.2), ("Rotate", 1.0, 0.9)],
             [("Contrast", 1.0, 0.6), ("Posterize", 1.0, 0.5), ("Brightness", 1.0, 0.4)]]


@pytest.fixture(scope="module")
def emu_rp():
    return G.load_emu_ragged_plan()


def launches():
    torch.cuda.synchronize()
    return int(_lib.lib.faa_launch_count())


def _layout(sizes, offs):
    """byte offsets of the images in one storage: image i `offs[i]` bytes past a 16-byte boundary, 16 to 31 bytes after
    the previous one (torch allocations start on 512-byte boundaries)"""
    at, out = 0, []
    for (h, w), o in zip(sizes, offs):
        at += 16
        at += (o - at) % 16
        out.append(at)
        at += h * w * 3
    return out, at + 16


def ragged_input(imgs, offs):
    o, n = _layout([a.shape[:2] for a in imgs], offs)
    host = np.full(n, SENTINEL ^ 0xFF, np.uint8)
    for a, k in zip(imgs, o):
        host[k:k + a.size] = a.reshape(-1)
    x = RaggedImages(torch.from_numpy(host).cuda(), o, [a.shape[:2] for a in imgs])
    assert [(x.storage.data_ptr() + k) % 16 for k in o] == [f % 16 for f in offs]
    return x


def ragged_output(sizes, offs):
    o, n = _layout(sizes, offs)
    return RaggedImages(torch.full((n,), SENTINEL, dtype=torch.uint8, device="cuda"), o, sizes)


def gaps_keep_the_sentinel(out):
    mask = torch.ones(out.storage.numel(), dtype=torch.bool, device=out.device)
    for o, nb in zip(out.offsets.tolist(), out.nbytes().tolist()):
        mask[o:o + nb] = False
    return bool((out.storage[mask] == SENTINEL).all())


def expected_launches(emu_rp, sizes, in_offs, out_offs, n_op, has_sg=True):
    """kernels per two-op window, from the planner: resolve + one pixel launch per cluster size + the re-aligning copy.
    Windows before the last write a fresh 16-byte aligned intermediate, which the next window reads."""
    n, aligned = [], [0] * len(sizes)
    for base in range(0, n_op, _lib.MAX_FUSED_OPS):
        ins = in_offs if base == 0 else aligned
        outs = out_offs if base + _lib.MAX_FUSED_OPS >= n_op else aligned
        _, _, pixel, _ = G.plan_ragged(emu_rp, sizes, ins, outs, has_sg)
        n.append(1 + len(pixel) + int(any(G.ragged_copied(w, o) for (_, w), o in zip(sizes, ins))))
    return n


def mix_cases(mix):
    return [G.ragged_case(i) for i in G.RAGGED_MIXES[mix][0]]


def case_images(cases, per_case, seed):
    """`per_case` images of each case's size: a ramp with noise and noise, in turn (one array each, shared)"""
    out = []
    for ci, c in enumerate(cases):
        two = images([c.shape, c.shape], seed + ci)
        out += [two[k % 2] for k in range(per_case)]
    return out


class Records:
    """image j runs program subs[j] of `policies`; its records are sample_parity of that program alone at the image's
    size, seeded per image, so the oracle draws the same for any image alone"""

    def __init__(self, policies, subs, sizes, seed):
        self.policies, self.subs, self.seed = policies, subs, seed
        single, ss, bb = {}, [], []
        for j, (k, (h, w)) in enumerate(zip(subs, sizes)):
            if k not in single:
                single[k] = CompiledPolicy([policies[k]])
            seed_all(seed + j)
            s, b = single[k].sample_parity(1, h, w, RAW)
            s["sub"] = k
            ss.append(s)
            bb.append(b)
        self.samples, self.boxes = np.concatenate(ss), np.concatenate(bb)

    def oracle(self, j, img):
        seed_all(self.seed + j)
        return np.asarray(pil_path.PolicyTransform([self.policies[self.subs[j]]])(PIL.Image.fromarray(img)))

    def take(self, idx):
        return self.samples[idx], self.boxes[idx]


class Call:
    """one ragged call: images at their cases' offsets, the output over the sentinel, the launch count"""

    def __init__(self, emu_rp, pol, imgs, in_offs, out_offs, has_sg=True):
        self.imgs, self.in_offs, self.out_offs = imgs, in_offs, out_offs
        self.sizes = [a.shape[:2] for a in imgs]
        self.x = ragged_input(imgs, in_offs)
        self.pol = pol
        self.want_launches = expected_launches(emu_rp, self.sizes, in_offs, out_offs, pol.n_op, has_sg)

    def run(self, samples=None, boxes=None, rng=None):
        """the call; its launch count is asserted by check_launches, after the bytes"""
        out = ragged_output(self.sizes, self.out_offs)
        n0 = launches()
        got = engine.augment_batch(self.pol, self.x, RAW, samples, boxes, rng=rng, out=out)
        self.launched = launches() - n0
        assert got is out and gaps_keep_the_sentinel(out)
        return out

    def check_launches(self):
        assert self.launched == sum(self.want_launches), (self.launched, self.want_launches)


def bad(got: RaggedImages, want, idx=None):
    """images of `idx` (default all) whose bytes differ from want[i]"""
    idx = range(len(got)) if idx is None else idx
    return [i for i in idx if not np.array_equal(got.image(i).cpu().numpy(), want[i])]


def check_uniform(pol, got, x, samples=None, boxes=None, seed=None, first=None):
    """each image == a uniform uint8 launch of that image alone (an aligned copy of its input)"""
    wrong = []
    for j in range(len(got)):
        a = x.image(j).clone()[None]
        if samples is not None:
            u = engine.augment_batch(pol, a, RAW, samples[j:j + 1], boxes[j:j + 1])
        else:
            u = engine.augment_batch(pol, a, RAW, rng=engine.make_rng(seed, first + j, RAW))
        if not torch.equal(u[0], got.image(j)):
            wrong.append(j)
    return wrong


def host_by_case(emu, pol, imgs, recs, groups):
    """the host build, one emulator call per group of same-sized images"""
    want = [None] * len(imgs)
    for idx in groups:
        s, b = recs.take(idx)
        ref = reference_output(emu, pol, np.stack([imgs[j] for j in idx]), RAW, s, b).numpy()
        for k, j in enumerate(idx):
            want[j] = ref[k]
    return want


def run_records(emu, emu_rp, cases, policies, seed, oracle_sample=2, has_sg=True):
    """every case image runs every program of `policies` in one call: host build, oracle and uniform-launch checks"""
    P = len(policies)
    pol = CompiledPolicy(policies)
    imgs = case_images(cases, P, seed)
    subs = [k for _ in cases for k in range(P)]
    in_offs = [c.in_off for c in cases for _ in range(P)]
    out_offs = [c.out_off for c in cases for _ in range(P)]
    call = Call(emu_rp, pol, imgs, in_offs, out_offs, has_sg)
    recs = Records(policies, subs, call.sizes, seed)
    got = call.run(recs.samples, recs.boxes)
    groups = [list(range(ci * P, (ci + 1) * P)) for ci in range(len(cases))]
    want = host_by_case(emu, pol, imgs, recs, groups)
    errors = [("host", cases[j // P].id, policies[subs[j]]) for j in bad(got, want)]
    # the oracle: every image up to 640 px, `oracle_sample` programs of each larger case
    pick = random.Random(seed)
    for ci, c in enumerate(cases):
        ks = range(P) if not c.big else pick.sample(range(P), oracle_sample)
        for k in ks:
            j = ci * P + k
            if not np.array_equal(want[j], recs.oracle(j, imgs[j])):
                errors.append(("oracle", c.id, policies[k]))
    errors += [("uniform", cases[j // P].id, policies[subs[j]])
               for j in check_uniform(pol, got, call.x, recs.samples, recs.boxes)]
    assert not errors, (len(errors), errors[:8])
    call.check_launches()
    return call, got


# ------------------------------------------------------------------------------------------------- records --
@pytest.mark.parametrize("mix", list(G.RAGGED_MIXES))
def test_records_every_program_at_every_geometry(emu, emu_rp, mix):
    cases = mix_cases(mix)
    ids, claimed = G.RAGGED_MIXES[mix]
    # the call's pixel launches are the claimed ones (the same cluster sizes and shared memory, 28 images per case)
    P = len(_reduced())
    _, _, pixel, _ = G.plan_ragged(emu_rp, [c.shape for c in cases for _ in range(P)],
                                   [c.in_off for c in cases for _ in range(P)], [c.out_off for c in cases for _ in range(P)])
    assert [(b, f, c, s) for b, f, c, s in pixel] == [(b, f * P, c * P, s) for b, f, c, s in claimed]
    run_records(emu, emu_rp, cases, _reduced(), seed=100 + len(ids))
    torch.cuda.empty_cache()


def test_records_the_full_program_list_at_two_4_cta_geometries(emu, emu_rp):
    """128 x 160 (staged, octets, chunk) and 31 x 600 (unstaged for size, chunk) with every program of the fast-path
    list: every image against the oracle"""
    cases = [G.ragged_case("128x160"), G.ragged_case("31x600")]
    assert {c.regime[0] for c in cases} == {4}
    run_records(emu, emu_rp, cases, _policies(), seed=7)


# --------------------------------------------------------------------------------------------------- Philox --
@pytest.mark.parametrize("policy", ["fa_resnet50_rimagenet", "every_class"])
@pytest.mark.parametrize("mix", list(G.RAGGED_MIXES))
def test_philox_every_geometry_equals_the_host_build(emu, emu_rp, mix, policy):
    """decisions of global sample first_index + position at each image's own size (two images per case)"""
    cases = mix_cases(mix)
    pol = CompiledPolicy(archive.fa_resnet50_rimagenet() if policy == "fa_resnet50_rimagenet" else _reduced())
    imgs = case_images(cases, 2, seed=len(mix))
    call = Call(emu_rp, pol, imgs, [c.in_off for c in cases for _ in range(2)], [c.out_off for c in cases for _ in range(2)])
    seed, first = 29, 4321
    got = call.run(rng=engine.make_rng(seed, first, RAW))
    want = [philox_reference(emu, pol, a[None], RAW, seed, first + j).numpy()[0] for j, a in enumerate(imgs)]
    assert not bad(got, want), (mix, policy, [cases[j // 2].id for j in bad(got, want)])
    assert not check_uniform(pol, got, call.x, seed=seed, first=first)
    call.check_launches()


# ------------------------------------------------------------------------------------------- further cases --
def test_three_op_policy_changes_the_geometry_between_windows(emu, emu_rp):
    """window 2 reads the library's aligned intermediate: images unstaged for their base or copied in window 1 are
    planned as at offset 0 there; the launch count of each window is the planner's"""
    cases = mix_cases("four_cluster_sizes")
    pol = CompiledPolicy(THREE_OPS)
    imgs = case_images(cases, 2, seed=3)
    sizes = [a.shape[:2] for a in imgs]
    in_offs, out_offs = [c.in_off for c in cases for _ in range(2)], [c.out_off for c in cases for _ in range(2)]
    g1, _, _, geo1 = G.plan_ragged(emu_rp, sizes, in_offs, [0] * len(sizes))
    g2, _, _, geo2 = G.plan_ragged(emu_rp, sizes, [0] * len(sizes), out_offs)
    moved = 0
    for j, c in enumerate(c for c in cases for _ in range(2)):
        r1 = G.ragged_regime(geo1[g1[j]], c.in_off, 0)
        r2 = G.ragged_regime(geo2[g2[j]], 0, c.out_off)
        _, _, _, alone = G.plan_ragged(emu_rp, [c.shape], [0], [c.out_off])
        assert r2 == G.ragged_regime(alone[0], 0, c.out_off)
        moved += r1[1] in ("base", "base + copy") and r2[1] == "staged"
    assert moved >= 6, moved
    # records drawn for the whole three-op policy, image by image (seeded per image, as the oracle below)
    recs = []
    for j, (h, w) in enumerate(sizes):
        seed_all(12 + j)
        recs.append(pol.sample_parity(1, h, w, RAW))
    samples, boxes = np.concatenate([s for s, _ in recs]), np.concatenate([b for _, b in recs])
    call = Call(emu_rp, pol, imgs, in_offs, out_offs)
    assert len(call.want_launches) == 2 and call.want_launches[0] != call.want_launches[1], call.want_launches
    got = call.run(samples, boxes)
    want = [reference_output(emu, pol, a[None], RAW, samples[j:j + 1], boxes[j:j + 1]).numpy()[0]
            for j, a in enumerate(imgs)]
    assert not bad(got, want)
    for j, a in enumerate(imgs):
        if max(a.shape[:2]) <= 640:
            seed_all(12 + j)
            assert np.array_equal(np.asarray(pil_path.PolicyTransform(THREE_OPS)(PIL.Image.fromarray(a))), want[j]), j
    call.check_launches()
    # window by window through the C ABI: each window's launch count
    d_s = torch.from_numpy(samples.view(np.uint8).copy()).cuda()
    d_b = torch.from_numpy(boxes.view(np.uint8).reshape(-1).copy()).cuda()
    out = ragged_output(sizes, out_offs)
    cur, counts = call.x, []
    stream = torch.cuda.current_stream().cuda_stream
    for base in range(0, pol.n_op, _lib.MAX_FUSED_OPS):
        nxt = out if base + _lib.MAX_FUSED_OPS >= pol.n_op else RaggedImages.empty(sizes)
        (h_in, d_in), (h_out, d_out) = cur.descriptors(), nxt.descriptors()
        n0 = launches()
        _lib.check(_lib.lib.faa_augment_ragged(pol.handle, h_in.ctypes.data, d_in.data_ptr(), len(sizes), h_out.ctypes.data,
                                               d_out.data_ptr(), d_s.data_ptr(), d_b.data_ptr(), None, base, stream))
        counts.append(launches() - n0)
        cur = nxt
    assert not bad(out, want)
    assert counts == call.want_launches


def test_policy_without_sharpness_then_gather_runs_without_scratch_images(emu, emu_rp):
    """no program has Sharpness followed by a gather (has_sg false): W % 4 == 0 images run without a scratch image and
    without allow bit 1"""
    policies = [p for p in _reduced() if not (p[0][0] == "Sharpness" and p[1][0] in GEO)]
    assert len(policies) == len(_reduced()) - 2
    cases = mix_cases("four_cluster_sizes")
    _, _, _, geoms = G.plan_ragged(emu_rp, [c.shape for c in cases], [c.in_off for c in cases],
                                   [c.out_off for c in cases], has_sg=False)
    assert not any(g["scratch"] or g["allow"] & 2 for g in geoms)
    assert sum(c.shape[1] % 4 == 0 for c in cases) >= 10
    run_records(emu, emu_rp, cases, policies, seed=41, has_sg=False)


def test_the_order_of_the_images_does_not_change_a_byte(emu, emu_rp):
    """the same call with the images reversed (each at its own offsets) and the records permuted to match"""
    cases = mix_cases("four_cluster_sizes") + mix_cases("photos_and_limits")
    policies = _reduced()
    pol = CompiledPolicy(policies)
    imgs = case_images(cases, 2, seed=5)
    in_offs, out_offs = [c.in_off for c in cases for _ in range(2)], [c.out_off for c in cases for _ in range(2)]
    subs = [j % len(policies) for j in range(len(imgs))]
    recs = Records(policies, subs, [a.shape[:2] for a in imgs], seed=9)
    c_fwd = Call(emu_rp, pol, imgs, in_offs, out_offs)
    fwd = c_fwd.run(recs.samples, recs.boxes)
    r = list(range(len(imgs)))[::-1]
    c_rev = Call(emu_rp, pol, [imgs[j] for j in r], [in_offs[j] for j in r], [out_offs[j] for j in r])
    rev = c_rev.run(recs.samples[r], recs.boxes[r])
    diff = [j for k, j in enumerate(r) if not torch.equal(rev.image(k), fwd.image(j))]
    assert not diff, [cases[j // 2].id for j in diff]
    # ... and what the host build computes, so that two equally wrong calls cannot pass
    sizes = [a.shape[:2] for a in imgs]
    groups = [[j for j in range(len(imgs)) if sizes[j] == s] for s in dict.fromkeys(sizes)]
    assert not bad(fwd, host_by_case(emu, pol, imgs, recs, groups))
    c_fwd.check_launches()
    c_rev.check_launches()


def test_statistics_ops_over_67_million_pixels_among_small_images(emu_rp):
    """three 8192 x 8192 images (the header's limit; 8 CTAs, unstaged, no chunk) with histogram and luma-mean ops in one
    call with images of 4, 2 and 1 CTAs: uint8 against the oracle"""
    rng = np.random.default_rng(67)
    ramp, flat = synth((8192, 8192), 1, rng), synth((8192, 8192), 2, rng)
    small = [G.ragged_case(i) for i in ("128x160", "8x1024", "3x4_in1")]
    policies = [[("Equalize", 1.0, 0.7), ("Contrast", 1.0, 0.6)],
                [("AutoContrast", 1.0, 0.5), ("Contrast", 1.0, 0.3)],
                [("Brightness", 1.0, 0.95), ("Contrast", 1.0, 0.05)],   # C_LUT with a luma mean in slot 1, no chunk
                [("Contrast", 1.0, 0.2), ("Equalize", 1.0, 0.9)]]
    imgs = [ramp, flat, ramp] + case_images(small, 1, seed=2)
    cases = [G.RAGGED_HUGE] * 3 + small
    subs = [0, 1, 2, 3, 0, 2]
    call = Call(emu_rp, CompiledPolicy(policies), imgs, [c.in_off for c in cases], [c.out_off for c in cases],
                has_sg=False)
    _, _, pixel, _ = G.plan_ragged(emu_rp, call.sizes, call.in_offs, call.out_offs, has_sg=False)
    assert [b for b, _, _, _ in pixel] == [8, 4, 2, 1]
    recs = Records(policies, subs, call.sizes, seed=67)
    got = call.run(recs.samples, recs.boxes)
    wrong = [j for j in range(len(imgs)) if not np.array_equal(got.image(j).cpu().numpy(), recs.oracle(j, imgs[j]))]
    assert not wrong, wrong
    call.check_launches()
    del got, call
    torch.cuda.empty_cache()
