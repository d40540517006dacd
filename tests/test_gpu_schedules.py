"""Call sequences of the launch planner against the host reference, bit for bit.

The planner (`augment_common` and the launch functions in csrc/faa_cabi.cu) is a state machine that spans calls: the
resolve-ahead speculation, two program slots with completion counters, one scratch image per slot, the ticket word, the
overlap test between consecutive calls and buffers that grow mid-sequence.  Every scenario here issues its calls on ONE
policy handle back to back, without a synchronize between them (outputs a later call overwrites are cloned by a
stream-ordered copy first), then synchronizes once and compares every image of every call with
helpers.philox_reference / reference_output - decisions from the emulator's Philox sampler, pixels from tests/emu,
the exact normalisation table: no GPU result is used as its own reference.

Each call also asserts the number of kernel launches the planner issues for it (`faa_launch_count`), so a scenario
cannot quietly run another schedule than the one it claims.  At the sizes used here (the split threshold is 4 Mpixels
per launch):
* chained, split (224 b >= 96): hit 3 = resolve-ahead + mid + light, miss 4 (+ the resolve of this batch);
* chained, split with the cluster kernel (380: no octet paths): hit 4, miss 5;
* chained, one pixel kernel (224 b64): hit 2, miss 3;
* self-resolving (CIFAR 32x32): 1;
* event schedule: resolved records, split 3 (resolve + light + mid), one pixel kernel 2; fused Mixup 2; uint8 output of
  one pixel kernel with resolve-ahead: miss 3, hit 2 (resolve-ahead on the side stream + pixel kernel);
* Lighting: +1 (per-image normalisation tables);
* faa_augment_host: 2 per chunk, 8 chunks from 64 images.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import philox_reference, reference_output, synth_batch

from fast_autoaugment_b200 import _lib, archive
from fast_autoaugment_b200.engine import (IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, FusedAugmenter, TailSpec, augment_batch,
                                          augment_tta, make_rng)

pytestmark = pytest.mark.gpu

H = W = 224
FP16 = TailSpec.imagenet(0, torch.float16)
FP32 = TailSpec.imagenet(0, torch.float32)
BF16_CUTOUT = TailSpec.imagenet(16, torch.bfloat16)
U8 = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, 0, torch.uint8)      # the augment stage of config 4


def _pol():
    return CompiledPolicy(archive.fa_resnet50_rimagenet())


def _launches():
    return int(_lib.lib.faa_launch_count())


def _inputs(n, b, seed, shape=(H, W)):
    """n different batches: host arrays (for the reference) and device copies"""
    xs = [synth_batch(b, shape, seed=seed + k) for k in range(n)]
    return xs, [torch.from_numpy(x).cuda() for x in xs]


def _first_bad(got, want):
    return [i for i in range(got.shape[0]) if not torch.equal(got[i], want[i])][:8]


class Sequence:
    """Calls on one handle, issued back to back; `check` synchronizes once and compares."""

    def __init__(self, emu, pol):
        self.emu, self.pol, self.calls = emu, pol, []

    def call(self, name, launches, fn, ref, clone=True, stream=None):
        """fn() issues the call and returns its output; ref() returns the host reference (run after the sequence)."""
        stream = stream or torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            n0 = _launches()
            out = fn()
            got = _launches() - n0
            if clone:                           # stream-ordered copy: later calls may overwrite `out`
                out = out.clone()
        self.calls.append((name, launches, got, out, ref))

    def philox(self, name, launches, aug, x, xh, out, first_index, stream=None):
        """a FusedAugmenter call (on the current stream, or `stream`) and its reference"""
        seed, tail = aug.rng.seed, aug.tail
        self.call(name, launches, lambda: aug(x, out, first_index),
                  lambda: philox_reference(self.emu, self.pol, xh, tail, seed, first_index), stream=stream)

    def check(self):
        torch.cuda.synchronize()
        wrong_launches = [(name, want, got) for name, want, got, _, _ in self.calls if want != got]
        wrong_values = []
        for name, _, _, out, ref in self.calls:
            got, want = out.cpu(), ref()
            assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
            bad = _first_bad(got, want)
            if bad:
                wrong_values.append((name, bad))
        assert not wrong_values and not wrong_launches, {"wrong values (call, first images)": wrong_values,
                                                         "wrong launch counts (call, expected, launched)": wrong_launches}


class _Counting:
    """FusedAugmenter wrapper that records the launches of every call (bench._Workload calls it directly)"""

    def __init__(self, aug):
        self.aug, self.launches = aug, []

    def _count(self, fn, *a, **k):
        n0 = _launches()
        r = fn(*a, **k)
        self.launches.append(_launches() - n0)
        return r

    def __call__(self, *a, **k):
        return self._count(self.aug, *a, **k)

    def plan_many(self, *a, **k):
        return self.aug.plan_many(*a, **k)

    def run_many(self, *a, **k):
        return self._count(self.aug.run_many, *a, **k)


@pytest.mark.parametrize("name,rank,world,hit,miss", [("imagenet224_b512", 0, 1, 3, 4), ("imagenet224_b512", 1, 2, 3, 4),
                                                      ("effnetb4_380_b256", 0, 1, 4, 5), ("effnetb4_380_b256", 1, 2, 4, 5),
                                                      ("cifar32_b512", 0, 1, 1, 1), ("cifar32_b512", 1, 2, 1, 1)])
def test_bench_loop_matches_reference(emu, name, rank, world, hit, miss):
    """a. bench.py's own loop (overlap_calls=True, warm-up calls, then run_many) with four DIFFERENT input sets: the four
    output sets hold steps (i * world + rank) * B of the last four steps"""
    import bench
    wl = bench._Workload(name, 3, rank, world)
    xs = [synth_batch(wl.B, (wl.H, wl.W), seed=40 + k) for k in range(wl.NSETS)]
    for k in range(wl.NSETS):
        wl.ins[k].copy_(torch.from_numpy(xs[k]))
    torch.cuda.synchronize()
    wl.fused = _Counting(wl.fused)
    barriers = []

    def barrier():                              # bench's barrier, but a synchronize only after the last step
        barriers.append(1)
        if len(barriers) == 3:
            torch.cuda.synchronize()

    warmup, steps = 3, 5
    wl.timed(steps, warmup, barrier)
    torch.cuda.synchronize()
    # the first call misses; with world 2 the second as well (the stride 2B is learnt from it); run_many only hits
    want = [miss, miss if world > 1 else hit, hit, steps * hit]
    assert wl.fused.launches == want, (wl.fused.launches, want)
    n = warmup + steps
    for i in range(n - wl.NSETS, n):
        ref = philox_reference(emu, wl.pol, xs[i % wl.NSETS], wl.tail, 3, (i * world + rank) * wl.B)
        got = wl.outs[i % wl.NSETS].cpu()
        assert torch.equal(got, ref), (name, rank, world, i, _first_bad(got, ref))


def test_resolve_ahead_transitions(emu):
    """b. 224 b512 with overlap_calls=True: hits, a stride change, first_index back to 0, a repeated index, a seed change
    at the predicted index, a partial batch (512 -> 64 -> 512: split / unsplit chained schedules, the cluster kernel
    at 64), then four augmenters on the one policy alternating fp16 / fp32 / bf16 + CutoutDefault / uint8 HWC"""
    B = 512
    pol = _pol()
    seq = Sequence(emu, pol)
    xh, xd = _inputs(4, B, seed=60)
    f16 = FusedAugmenter(pol, FP16, H, W, 7, overlap_calls=True)
    out = lambda aug, b=B: aug.empty_out(b)                                              # noqa: E731
    for k, idx in enumerate((0, 512, 1024, 1536)):                                      # a run of hits
        seq.philox("hit run %d" % k, 4 if k == 0 else 3, f16, xd[k], xh[k], out(f16), idx)
    seq.philox("stride change", 4, f16, xd[0], xh[0], out(f16), 2560)
    seq.philox("new stride", 3, f16, xd[1], xh[1], out(f16), 3584)
    seq.philox("back to 0", 4, f16, xd[2], xh[2], out(f16), 0)
    seq.philox("after 0", 3, f16, xd[3], xh[3], out(f16), 512)
    seq.philox("repeated index", 4, f16, xd[0], xh[0], out(f16), 512)
    f16.rng.seed = 8                                                                    # the speculation predicted 1024
    seq.philox("seed change", 4, f16, xd[1], xh[1], out(f16), 1024)
    seq.philox("after seed change", 3, f16, xd[2], xh[2], out(f16), 1536)
    seq.philox("partial batch 64", 3, f16, xd[3][:64], xh[3][:64], out(f16, 64), 2048)
    seq.philox("full batch after partial", 4, f16, xd[0], xh[0], out(f16), 2112)
    seq.philox("hit after partial", 3, f16, xd[1], xh[1], out(f16), 2624)
    # programs do not depend on the output type: fp32 hits fp16's speculation; CutoutDefault changes the key
    f32 = FusedAugmenter(pol, FP32, H, W, 8, overlap_calls=True)
    bfc = FusedAugmenter(pol, BF16_CUTOUT, H, W, 8, overlap_calls=True)
    u8 = FusedAugmenter(pol, U8, H, W, 8, overlap_calls=True)
    idx = 3136
    for k, (aug, n) in enumerate(((f32, 3), (bfc, 4), (u8, 4), (f16, 3), (f32, 3), (bfc, 4), (u8, 4))):
        seq.philox("alternating %d %s" % (k, aug.tail.out_dtype), n, aug, xd[k % 4], xh[k % 4], out(aug), idx)
        idx += B
    seq.check()


def test_overlap_refusal(emu):
    """c. overlap_calls=True with one output buffer reused by every call, a call reading the previous call's uint8 output
    and a call writing into the previous call's input; then the default setting with one input buffer rewritten by copy_
    before every call (the GpuAugmentedLoader pattern)"""
    B = 96
    pol = _pol()
    seq = Sequence(emu, pol)
    xh, xd = _inputs(4, B, seed=70)
    u8 = FusedAugmenter(pol, U8, H, W, 5, overlap_calls=True)
    same = u8.empty_out(B)
    for k in range(3):
        seq.philox("reused output %d" % k, 4 if k == 0 else 3, u8, xd[k], xh[k], same, k * B)
    o1, o2, o3 = u8.empty_out(B), u8.empty_out(B), u8.empty_out(B)
    seq.philox("producer", 3, u8, xd[3], xh[3], o1, 3 * B)
    ref1 = lambda: philox_reference(emu, pol, xh[3], U8, 5, 3 * B).numpy()           # noqa: E731
    seq.call("reads previous output", 3, lambda: u8(o1, o2, 4 * B), lambda: philox_reference(emu, pol, ref1(), U8, 5, 4 * B))
    buf = xd[0].clone()
    seq.philox("input of the next", 3, u8, buf, xh[0], o3, 5 * B)
    seq.philox("writes previous input", 3, u8, xd[1], xh[1], buf, 6 * B)
    # default setting, a separate handle (the overlap promise belongs to the handle)
    pol2 = _pol()
    seq2 = Sequence(emu, pol2)
    f = FusedAugmenter(pol2, FP16, H, W, 6)
    staged = torch.empty_like(xd[0])
    for k in range(4):
        def call(k=k):
            staged.copy_(xd[k])
            return f(staged, f.empty_out(B), k * B)
        seq2.call("copy_ then call %d" % k, 4 if k == 0 else 3, call, lambda k=k: philox_reference(emu, pol2, xh[k], FP16, 6, k * B))
    seq.check()
    seq2.check()


def test_mixed_schedules_on_one_handle(emu):
    """d. chained, parity-mode event call, fused Mixup, TTA, Lighting (three rgb), a uint8 event call that resolves ahead
    on the side stream followed by a chained miss and hit (the side-stream resolve-ahead writes the slot the chained
    step resolves ahead into), the host-buffer entry, chained again"""
    from fast_autoaugment_b200.data import Lighting
    B = 96
    pol = _pol()
    seq = Sequence(emu, pol)
    xh, xd = _inputs(4, B, seed=80)
    f16 = FusedAugmenter(pol, FP16, H, W, 11)
    seq.philox("chained", 4, f16, xd[0], xh[0], f16.empty_out(B), 0)
    # parity-mode records (uploaded before the sequence: no synchronous copy between the calls)
    from helpers import seed_all
    seed_all(3)
    samples, boxes = pol.sample_parity(B, H, W, FP16)
    d_s = torch.from_numpy(samples.view(np.uint8).copy()).cuda()
    d_b = torch.from_numpy(boxes.view(np.uint8).copy()).cuda()
    seq.call("parity event", 3, lambda: augment_batch(pol, xd[1], FP16, d_s, d_b),
             lambda: reference_output(emu, pol, xh[1], FP16, samples, boxes))
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1))
    perm_d = perm.to(torch.int32).cuda()
    lam = 0.7
    seq.call("fused mixup", 2, lambda: augment_batch(pol, xd[2], FP32, rng=make_rng(11, 5000, FP32), partner=perm_d, lam=lam),
             lambda: philox_reference(emu, pol, xh[2], FP32, 11, 5000, partner=perm.numpy(), lam=lam))
    xt = xd[3][:32]
    seq.call("tta", 4, lambda: augment_tta(pol, xt, FP16, 3, seed=11, first_index=7000),
             lambda: philox_reference(emu, pol, xh[3][:32], FP16, 11, 7000, replicas=3))
    torch.manual_seed(4)
    rgbs = [Lighting(0.1).sample_rgb(B).float() for _ in range(3)]
    rgbs_d = [r.cuda() for r in rgbs]
    for k in range(3):
        seq.call("lighting %d" % k, 5 if k == 0 else 4,
                 lambda k=k: augment_batch(pol, xd[k], FP32, rng=make_rng(11, 9000 + k * B, FP32), lighting_rgb=rgbs_d[k]),
                 lambda k=k: philox_reference(emu, pol, xh[k], FP32, 11, 9000 + k * B, lighting_rgb=rgbs[k]))
    u8 = FusedAugmenter(pol, U8, H, W, 12)
    seq.philox("uint8 event, resolves ahead", 3, u8, xd[0][:64], xh[0][:64], u8.empty_out(64), 0)
    seq.philox("chained miss after it", 4, f16, xd[1], xh[1], f16.empty_out(B), 96)
    seq.philox("chained hit", 3, f16, xd[2], xh[2], f16.empty_out(B), 192)
    hin = torch.from_numpy(xh[3][:64].copy()).pin_memory()
    hout = torch.empty((64, 3, H, W), dtype=torch.float16).pin_memory()
    tc, rng_h = FP16.c_struct(H, W), make_rng(13, 400, FP16)

    def host_entry():
        _lib.check(_lib.lib.faa_augment_host(pol.handle, hin.data_ptr(), hout.data_ptr(), None, 64, H, W, C.byref(tc),
                                             C.byref(rng_h), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return hout
    seq.call("host entry", 16, host_entry, lambda: philox_reference(emu, pol, xh[3][:64], FP16, 13, 400), clone=False)
    seq.philox("chained after the host entry", 4, f16, xd[0], xh[0], f16.empty_out(B), 288)
    seq.check()


def test_buffer_growth_in_flight(emu):
    """e. 96 -> 1024 -> 96 images with overlap: the program slots and scratch images are regrown mid-sequence"""
    pol = _pol()
    seq = Sequence(emu, pol)
    xh, xd = _inputs(2, 96, seed=90)
    bh, bd = _inputs(2, 1024, seed=95)
    f = FusedAugmenter(pol, FP16, H, W, 21, overlap_calls=True)
    seq.philox("96 a", 4, f, xd[0], xh[0], f.empty_out(96), 0)
    seq.philox("96 b", 3, f, xd[1], xh[1], f.empty_out(96), 96)
    seq.philox("1024 a", 4, f, bd[0], bh[0], f.empty_out(1024), 192)
    seq.philox("1024 b", 3, f, bd[1], bh[1], f.empty_out(1024), 1216)
    seq.philox("96 c", 4, f, xd[0], xh[0], f.empty_out(96), 2240)
    seq.philox("96 d", 3, f, xd[1], xh[1], f.empty_out(96), 2336)
    seq.check()


@pytest.mark.parametrize("schedule", ["chained", "event"])
def test_two_streams_alternating(emu, schedule):
    """f. calls alternating between two streams on one handle: a call on the other stream must not rewrite the program
    slot (or poll a ticket) of the previous call's kernels, whichever schedule either of them ran"""
    pol = _pol()
    seq = Sequence(emu, pol)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    if schedule == "chained":
        B = 96
        xh, xd = _inputs(4, B, seed=100)
        f = FusedAugmenter(pol, FP16, H, W, 31, overlap_calls=True)
        outs = [f.empty_out(B) for _ in range(6)]
        torch.cuda.synchronize()
        for k in range(6):
            seq.philox("chained %d" % k, 4 if k == 0 else 3, f, xd[k % 4], xh[k % 4], outs[k], k * B, stream=(s1, s2)[k % 2])
    else:
        from helpers import seed_all
        B = 64
        xh, xd = _inputs(4, B, seed=110)
        u8 = FusedAugmenter(pol, U8, H, W, 32)
        f = FusedAugmenter(pol, FP16, H, W, 33)
        outs = [u8.empty_out(B) for _ in range(4)]
        fouts = [f.empty_out(B) for _ in range(2)]
        seed_all(6)
        records = []
        for k in range(2):
            s, b = pol.sample_parity(B, H, W, FP16)
            records.append((s, b, torch.from_numpy(s.view(np.uint8).copy()).cuda(), torch.from_numpy(b.view(np.uint8).copy()).cuda()))
        torch.cuda.synchronize()
        for k in range(4):                      # uint8 event calls resolving ahead on the side stream: hits after the first
            seq.philox("uint8 event %d" % k, 3 if k == 0 else 2, u8, xd[k], xh[k], outs[k], k * B, stream=(s1, s2)[k % 2])
        for k in range(2):                      # resolved records
            seq.call("parity event %d" % k, 2, lambda k=k: augment_batch(pol, xd[k], FP16, records[k][2], records[k][3]),
                     lambda k=k: reference_output(emu, pol, xh[k], FP16, records[k][0], records[k][1]), stream=(s1, s2)[k % 2])
        # a chained miss on the other stream right after an event call, then its hit back on the first stream
        seq.philox("chained after event", 3, f, xd[2], xh[2], fouts[0], 1000, stream=s1)
        seq.philox("chained hit", 2, f, xd[3], xh[3], fouts[1], 1000 + B, stream=s2)
    seq.check()


def test_long_persistent_rows_b2048(emu):
    """g. 224 b2048 uint8 HWC (the augment stage of config 4), three chained steps.  The emulator checks a fixed sample
    of 256 images per step; every image of every step equals the records route (the emulator's records through the
    event schedule) on a fresh handle"""
    B = 2048
    pol = _pol()
    x = synth_batch(B, (H, W), seed=120)
    xs = [x, np.ascontiguousarray(x[::-1])]
    xd = [torch.from_numpy(a).cuda() for a in xs]
    f = FusedAugmenter(pol, U8, H, W, 41, overlap_calls=True)
    outs = [f.empty_out(B) for _ in range(3)]
    got = []
    for k in range(3):
        n0 = _launches()
        f(xd[k % 2], outs[k], k * B)
        got.append(_launches() - n0)
    torch.cuda.synchronize()
    assert got == [4, 3, 3], got
    from helpers import emu_philox_records
    sample = np.sort(np.random.default_rng(0).choice(B, 256, replace=False))
    fresh = _pol()
    for k in range(3):
        s, b = emu_philox_records(emu, pol, B, H, W, U8, 41, k * B)
        res = outs[k].cpu()
        want = reference_output(emu, pol, xs[k % 2][sample], U8, s[sample], b[sample])
        assert torch.equal(res[torch.from_numpy(sample)], want), (k, _first_bad(res[torch.from_numpy(sample)], want))
        rec = augment_batch(fresh, xd[k % 2], U8, torch.from_numpy(s.view(np.uint8).copy()).cuda(),
                            torch.from_numpy(b.view(np.uint8).copy()).cuda()).cpu()
        assert torch.equal(res, rec), (k, _first_bad(res, rec))
