"""GPU parity of the lean light launch (LaunchPlan::lean_light) against the host build, bit for bit.

A Philox launch of 224 x 224 images at the image's own size, without a crop, runs the lean variant of the light kernel
(octet paths only) beside the mid kernel, which takes the pairs those paths cannot finish.  Every ordered pair of the
policy ops runs through it: one policy per first op whose sub-policies are that op followed by each op, both gated on,
with a seed whose Philox draws pick every sub-policy of the batch (mirror signs and flips are drawn per image).  Each
batch is checked in fp16, bf16, fp32 and uint8 HWC, and with per-image Lighting tables in fp16 and fp32."""
import numpy as np
import pytest
import torch

import geometry_cases as G
from helpers import ALL_OPS, emu_philox_records, exact_norm_table, philox_reference, reference_output, synth_batch

from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, TailSpec, augment_batch, make_rng

pytestmark = pytest.mark.gpu

H = W = 224
B = 96
FIRST = 5000


def _seed_covering(emu, pol, tail):
    """the first seed whose Philox draws give every sub-policy to some image of the batch"""
    for seed in range(1, 200):
        samples, _ = emu_philox_records(emu, pol, B, H, W, tail, seed, FIRST)
        if len(set(samples["sub"].tolist())) == pol.n_sub:
            return seed
    raise AssertionError("no covering seed")


@pytest.mark.parametrize("first_op", ALL_OPS)
def test_every_ordered_pair_through_the_lean_launch(emu, first_op, monkeypatch):
    monkeypatch.setenv("FAA_SPLIT_MIN", "0")
    rng = np.random.default_rng(ALL_OPS.index(first_op))
    policies = [[(first_op, 1.0, float(rng.random())), (b, 1.0, float(rng.random()))] for b in ALL_OPS]
    u8 = TailSpec(None, 0, True, IMAGENET_MEAN, IMAGENET_STD, 0, torch.uint8)
    for tail in (u8, TailSpec.imagenet(0, torch.float16)):
        p = G.plan(emu, H, W, B, u8=tail.out_dtype == torch.uint8, split_min=0, philox=True, allow_ahead=True)
        assert p.allow & 8 and p.no_heavy, p                      # the lean light kernel, the mid kernel, no cluster kernel
    seed = _seed_covering(emu, CompiledPolicy(policies), u8)
    xh = synth_batch(B, (H, W), seed=17 + ALL_OPS.index(first_op))
    x = torch.from_numpy(xh).cuda()
    want_u8 = philox_reference(emu, CompiledPolicy(policies), xh, u8, seed, FIRST)
    samples, boxes = emu_philox_records(emu, CompiledPolicy(policies), B, H, W, u8, seed, FIRST)
    assert samples["flip"].any() and not samples["flip"].all()

    def check(got, want, what):
        bad = [(i, policies[samples["sub"][i]], int(samples["flip"][i])) for i in range(B) if not torch.equal(got[i], want[i])]
        assert not bad, (what, len(bad), bad[:4])

    check(augment_batch(CompiledPolicy(policies), x, u8, rng=make_rng(seed, FIRST, u8)).cpu(), want_u8, "uint8")
    tab = torch.from_numpy(exact_norm_table(IMAGENET_MEAN, IMAGENET_STD))
    xc = want_u8.permute(0, 3, 1, 2).long()
    want32 = torch.stack([tab[c][xc[:, c]] for c in range(3)], 1)
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        tail = TailSpec.imagenet(0, dt)
        got = augment_batch(CompiledPolicy(policies), x, tail, rng=make_rng(seed, FIRST, tail)).cpu()
        check(got, want32.to(dt), str(dt))
    from fast_autoaugment_b200.data import Lighting
    torch.manual_seed(ALL_OPS.index(first_op))
    rgb = Lighting(0.1).sample_rgb(B).float()
    for dt in (torch.float16, torch.float32):
        tail = TailSpec.imagenet(0, dt)
        got = augment_batch(CompiledPolicy(policies), x, tail, rng=make_rng(seed, FIRST, tail), lighting_rgb=rgb.cuda()).cpu()
        want = reference_output(emu, CompiledPolicy(policies), xh, tail, samples, boxes, lighting_rgb=rgb)
        check(got, want, "Lighting %s" % dt)
