"""Launch geometries of the policy kernels: one case per planner regime.

The launch planner (`plan_launch`, csrc/faa_core.cuh) picks, separately for each kernel of a launch, which code runs:
whether the band is staged into shared memory by TMA, whether the light kernel's (narrower) band is, whether the
materialisation chunk exists, whether the octet paths and the lean gathers exist, whether the mid kernel runs and with
which bands, and whether the cluster kernel is launched at all (`no_heavy`).  Those choices depend on the image size
and on the buffers' addresses, so every regime is a separate thing to test.

`plan()` below asks the planner itself, through the host build of faa_core.cuh (tests/emu).
tests/test_geometry_plan.py checks that every case of CASES is in the regime it claims and that every regime has a
case; tests/test_gpu_geometries.py runs every case on the device against the oracle and asserts the launch count.
CROP_CASES (RandomCrop: crop_pad and outputs smaller than the image) and MIX_CASES (fused Mixup, two sources) do the
same for the other two inputs of the planner that change what the kernels run; tests/test_gpu_crop_mix_geometries.py
runs them on the device.

RAGGED_CASES does it for the ragged policy launch (`faa_augment_ragged`, planned by `plan_ragged`): one image per
per-image geometry, named by `ragged_regime()`, and RAGGED_MIXES, the calls tests/test_gpu_ragged_geometries.py makes
of them with the pixel launches each one claims.
"""
import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


STAGE_LIMIT = 150 * 1024     # bytes of staged band(s) per cluster-kernel CTA (both sources' together)


@dataclass
class Plan:
    W: int
    bands: int
    stage: bool               # TMA staging of the cluster kernel's band
    stage_off: str            # why not: "size" (H*W*3 % 16), "base" (input address), "band" (too large), "" if staged;
                              # two sources: "doubled band" when one source's band would stage but two do not fit
    light_bands: int
    light_staged: bool        # the light kernel's band is staged
    octets: bool              # the 8-pixel paths
    mat: bool                 # the materialisation chunk (>= 3 rows)
    split: bool               # light (+ mid) kernels take the programs they cover
    use_mid: bool             # the mid kernel runs
    mid_bands: int
    mid_threads: int
    no_heavy: bool            # the cluster kernel is not launched
    allow: int                # resolve-kernel allow bits: 1 chunk, 2 scratch, 4 lean gathers
    band_cap: int = 0         # bytes of one source's staged cluster-kernel band (0: unstaged)
    crop: bool = False        # RandomCrop: crop_pad > 0 or an output smaller than the image
    smaller: bool = False     # the output is smaller than the image
    two_src: bool = False     # fused Mixup
    self_resolving: bool = False
    use_chain: bool = False   # chained schedule (Philox records, resolve-ahead allowed)

    def launches(self):
        """kernels of one call on resolved records (event schedule, faa_cabi.cu launch_event): the resolve kernel, then
        either the cluster kernel alone or light + (mid) + (cluster unless no_heavy); a self-resolving launch is one
        kernel"""
        if self.self_resolving:
            return 1
        if not self.split:
            return 2
        return 2 + int(self.use_mid) + int(not self.no_heavy)


def plan(emu, H, W, batch, u8=False, in_off=0, out_off=0, split_min=-1, has_sg=True, out_h=None, out_w=None, crop_pad=0,
         two_src=False, philox=False, allow_ahead=False):
    """the planner's decisions for a launch of the final window (apply_tail), input and output at `in_off` / `out_off`
    bytes from a 256-byte aligned allocation (split_min -1: the library's default).  By default a single-source launch
    on resolved records, of the image's own size, no crop; out_h / out_w / crop_pad: RandomCrop; two_src: fused Mixup;
    philox / allow_ahead: records drawn on the device, the next batch may be resolved ahead"""
    out_h, out_w = H if out_h is None else out_h, W if out_w is None else out_w
    names = emu.faa_emu_plan_fields().decode().split()
    out = (C.c_int32 * len(names))()
    assert emu.faa_emu_plan(H, W, out_h, out_w, batch, crop_pad, int(u8), in_off % 16, out_off % 16, int(two_src), 1,
                            int(has_sg), split_min, int(philox), int(allow_ahead), out) == len(names)
    d = dict(zip(names, out))
    stage_off = "" if d["stage"] else "size" if (H * W * 3) % 16 else "base" if in_off % 16 else "band"
    if stage_off == "band" and two_src and plan(emu, H, W, batch, u8, in_off, out_off, split_min, has_sg, out_h, out_w,
                                                 crop_pad).stage:
        stage_off = "doubled band"
    return Plan(W, d["bands"], bool(d["stage"]), stage_off, d["light_bands"], bool(d["light_staged"]), bool(d["octets"]),
                d["mat_cap"] > 0, bool(d["use_split"]), bool(d["use_mid"]), d["mid_bands"], d["mid_threads"],
                bool(d["no_heavy"]), d["allow"], d["band_cap"], crop_pad > 0 or (out_h, out_w) != (H, W),
                (out_h, out_w) != (H, W), two_src, bool(d["self_resolving"]), bool(d["use_chain"]))


def regime(p: Plan):
    """the regime names of the case table (the code a split float launch runs)"""
    if p.two_src:       # fused Mixup: the cluster kernel alone, no chunk, no scratch image
        return "mix%s, %s" % (" with a crop" if p.crop else "", "staged" if p.stage else "unstaged (%s)" % p.stage_off)
    if p.crop:
        return _crop_regime(p)
    if not p.split:
        return "one pixel kernel"
    if p.use_mid:
        if not p.no_heavy:
            return "mid %d bands + cluster kernel (%s)" % (p.mid_bands, "no chunk" if not p.mat else "no octets")
        if not p.light_staged:
            return "octets, unstaged light band, mid %d bands" % p.mid_bands
        return "mid %d bands, %d threads" % (p.mid_bands, p.mid_threads)
    if p.stage:
        return "staged, no mid kernel (%s)" % ("W % 4" if p.W % 4 else "output address")
    if not p.mat:
        return "unstaged (%s), no chunk" % p.stage_off
    return "unstaged (%s)" % p.stage_off


def _crop_regime(p: Plan):
    """RandomCrop launches: no mid kernel (crop_pad > 0 or a smaller output), so a split launch runs the light and the
    cluster kernel on bands that include the crop slack; uint8 output with a crop does not split"""
    if not p.split:
        return "crop, one pixel kernel"
    if not p.stage:
        return "crop, unstaged (%s)%s" % (p.stage_off, "" if p.mat else ", no chunk")
    if p.band_cap + 4096 > STAGE_LIMIT:          # within 4 KB of the limit
        return "crop, band at the limit%s" % ("" if p.light_staged else ", light band unstaged")
    if not p.light_staged:
        return "crop, staged, light band unstaged"
    if p.smaller:
        return "crop to a smaller output, staged"
    return "crop, staged, %s" % ("octets" if p.octets else "no octets")


@dataclass
class Case:
    shape: tuple
    regime: str
    launches: int             # kernels per split float call on resolved records (the unsplit path always launches 2)
    why: str                  # how the planner arrives there
    in_off: int = 0           # input byte offset (4-byte aligned)
    out_off: int = 0          # fp16 / bf16 output byte offset (8-byte aligned)
    big: bool = False         # reduced program list, emulator reference + an oracle sample

    @property
    def id(self):
        s = "%dx%d" % self.shape
        return s + ("_in%d" % self.in_off if self.in_off else "") + ("_out%d" % self.out_off if self.out_off else "")


# Launch counts (kernels per split float call on resolved records): resolve + light + mid = 3 when no program can be
# heavy (no_heavy); + the cluster kernel = 4 when the mid kernel runs but some programs stay heavy; resolve + light +
# cluster = 3 when the mid kernel cannot run.  Band sizes are the largest band, rounded up to 128 bytes.
CASES = [
    Case((240, 240), "mid 4 bands, 256 threads", 3, "8 bands; W % 8 == 0: octets + lean gathers; mid halves to 4 bands of 44 KB (2 would be 85 KB)"),
    Case((256, 256), "mid 4 bands, 512 threads", 3, "as 240, but a 4-band mid band is 50 KB > 48 KB: 512 threads"),
    Case((260, 260), "mid 4 bands + cluster kernel (no octets)", 4, "W % 8 == 4: no octets, so no lean gathers (allow bit 4) and two-gather programs stay heavy"),
    Case((300, 300), "mid 4 bands + cluster kernel (no octets)", 4, "W % 8 == 4 as 260; mid bands of 68 KB"),
    Case((380, 380), "mid 8 bands + cluster kernel (no octets)", 4, "W % 8 == 4; 4-band mid bands would be 108 KB > 80 KB: 8 bands of 56 KB"),
    Case((456, 456), "mid 8 bands, 512 threads", 3, "4-band mid bands would be 155 KB > 80 KB: 8 bands of 79 KB; light band 79 KB: staged"),
    Case((528, 528), "octets, unstaged light band, mid 8 bands", 3, "light band 105 KB > 100 KB: the light kernel reads global memory; cluster band <= 150 KB: staged"),
    Case((600, 600), "octets, unstaged light band, mid 8 bands", 3, "light band 135 KB; mid bands of 135 KB"),
    Case((480, 640), "octets, unstaged light band, mid 8 bands", 3, "light band 116 KB"),
    Case((640, 480), "octets, unstaged light band, mid 8 bands", 3, "light band 115 KB"),
    Case((427, 640), "octets, unstaged light band, mid 8 bands", 3, "H * W * 3 % 16 == 0 although H is odd; light band 105 KB"),
    Case((375, 500), "unstaged (size)", 3, "375 * 500 * 3 % 16 == 4: no TMA staging, so no octets and no mid kernel; chunk of 49 rows"),
    Case((500, 375), "unstaged (size)", 3, "W % 4 == 3: no aligned class, every program is C_GENERIC or C_MAT; no scratch image"),
    Case((333, 500), "unstaged (size)", 3, "333 * 500 * 3 % 16 == 12"),
    Case((224, 224), "unstaged (base)", 3, "input 4 bytes past a 16-byte boundary: no staging, so no octets / mid", in_off=4),
    Case((600, 600), "unstaged (base)", 3, "as 600 with the input 4 bytes past 16", in_off=4),
    Case((224, 224), "staged, no mid kernel (output address)", 3, "fp16 / bf16 output 8 bytes past 16: no octets, no mid kernel", out_off=8),
    Case((768, 1024), "unstaged (band)", 3, "8 bands of 294 KB > 150 KB", big=True),
    Case((1200, 1600), "unstaged (band)", 3, "8 bands of 713 KB", big=True),
    Case((2048, 1536), "unstaged (band)", 3, "pitch 4608 B: a chunk of 16384 / 4608 = 3 rows", big=True),
    Case((1536, 2048), "unstaged (band), no chunk", 3, "pitch 6144 B: 16384 / pitch = 2 rows < 3, no chunk (allow bit 0): slot-1 statistics "
         "are taken lazily (found a C_LUT program with Contrast behind a LUT op computing its mean wrongly here)", big=True),
    Case((3000, 4000), "unstaged (band), no chunk", 3, "pitch 12000 B: 1 row", big=True),
    Case((8192, 8), "mid 4 bands, 512 threads", 3, "header limit: 24-byte rows; mid halves to 4 bands of 48.1 KB", big=True),
    Case((8, 8192), "mid 8 bands + cluster kernel (no chunk)", 4, "header limit: 8 one-row bands of 72 KB, octets; pitch 24576 B: no chunk", big=True),
    Case((2, 8192), "mid 1 bands + cluster kernel (no chunk)", 4, "header limit: 2 bands (2 rows), the mid kernel runs 1 band of 48 KB; no chunk", big=True),
    Case((8192, 2), "staged, no mid kernel (W % 4)", 3, "header limit: 8 bands of 6 KB; W % 4 == 2: no mid kernel, C_GENERIC only", big=True),
    Case((8192, 8192), "unstaged (band), no chunk", 3, "header limit: bands of 24 MB; 67 M pixels per histogram", big=True),
]

# every regime the table must cover (a new planner branch adds its regime here, and a case to CASES)
REGIMES = [
    "mid 4 bands, 256 threads",
    "mid 4 bands, 512 threads",
    "mid 8 bands, 512 threads",
    "mid 4 bands + cluster kernel (no octets)",
    "mid 8 bands + cluster kernel (no octets)",
    "mid 8 bands + cluster kernel (no chunk)",
    "mid 1 bands + cluster kernel (no chunk)",
    "octets, unstaged light band, mid 8 bands",
    "staged, no mid kernel (output address)",
    "staged, no mid kernel (W % 4)",
    "unstaged (size)",
    "unstaged (base)",
    "unstaged (band)",
    "unstaged (band), no chunk",
]

# image sizes the ImageNet loaders feed the policy (data.py EFFICIENTNET_SIZES; ImageNetChain runs it on the source
# photo: common camera / ImageNet shapes) and the header's size limits
PHOTO_SHAPES = [(375, 500), (500, 375), (333, 500), (480, 640), (640, 480), (427, 640), (768, 1024), (1200, 1600),
                (2048, 1536), (1536, 2048), (3000, 4000)]
LIMIT_SHAPES = [(8, 8192), (8192, 8), (2, 8192), (8192, 2), (8192, 8192)]


@dataclass
class TailCase:
    """a RandomCrop launch (CROP_CASES) or a fused Mixup launch (MIX_CASES): the input shape, the output size and the
    tail's crop padding (a hint: records may reach further, the rows outside the staged band come from global memory)"""
    shape: tuple
    out: tuple
    pad: int
    regime: str
    launches: int             # kernels per float call on resolved records with FAA_SPLIT_MIN 0 (the unsplit path: 2)
    why: str
    in_off: int = 0           # input byte offset (4-byte aligned)
    u8: bool = False          # uint8 HWC output
    two_src: bool = False
    big: bool = False         # reduced program list, emulator reference + an oracle sample

    def plan(self, emu, batch=64, split_min=0):
        return plan(emu, *self.shape, batch, u8=self.u8, in_off=self.in_off, split_min=split_min, out_h=self.out[0],
                    out_w=self.out[1], crop_pad=self.pad, two_src=self.two_src)

    @property
    def id(self):
        s = ("mix_" if self.two_src else "crop_") + "%dx%d" % self.shape
        return (s + ("_to%dx%d" % self.out if self.out != self.shape else "") + ("_pad%d" % self.pad if self.pad else "") +
                ("_in%d" % self.in_off if self.in_off else "") + ("_u8" if self.u8 else ""))


# A split crop launch is resolve + light + cluster kernel (3): the mid kernel needs the image's own geometry.  A crop moves
# the octet paths to the images at offset (0, 0) and makes the pointwise programs of the others C_GENERIC when crop_dx % 4
# != 0 (build_prog): those go to the cluster kernel.
CROP_CASES = [
    TailCase((32, 32), (32, 32), 4, "crop, staged, octets", 3, "CIFAR: one band of 3 KB; images at (0, 0) take the octets"),
    TailCase((224, 224), (224, 224), 4, "crop, staged, octets", 3, "8 bands of 25 KB, the light kernel 7"),
    TailCase((224, 224), (224, 224), 16, "crop, staged, octets", 3, "bands of 41 KB (16 rows of crop slack on each side)"),
    TailCase((8192, 8), (8192, 8), 4, "crop, staged, octets", 3, "header limit: 24-byte rows, bands of 24 KB", big=True),
    TailCase((300, 300), (300, 300), 4, "crop, staged, no octets", 3, "W % 8 == 4: no octets; bands of 42 KB"),
    TailCase((224, 224), (224, 224), 127, "crop, band at the limit, light band unstaged", 3,
             "127 rows of slack: every band is the whole image, 150528 B <= 150 KB; the light kernel's 7 bands are too "
             "(> 100 KB) and read global memory"),
    TailCase((380, 380), (380, 380), 32, "crop, staged, light band unstaged", 3, "bands of 127 KB: staged for the "
             "cluster kernel, over 100 KB for the light kernel"),
    TailCase((224, 224), (200, 200), 0, "crop to a smaller output, staged", 3, "output rows != image rows, no padding: "
             "offsets in [0, 24]; output bands of 25 rows against image bands of 28; no octets; light kernel 8 bands"),
    TailCase((256, 256), (224, 224), 8, "crop to a smaller output, staged", 3, "offsets in [-8, 40]; bands of 52 KB"),
    TailCase((240, 240), (224, 224), 8, "crop to a smaller output, staged", 3, "offsets in [-8, 24]; bands of 37 KB"),
    TailCase((456, 456), (456, 456), 64, "crop, unstaged (band)", 3, "bands of 57 + 2 * 64 rows + halo: 250 KB > 150 KB"),
    TailCase((600, 600), (600, 600), 127, "crop, unstaged (band)", 3, "bands of 75 + 2 * 127 rows + halo: 582 KB"),
    TailCase((375, 500), (368, 496), 4, "crop, unstaged (size)", 3, "375 * 500 * 3 % 16 == 4; light kernel 5 bands"),
    TailCase((224, 224), (224, 224), 4, "crop, unstaged (base)", 3, "input 4 bytes past a 16-byte boundary", in_off=4),
    TailCase((1536, 2048), (1536, 2048), 8, "crop, unstaged (band), no chunk", 3,
             "pitch 6144 B: a chunk of band + 2 * 8 rows > 24 KB, 16384 / pitch = 2 rows < 3", big=True),
    TailCase((8, 8192), (8, 8192), 4, "crop, unstaged (band), no chunk", 3, "header limit: 8 one-row bands + 4 rows of "
             "slack on each side = the whole 192 KB image", big=True),
    TailCase((224, 224), (224, 224), 4, "crop, one pixel kernel", 2, "uint8 HWC output splits only through the octet "
             "paths without a crop: the cluster kernel alone", u8=True),
]

# Fused Mixup (NSRC = 2) never splits: resolve + cluster kernel (2), no materialisation chunk and no scratch image, so
# two-op programs run the lazy C_GENERIC path and Sharpness -> gather programs are evaluated lazily.  Both sources' bands
# are staged together, within 150 KB.
MIX_CASES = [
    TailCase((224, 224), (224, 224), 0, "mix, staged", 2, "2 x 20 KB", two_src=True),
    TailCase((256, 256), (256, 256), 0, "mix, staged", 2, "2 x 26 KB", two_src=True),
    TailCase((380, 380), (380, 380), 0, "mix, staged", 2, "2 x 56 KB", two_src=True),
    TailCase((8, 8192), (8, 8192), 0, "mix, staged", 2, "2 x 72 KB: the closest to the limit", two_src=True, big=True),
    TailCase((2, 8192), (2, 8192), 0, "mix, staged", 2, "2 one-row bands of 48 KB", two_src=True, big=True),
    TailCase((8192, 2), (8192, 2), 0, "mix, staged", 2, "W % 4 == 2: C_GENERIC only; 2 x 6 KB", two_src=True, big=True),
    TailCase((456, 456), (456, 456), 0, "mix, unstaged (doubled band)", 2, "2 x 79 KB > 150 KB; a single source stages",
             two_src=True),
    TailCase((600, 600), (600, 600), 0, "mix, unstaged (doubled band)", 2, "2 x 135 KB", two_src=True),
    TailCase((375, 500), (375, 500), 0, "mix, unstaged (size)", 2, "375 * 500 * 3 % 16 == 4", two_src=True),
    TailCase((224, 224), (224, 224), 0, "mix, unstaged (base)", 2, "input 4 bytes past a 16-byte boundary", in_off=4,
             two_src=True),
    TailCase((768, 1024), (768, 1024), 0, "mix, unstaged (band)", 2, "one source's band is already 294 KB",
             two_src=True, big=True),
    TailCase((224, 224), (224, 224), 16, "mix with a crop, staged", 2, "2 x 41 KB", two_src=True),
    TailCase((380, 380), (380, 380), 32, "mix with a crop, unstaged (doubled band)", 2, "2 x 127 KB", two_src=True),
]

# every regime of the crop and Mixup tables
CROP_REGIMES = [
    "crop, staged, octets",
    "crop, staged, no octets",
    "crop, band at the limit, light band unstaged",
    "crop, staged, light band unstaged",
    "crop to a smaller output, staged",
    "crop, unstaged (band)",
    "crop, unstaged (size)",
    "crop, unstaged (base)",
    "crop, unstaged (band), no chunk",
    "crop, one pixel kernel",
]
MIX_REGIMES = [
    "mix, staged",
    "mix, unstaged (doubled band)",
    "mix, unstaged (size)",
    "mix, unstaged (base)",
    "mix, unstaged (band)",
    "mix with a crop, staged",
    "mix with a crop, unstaged (doubled band)",
]


# ------------------------------------------------------------------------------------- ragged policy launches --
# `faa_augment_ragged` gives every image the cluster-kernel geometry `plan_launch` picks for a uniform uint8 launch of
# that image alone (`plan_ragged`, csrc/faa_core.cuh) and groups the images into one pixel launch per cluster size; the
# launch's dynamic shared memory is the largest band + chunk among its images.  A W % 4 == 0 image whose input does not
# start on a 4-byte boundary is first copied to an aligned buffer (one more launch for the whole call).
def load_emu_ragged_plan():
    """the host build of `plan_ragged` (tests/emu/faa_emu_ragged_plan.cpp), built on demand with g++"""
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_ragged_plan.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_ragged_plan.cpp")
    core = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.faa_emu_ragged_geom_fields.restype = C.c_char_p
    lib.faa_emu_plan_ragged.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.faa_emu_plan_ragged.restype = C.c_int
    return lib


def plan_ragged(lib, sizes, in_mod16=None, out_mod16=None, has_sg=True):
    """(geom_of [n], order [n], launches [(bands, first, count, smem)], geoms [dict]) of plan_ragged"""
    n = len(sizes)
    hw = np.ascontiguousarray(np.array(sizes, np.int32).reshape(-1, 2))
    im = np.ascontiguousarray(np.zeros(n, np.int32) if in_mod16 is None else np.array(in_mod16, np.int32) % 16)
    om = np.ascontiguousarray(np.zeros(n, np.int32) if out_mod16 is None else np.array(out_mod16, np.int32) % 16)
    names = lib.faa_emu_ragged_geom_fields().decode().split()
    geom_of, order = np.zeros(n, np.int32), np.zeros(n, np.int32)
    launches = np.zeros((4, 4), np.int32)
    geoms = np.zeros((max(n, 1), len(names)), np.int32)
    ng = C.c_int32()
    nl = lib.faa_emu_plan_ragged(n, hw.ctypes.data, im.ctypes.data, om.ctypes.data, int(has_sg), geom_of.ctypes.data,
                                 order.ctypes.data, launches.ctypes.data, geoms.ctypes.data, C.byref(ng))
    return geom_of, order, [tuple(int(v) for v in launches[k]) for k in range(nl)], \
        [dict(zip(names, (int(v) for v in geoms[k]))) for k in range(ng.value)]


def ragged_copied(W, in_off):
    """the library re-aligns the input first (faa_cabi.cu faa_augment_ragged): the kernel's 32-bit loads of W % 4 == 0
    rows need a 4-byte aligned base"""
    return W % 4 == 0 and in_off % 4 != 0


def ragged_regime(g, in_off=0, out_off=0):
    """an image's regime in a ragged launch, from its `plan_ragged` geometry `g` and its input / output byte offsets
    mod 16: (CTAs per image, staging, octets, chunk, scratch image).  Staging: "staged" (TMA), else why not, in the
    planner's order - "base + copy" (read from the re-aligned copy), "size" (H * W * 3 % 16), "base" (input address),
    "band" (over 150 KB).  Octets: the 8-pixel paths, else why not - W % 8, the output address, or an unstaged band."""
    H, W = g["H"], g["W"]
    if g["stage"]:
        staging = "staged"
    elif ragged_copied(W, in_off):
        staging = "base + copy"
    elif (H * W * 3) % 16:
        staging = "size"
    elif in_off % 16:
        staging = "base"
    else:
        staging = "band"
    if g["octets"]:
        octets = "octets"
    else:
        octets = "no octets (%s)" % ("W % 8" if W % 8 else "output address" if out_off % 16 else "unstaged")
    return (g["bands"], staging, octets, "chunk" if g["mat_cap"] else "no chunk",
            "scratch" if g["scratch"] else "no scratch")


# the values of each dimension of ragged_regime() the table must cover
RAGGED_DIMENSIONS = [
    (1, 2, 4, 8),
    ("staged", "base + copy", "size", "base", "band"),
    ("octets", "no octets (W % 8)", "no octets (output address)", "no octets (unstaged)"),
    ("chunk", "no chunk"),
    ("scratch", "no scratch"),
]


@dataclass
class RaggedCase:
    """one image of a ragged launch: its size, the byte offsets mod 16 of its input and output, and the regime it claims
    (ragged_regime) under a policy with a Sharpness -> gather program"""
    shape: tuple
    regime: tuple
    why: str
    in_off: int = 0           # 0, 4, or odd (a W % 4 == 0 image is then copied first)
    out_off: int = 0          # 0 or 4 (uint8 outputs of W % 4 == 0 images must be 4-byte aligned)

    @property
    def id(self):
        s = "%dx%d" % self.shape
        return s + ("_in%d" % self.in_off if self.in_off else "") + ("_out%d" % self.out_off if self.out_off else "")

    @property
    def big(self):
        return max(self.shape) > 640


def _rc(shape, bands, staging, octets, chunk, scratch, why, in_off=0, out_off=0):
    return RaggedCase(shape, (bands, staging, octets, chunk, scratch), why, in_off, out_off)


ST, COPY, SIZE, BASE, BAND = "staged", "base + copy", "size", "base", "band"
OCT, W8, OUTA, UNST = "octets", "no octets (W % 8)", "no octets (output address)", "no octets (unstaged)"
CH, NOCH, SCR, NOSCR = "chunk", "no chunk", "scratch", "no scratch"

# Band and chunk sizes are bytes of dynamic shared memory; a launch takes the largest band + chunk of its images.
RAGGED_CASES = [
    _rc((128, 160), 4, ST, OCT, CH, SCR, "20480 quads: 4 CTAs of 32 rows; band 16384 B + chunk 16352 B"),
    _rc((128, 164), 4, ST, W8, CH, SCR, "W % 8 == 4: no octets; band 16768 B"),
    _rc((128, 160), 4, ST, OUTA, CH, SCR, "output 4 bytes past 16: no octets", out_off=4),
    _rc((128, 160), 4, BASE, UNST, CH, SCR, "input 4 bytes past 16: no TMA staging, the chunk only", in_off=4),
    _rc((128, 160), 4, COPY, UNST, CH, SCR, "odd input byte offset: re-aligned copy, planned unstaged", in_off=1),
    _rc((8, 4000), 4, ST, OCT, NOCH, SCR, "2-row bands of 48000 B; pitch 12000 B: 16384 / pitch = 1 row, no chunk"),
    _rc((8, 4000), 4, COPY, UNST, NOCH, SCR, "copied, no chunk: the lazy statistics from global memory", in_off=1),
    _rc((5, 7620), 4, SIZE, W8, NOCH, SCR, "5 * 7620 * 3 % 16 == 4; W % 8 == 4; pitch 22860 B: no chunk"),
    _rc((6, 3679), 4, SIZE, W8, NOCH, NOSCR, "W % 4 == 3: C_GENERIC only, no scratch image; no chunk"),
    _rc((31, 600), 4, SIZE, UNST, CH, SCR, "31 * 600 * 3 % 16 == 8; W % 8 == 0 but unstaged: no octets"),
    _rc((624, 640), 8, ST, OCT, CH, SCR, "78 + 2 halo rows of 1920 B: a staged band of exactly 153600 B, the limit; "
        "+ chunk 15392 B = 168992 B of dynamic shared memory"),
    _rc((632, 640), 8, BAND, UNST, CH, SCR, "79 + 2 rows: 155520 B > 150 KB, unstaged; chunk 15392 B"),
    _rc((2048, 1536), 8, BAND, UNST, CH, SCR, "pitch 4608 B: a chunk of 3 rows"),
    _rc((3000, 4000), 8, BAND, UNST, NOCH, SCR, "pitch 12000 B: 1 row, no chunk; no dynamic shared memory at all"),
    _rc((17, 2048), 8, ST, OCT, NOCH, SCR, "3-row bands of 18432 B + halo; pitch 6144 B: 2 rows, no chunk"),
    _rc((768, 1024), 8, COPY, UNST, CH, SCR, "a copied photo: 2.4 MB re-aligned", in_off=1),
    _rc((8, 1024), 2, ST, OCT, CH, SCR, "2048 quads: 2 CTAs of 4 rows"),
    _rc((3000, 2), 2, ST, W8, CH, NOSCR, "3000 quads; W % 4 == 2: no scratch image"),
    _rc((2, 8192), 2, BASE, UNST, NOCH, SCR, "header limit: 2 one-row bands, input 4 bytes past 16; no chunk", in_off=4),
    _rc((1, 1), 1, SIZE, W8, CH, NOSCR, "one pixel"),
    _rc((64, 2), 1, ST, W8, CH, NOSCR, "32 quads: one CTA, a staged band of 384 B"),
    _rc((3, 4), 1, COPY, W8, CH, SCR, "copied though 36 bytes would not stage anyway", in_off=1),
    _rc((1, 8192), 1, ST, OCT, NOCH, SCR, "one row: one CTA, a staged band, pitch 24576 B: no chunk"),
    _rc((8, 8192), 8, ST, OCT, NOCH, SCR, "header limit: 8 one-row bands of 73728 B, no chunk"),
    _rc((8192, 8), 8, ST, OCT, CH, SCR, "header limit: 24-byte rows, bands of 24704 B"),
    _rc((2, 8192), 2, ST, OCT, NOCH, SCR, "header limit: 2 one-row bands"),
    _rc((8192, 2), 8, ST, W8, CH, NOSCR, "header limit: 6-byte rows, W % 4 == 2"),
]

# the header's largest image, its own GPU test (67 M pixels per histogram)
RAGGED_HUGE = _rc((8192, 8192), 8, BAND, UNST, NOCH, SCR, "header limit: bands of 24 MB, no chunk")


def ragged_case(case_id):
    return next(c for c in RAGGED_CASES + [RAGGED_HUGE] if c.id == case_id)


# The calls of tests/test_gpu_ragged_geometries.py, one image per case in this order, and the pixel launches plan_ragged
# gives them: (CTAs per image, first, count, dynamic shared memory), largest images first.  Each call holds staged,
# unstaged, chunk-less and copied images together; the first two have all four cluster sizes (four pixel launches, the
# most a call can have).  Shared memory set by an image other than the launch's first: four_cluster_sizes - 624x640
# behind 632x640 (8 CTAs), 8x4000 behind 5x7620 (4 CTAs); photos_and_limits - 8x8192 behind 2048x1536 and 768x1024;
# smem_from_the_second_image - 624x640 behind 3000x4000, which needs none.
RAGGED_MIXES = {
    "four_cluster_sizes": (
        ["632x640", "128x160", "128x164", "128x160_out4", "128x160_in4", "128x160_in1", "8x4000", "8x4000_in1", "5x7620",
         "6x3679", "31x600", "624x640", "17x2048", "8x1024", "3000x2", "2x8192_in4", "1x1", "64x2", "3x4_in1", "1x8192"],
        [(8, 0, 3, 168992), (4, 3, 10, 48000), (2, 13, 3, 33824), (1, 16, 4, 24576)]),
    "photos_and_limits": (
        ["2048x1536", "768x1024_in1", "8x8192", "8192x8", "2x8192", "8192x2", "128x160_in1", "3x4_in1"],
        [(8, 0, 5, 73728), (4, 5, 1, 16352), (2, 6, 1, 49152), (1, 7, 1, 96)]),
    "smem_from_the_second_image": (
        ["3000x4000", "624x640", "128x160", "3x4_in1"],
        [(8, 0, 2, 168992), (4, 2, 1, 32736), (1, 3, 1, 96)]),
}
