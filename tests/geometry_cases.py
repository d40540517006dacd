"""Launch geometries of the policy kernels: one case per planner regime.

The launch planner (`plan_launch`, csrc/faa_core.cuh) picks, separately for each kernel of a launch, which code runs:
whether the band is staged into shared memory by TMA, whether the light kernel's (narrower) band is, whether the
materialisation chunk exists, whether the octet paths and the lean gathers exist, whether the mid kernel runs and with
which bands, and whether the cluster kernel is launched at all (`no_heavy`).  Those choices depend on the image size
and on the buffers' addresses, so every regime is a separate thing to test.

`plan()` below asks the planner itself, through the host build of faa_core.cuh (tests/emu).
tests/test_geometry_plan.py checks that every case of CASES is in the regime it claims and that every regime has a
case; tests/test_gpu_geometries.py runs every case on the device against the oracle and asserts the launch count.
"""
import ctypes as C
from dataclasses import dataclass


@dataclass
class Plan:
    W: int
    bands: int
    stage: bool               # TMA staging of the cluster kernel's band
    stage_off: str            # why not: "size" (H*W*3 % 16), "base" (input address), "band" (too large), "" if staged
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

    def launches(self):
        """kernels of one call on resolved records (event schedule, faa_cabi.cu launch_event): the resolve kernel, then
        either the cluster kernel alone or light + (mid) + (cluster unless no_heavy)"""
        if not self.split:
            return 2
        return 2 + int(self.use_mid) + int(not self.no_heavy)


def plan(emu, H, W, batch, u8=False, in_off=0, out_off=0, split_min=-1, has_sg=True):
    """the planner's decisions for a single-source launch on resolved records, of the image's own size, no crop, final
    window (apply_tail), input and output at `in_off` / `out_off` bytes from a 256-byte aligned allocation
    (split_min -1: the library's default)"""
    names = emu.faa_emu_plan_fields().decode().split()
    out = (C.c_int32 * len(names))()
    assert emu.faa_emu_plan(H, W, H, W, batch, 0, int(u8), in_off % 16, out_off % 16, 0, 1, int(has_sg), split_min, 0, 0,
                            out) == len(names)
    d = dict(zip(names, out))
    stage_off = "" if d["stage"] else "size" if (H * W * 3) % 16 else "base" if in_off % 16 else "band"
    return Plan(W, d["bands"], bool(d["stage"]), stage_off, d["light_bands"], bool(d["light_staged"]), bool(d["octets"]),
                d["mat_cap"] > 0, bool(d["use_split"]), bool(d["use_mid"]), d["mid_bands"], d["mid_threads"],
                bool(d["no_heavy"]), d["allow"])


def regime(p: Plan):
    """the regime names of the case table (the code a split float launch runs)"""
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
