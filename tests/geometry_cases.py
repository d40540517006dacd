"""Launch geometries of the policy kernels: one case per planner regime, and a restatement of the planner.

`augment_common` (csrc/faa_cabi.cu) picks, separately for each kernel of a launch, which code runs: whether the band
is staged into shared memory by TMA, whether the light kernel's (narrower) band is, whether the materialisation chunk
exists, whether the octet paths and the lean gathers exist, whether the mid kernel runs and with which bands, and
whether the cluster kernel is launched at all (`no_heavy`).  Those choices depend on the image size and on the buffers'
addresses, so every regime is a separate thing to test.

`plan()` below is a RESTATEMENT of those decisions in Python, written from the C++ and citing it; it is not shared
with the library.  tests/test_geometry_plan.py checks that every case of CASES is in the regime it claims and that
every regime has a case; tests/test_gpu_geometries.py runs every case on the device against the oracle and asserts
the planner's launch count, which cross-checks this restatement against the real planner.
"""
from dataclasses import dataclass

SPLIT_MIN = 4 << 20            # faa_cabi.cu:968: pixels per launch from which the split kernels run


# ---- csrc/faa_kernels.cu:2271-2302 and :224-238 ------------------------------------------------------------------
def pick_bands(H, W, out_h, out_w):
    """faa_kernels.cu:2271: >= ~1024 output quads per CTA, a power of two <= 8"""
    quads = out_h * ((out_w + 3) // 4)
    b = 1
    while b < 8 and quads // (b * 2) >= 1024 and b * 2 <= H and b * 2 <= out_h:
        b *= 2
    return b


def band_range(band, bands, H, W, out_h, crop_pad):
    """faa_kernels.cu:224: byte range [lo, lo + len) of the rows band `band` may touch"""
    img_bytes = H * W * 3
    y0, y1 = band * H // bands, (band + 1) * H // bands
    oy0, oy1 = band * out_h // bands, (band + 1) * out_h // bands
    r0 = min(y0, oy0 - crop_pad) - 1
    r1 = max(y1, oy1 + crop_pad) + 1
    r0, r1 = max(r0, 0), min(r1, H)
    if r1 <= r0:
        return 0, 0
    row = W * 3
    lo = (r0 * row) & ~15
    hi = min((r1 * row + 15) & ~15, img_bytes)
    return lo, hi - lo


def band_capacity(bands, H, W, out_h, crop_pad):
    """faa_kernels.cu:2294: the largest band, rounded up to 128 bytes"""
    cap = max(band_range(b, bands, H, W, out_h, crop_pad)[1] for b in range(bands))
    return (cap + 127) & ~127


def light_bands(bands, out_h, out_w):
    """faa_cabi.cu:926-938: the light kernel takes the band count in 5..8 that fills 256-thread iterations best"""
    if bands != 8:
        return bands
    qpr = (out_w + 3) // 4
    best, lb = -1.0, bands
    for b in range(8, 4, -1):
        rows = (out_h + b - 1) // b
        quads = rows * qpr
        iters = (quads + 255) // 256
        eff = quads / (iters * 256.0) * (out_h / (rows * b))
        if eff > best + 0.02:
            best, lb = eff, b
    return lb


@dataclass
class Plan:
    W: int
    bands: int
    stage: bool               # :922 TMA staging of the cluster kernel's band
    stage_off: str            # why not: "size" (H*W*3 % 16), "base" (input address), "band" (> 150 KB), "" if staged
    light_bands: int
    light_staged: bool        # :939 the light kernel's band is staged (<= 100 KB)
    octets: bool              # :943 the 8-pixel paths
    mat: bool                 # :947-954 the materialisation chunk (>= 3 rows)
    split: bool               # :971 light (+ mid) kernels take the programs they cover
    use_mid: bool             # :980 the mid kernel runs
    mid_bands: int            # :632 mid_params
    mid_threads: int          # faa_kernels.cu:2367: 512 threads when a mid band is > 48 KB
    no_heavy: bool            # :1000 the cluster kernel is not launched
    allow: int                # resolve-kernel allow bits: 1 chunk, 2 scratch, 4 lean gathers

    def launches(self):
        """kernels of one call on resolved records (event schedule, faa_cabi.cu:795-861): the resolve kernel, then
        either the cluster kernel alone or light + (mid) + (cluster unless no_heavy)"""
        if not self.split:
            return 2
        return 2 + int(self.use_mid) + int(not self.no_heavy)


def plan(H, W, batch, u8=False, in_off=0, out_off=0, split_min=SPLIT_MIN, has_sg=True):
    """faa_cabi.cu:906-1000 for a single-source launch of the image's own size, no crop, final window (apply_tail),
    input and output at `in_off` / `out_off` bytes from a 256-byte aligned allocation"""
    out_h, out_w, crop_pad = H, W, 0
    bands = pick_bands(H, W, out_h, out_w)
    cap = band_capacity(bands, H, W, out_h, crop_pad)
    if (H * W * 3) % 16:
        stage_off = "size"
    elif in_off % 16:
        stage_off = "base"
    elif cap > 150 * 1024:
        stage_off = "band"
    else:
        stage_off = ""
    stage = stage_off == ""
    lb = light_bands(bands, out_h, out_w)
    light_staged = stage and band_capacity(lb, H, W, out_h, crop_pad) <= 100 * 1024
    octets = W % 8 == 0 and out_off % 16 == 0 and stage
    pitch = W * 3
    band_rows = (H + bands - 1) // bands + 2 + 2 * crop_pad
    rows = band_rows if band_rows * pitch <= 24576 else 16384 // pitch
    rows = min(rows, H + 2)
    mat = rows >= 3
    allow = 1 if mat else 0
    split = (not u8 or octets) and batch * H * W >= split_min
    use_mid = split and stage and W % 4 == 0 and out_off % 16 == 0
    if split and octets:
        allow |= 4
    if (has_sg or use_mid) and W % 4 == 0:
        allow |= 2
    no_heavy = use_mid and (allow & 6) == 6 and mat
    mb = bands
    while mb > 1 and band_capacity(mb // 2, H, W, out_h, 0) <= 80 * 1024:
        mb //= 2
    mid_threads = 512 if band_capacity(mb, H, W, out_h, 0) > 48 * 1024 else 256
    return Plan(W, bands, stage, stage_off, lb, light_staged, octets, mat, split, use_mid, mb if use_mid else 0,
                mid_threads if use_mid else 0, no_heavy, allow)


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
