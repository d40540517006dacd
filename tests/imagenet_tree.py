"""ImageNet directory trees in the reference's layout (``<root>/imagenet-pytorch/{train,val}/<class>/<file>``), written
from a seed with Pillow for the tests of ``data.imagenet_index`` and the streamed loaders over it."""
import io
import os

import PIL.Image

from jpeg_cases import content, encode, pillow

SIZES = [(96, 128), (128, 96), (80, 80), (120, 160), (64, 200), (150, 100)]


def baseline_file(i, seed):
    """a file the device decoder takes: 4:4:4 / 4:2:2 / 4:2:0, grayscale or with restart intervals, at mixed sizes"""
    h, w = SIZES[(i + seed) % len(SIZES)]
    a = content("photo", h, w, seed * 1000 + i)
    if i % 5 == 4:
        return encode(a, gray=True, quality=85)
    opts = {"subsampling": i % 3, "quality": (75, 90, 95)[i % 3]}
    if i % 4 == 3:
        opts["restart_marker_blocks"] = 1 + i % 3
    return encode(a, **opts)


def refused_files(seed):
    """{name: bytes} of files the device decoder refuses and Pillow opens: progressive, CMYK, a PNG named .JPEG"""
    a = content("photo", 72, 88, seed)
    cmyk, png = io.BytesIO(), io.BytesIO()
    PIL.Image.fromarray(content("photo", 64, 96, seed + 1)).convert("CMYK").save(cmyk, "JPEG", quality=85)
    PIL.Image.fromarray(content("photo", 56, 40, seed + 2)).save(png, "PNG")
    return {"progressive.JPEG": encode(a, quality=85, progressive=True), "cmyk.JPEG": cmyk.getvalue(),
            "png_named.JPEG": png.getvalue()}


def write(path, b):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(b)


def write_tree(root, seed, n_classes=3, per_class=10, n_val=4, refused=True, text=True):
    """The split folders under ``root/imagenet-pytorch``; returns that directory.  Class k holds ``per_class`` baseline
    files (``val``: ``n_val``); with ``refused`` class 0 of both splits also holds the files of ``refused_files``, and
    with ``text`` a text file that the extension filter skips."""
    base = os.path.join(str(root), "imagenet-pytorch")
    k = 0
    for split, n in (("train", per_class), ("val", n_val)):
        for c in range(n_classes):
            d = os.path.join(base, split, "n%08d" % (1000 + 7 * c))
            for i in range(n):
                write(os.path.join(d, "%s_%d_%03d.JPEG" % (split, c, i)), baseline_file(k, seed))
                k += 1
            if c == 0 and refused:
                for name, b in refused_files(seed + c).items():
                    write(os.path.join(d, name), b)
            if c == 0 and text:
                write(os.path.join(d, "notes.txt"), b"not an image\n")
    return base


def pillow_pixels(paths):
    out = []
    for p in paths:
        with open(p, "rb") as f:
            out.append(pillow(f.read()))
    return out


def cut_scan(b):
    """the file cut halfway through its entropy-coded scan (the header parses; the decode status says truncated)"""
    from fast_autoaugment_b200.engine import parse_jpeg
    hdr, _ = parse_jpeg(b)
    return b[:int(hdr["scan_off"][0]) + int(hdr["scan_len"][0]) // 2]
