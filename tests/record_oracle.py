"""The oracle of one decision record: what `oracle.pil_path` computes for an image, given the draws instead of taking them.

`PolicyTransform` draws its decisions from Python's `random` and numpy's global state while it renders, so it can only
check records that `CompiledPolicy.sample_parity` replayed from those same generators.  A launch that draws on the device
(Philox: `FusedAugmenter`, `augment_batch(rng=...)`, `run_many`, `augment_tta`) writes records no global generator
produced.  `render_record` renders such a record with the same Pillow calls as `pil_path.run_op`, reading each draw from
the record:

* `sub` selects the sub-policy; bit j of `gate` applies its op j (the draw `random.random() > pr` failed);
* bit j of `sign` negates a mirrored magnitude (`sample_parity` sets it when `random.random() > 0.5`, where
  `pil_path._mirror_draw` negates);
* a Cutout op draws its record box as Pillow's inclusive rectangle in `CUTOUT_RGB`; `x1 == -1` means no box
  (`Cutout` at a magnitude <= 0 returns the image);
* the horizontal flip comes last.

tests/test_lean_geometry_host.py pins it: under `seed_all(k)` it equals `PolicyTransform` byte for byte on the records of
`sample_parity`, for every single op, every ordered pair, boxes at the image borders and at level 0."""
import numpy as np
import PIL.Image
import PIL.ImageDraw

from oracle import pil_path

# ops whose magnitude takes a random sign (pil_path.run_op calls _mirror_draw): name -> Pillow call at magnitude v
_MIRRORED = {
    "ShearX": lambda img, v: pil_path._affine(img, (1, v, 0, 0, 1, 0)),
    "ShearY": lambda img, v: pil_path._affine(img, (1, 0, 0, v, 1, 0)),
    "TranslateX": lambda img, v: pil_path._affine(img, (1, 0, v * img.size[0], 0, 1, 0)),
    "TranslateY": lambda img, v: pil_path._affine(img, (1, 0, 0, 0, 1, v * img.size[1])),
    "TranslateXAbs": lambda img, v: pil_path._affine(img, (1, 0, v, 0, 1, 0)),
    "TranslateYAbs": lambda img, v: pil_path._affine(img, (1, 0, 0, 0, 1, v)),
    "Rotate": lambda img, v: img.rotate(v),
}
_BOXED = ("Cutout", "CutoutAbs")


def render_op(img, name, level, negate, box):
    """op `name` at `level` with the record's draws: `negate` the mirror sign, `box` (x0, y0, x1, y1) the Cutout box"""
    img = img.copy()                                        # pil_path.apply_op
    v = pil_path.magnitude(name, level)
    if name in _MIRRORED:
        return _MIRRORED[name](img, -v if negate else v)
    if name in _BOXED:
        x0, y0, x1, y1 = (int(c) for c in box)
        if x1 == -1:
            return img
        PIL.ImageDraw.Draw(img).rectangle((x0, y0, x1, y1), pil_path.CUTOUT_RGB)
        return img
    return pil_path.run_op(img, name, v)                    # no draw inside


def render_record(policies, image, sample, boxes):
    """uint8 [H, W, 3] result of one record (`_lib.SAMPLE_DTYPE`) and its boxes ([n_op] `_lib.BOX_DTYPE`) on `image`"""
    img = PIL.Image.fromarray(np.ascontiguousarray(image))
    gate, sign = int(sample["gate"]), int(sample["sign"])
    for j, (name, _, level) in enumerate(policies[int(sample["sub"])]):
        if (gate >> j) & 1:
            b = boxes[j]
            img = render_op(img, name, level, (sign >> j) & 1, (b["x0"], b["y0"], b["x1"], b["y1"]))
    out = np.asarray(img)
    return np.ascontiguousarray(out[:, ::-1]) if sample["flip"] else out


def render_batch(policies, batch, samples, boxes, idx=None, threads=8):
    """{i: render_record(...)} for the images `idx` (default: all), on `threads` threads (Pillow releases the GIL)"""
    import concurrent.futures
    idx = range(batch.shape[0]) if idx is None else idx
    with concurrent.futures.ThreadPoolExecutor(threads) as ex:
        outs = ex.map(lambda i: render_record(policies, batch[i], samples[i], boxes[i]), idx)
        return dict(zip(idx, outs))
