"""Golden vectors for the device JPEG decoder: JPEG files written by Pillow and Pillow's own decode of each.

Pillow (libjpeg-turbo) encodes `gen.synth_image` content and one high-contrast noise image over qualities 10-100,
subsampling 0 / 1 / 2 (4:4:4, 4:2:2, 4:2:0), optimised Huffman tables, restart markers (every MCU / every MCU row),
16-bit quantisation tables, grayscale and sizes from 1x1 to 640x480; plus three files the decoder must refuse (progressive,
CMYK, truncated).  Stored per file: the bytes, and `np.asarray(Image.open(f))` (grayscale replicated to three channels)
in full for small images, as a SHA-256 plus three sampled rows for large ones.  For one colour and one grayscale file the
reference's `_transform(224)` (make_preprocess_golden.reference_transform) is stored as well: the 8-bit crop's SHA-256 and its
rows TF_ROWS, and those rows of every channel of the normalised tensor (the whole tensor follows from the crop).

Usage:  python tests/golden/make_jpeg_golden.py
"""
from __future__ import annotations

import hashlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden import gen  # noqa: E402

FULL_PIXELS = 80 * 80   # larger decodes are stored as hash + sampled rows
TF_ROWS = [0, 57, 111, 223]


def noise_image(h, w, seed=7):
    """Saturated 8x8 blocks next to uniform noise: the IDCT over- and undershoots that exercise the range limit."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
    blk = rng.integers(0, 2, (-(-h // 8), -(-w // 8), 1)).astype(np.uint8) * 255
    sat = np.repeat(np.repeat(blk, 8, 0), 8, 1)[:h, :w]
    checker = ((np.arange(h)[:, None] // 8 + np.arange(w)[None, :] // 8) % 2 == 0)[..., None]
    return np.where(checker, np.broadcast_to(sat, img.shape), img).astype(np.uint8)


def corpus():
    """[(name, PIL image, save kwargs, expected outcome)] — outcome "ok", or the exception class name."""
    from PIL import Image

    out = []
    for i, (h, w) in enumerate([(1, 1), (7, 9), (8, 8), (15, 17), (33, 65)]):
        img = Image.fromarray(gen.synth_image(h, w, seed=i))
        for sub in (0, 1, 2):
            out.append((f"s{h}x{w}_q75_sub{sub}", img, dict(quality=75, subsampling=sub), "ok"))
        out.append((f"s{h}x{w}_q75_gray", img.convert("L"), dict(quality=75), "ok"))
    base = Image.fromarray(gen.synth_image(224, 224, seed=5))
    for q in (10, 50, 95, 100):
        out.append((f"s224_q{q}_sub2", base, dict(quality=q, subsampling=2), "ok"))
    out.append(("s224_q75_sub0_opt", base, dict(quality=75, subsampling=0, optimize=True), "ok"))
    out.append(("s224_q75_sub1_rst_blocks1", base, dict(quality=75, subsampling=1, restart_marker_blocks=1), "ok"))
    out.append(("s224_q75_sub2_rst_rows1", base, dict(quality=75, subsampling=2, restart_marker_rows=1), "ok"))
    out.append(("s224_q90_gray_rst_rows2", base.convert("L"), dict(quality=90, restart_marker_rows=2), "ok"))
    out.append(("s224_qt16_sub2", base, dict(qtables=[[300] * 64, [400] * 64], subsampling=2), "ok"))
    out.append(("s300x400_q75_sub1", Image.fromarray(gen.synth_image(300, 400, seed=6)), dict(quality=75, subsampling=1), "ok"))
    big = Image.fromarray(gen.synth_image(479, 641, seed=7))
    out.append(("s479x641_q75_sub2_rst_rows1", big, dict(quality=75, subsampling=2, restart_marker_rows=1), "ok"))
    out.append(("s479x641_q50_sub0_opt", big, dict(quality=50, subsampling=0, optimize=True), "ok"))
    out.append(("s480x640_q75_sub2", Image.fromarray(gen.synth_image(480, 640, seed=8)), dict(quality=75, subsampling=2), "ok"))
    out.append(("noise64x64_q100_sub0", Image.fromarray(noise_image(64, 64)), dict(quality=100, subsampling=0), "ok"))
    out.append(("noise48x72_q10_sub2", Image.fromarray(noise_image(48, 72, seed=8)), dict(quality=10, subsampling=2), "ok"))
    out.append(("noise40x40_q100_gray", Image.fromarray(noise_image(40, 40, seed=9)).convert("L"), dict(quality=100), "ok"))
    small = Image.fromarray(gen.synth_image(33, 65, seed=4))
    out.append(("bad_progressive", small, dict(quality=75, progressive=True), "NotImplementedError"))
    out.append(("bad_cmyk", small.convert("CMYK"), dict(quality=75), "NotImplementedError"))
    out.append(("bad_truncated", base, dict(quality=75, subsampling=2), "ValueError"))
    return out


def main():
    from PIL import Image

    from tests.golden.make_preprocess_golden import reference_transform

    z, names = {}, []
    for k, (name, img, kw, outcome) in enumerate(corpus()):
        buf = io.BytesIO()
        img.save(buf, "JPEG", **kw)
        data = buf.getvalue()
        if name == "bad_truncated":
            data = data[: len(data) * 3 // 5]
        z[f"f{k}_jpeg"] = np.frombuffer(data, np.uint8)
        names.append(dict(name=name, outcome=outcome))
        if outcome != "ok":
            continue
        a = np.asarray(Image.open(io.BytesIO(data)))
        if a.ndim == 2:
            a = np.repeat(a[..., None], 3, -1)
        a = np.ascontiguousarray(a)
        names[-1].update(h=a.shape[0], w=a.shape[1])
        if a.shape[0] * a.shape[1] <= FULL_PIXELS:
            z[f"f{k}_pil"] = a
        else:
            rows = np.array([0, a.shape[0] // 2, a.shape[0] - 1])
            z[f"f{k}_sha"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest(), np.uint8)
            z[f"f{k}_rows"] = rows
            z[f"f{k}_rowdata"] = a[rows]
    tf, _ = reference_transform()
    from torchvision.transforms import CenterCrop, InterpolationMode, Resize

    for tag, name in (("color", "s300x400_q75_sub1"), ("gray", "s224_q90_gray_rst_rows2")):
        k = next(i for i, n in enumerate(names) if n["name"] == name)
        pil = Image.open(io.BytesIO(z[f"f{k}_jpeg"].tobytes()))
        z[f"tf_{tag}_file"] = np.array(k)
        z[f"tf_{tag}_f32_rows"] = tf(pil).numpy()[:, TF_ROWS]
        u8 = np.ascontiguousarray(CenterCrop(224)(Resize(224, interpolation=InterpolationMode.BICUBIC)(pil)).convert("RGB"))
        z[f"tf_{tag}_u8_sha"] = np.frombuffer(hashlib.sha256(u8.tobytes()).digest(), np.uint8)
        z[f"tf_{tag}_u8_rows"] = u8[TF_ROWS]
    z["names"] = np.frombuffer(json.dumps(names).encode(), np.uint8)
    path = os.path.join(HERE, "jpeg.npz")
    np.savez_compressed(path, **z)
    print(len(names), "files,", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
