"""CPU tier of the device JPEG decoder (macaw_llm_b200/jpeg.py, csrc/jpeg.cu): the host parser (tables, segments, MCU
counts, refusals), the numpy restatement of libjpeg-turbo's arithmetic (tests/jpeg_ref.py) against Pillow's decodes
stored in tests/golden/jpeg.npz, the C layout of the descriptors and the argument checks of mm_jpeg_decode."""
import ctypes
import hashlib
import json
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from tests import helpers as H
from tests import jpeg_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(os.path.join(H.GOLDEN, "jpeg.npz"))
NAMES = json.loads(Z["names"].tobytes())
MEAN_STD = (np.array([0.48145466, 0.4578275, 0.40821073], np.float32), np.array([0.26862954, 0.26130258, 0.27577711], np.float32))


def fixture(name):
    k = next(i for i, n in enumerate(NAMES) if n["name"] == name)
    return k, Z[f"f{k}_jpeg"].tobytes()


def pil_matches(k, a):
    """a (H, W, 3) uint8 equals Pillow's decode of fixture k (the full array, or its SHA-256 and sampled rows)."""
    if f"f{k}_pil" in Z.files:
        return np.array_equal(a, Z[f"f{k}_pil"])
    return (np.array_equal(a[Z[f"f{k}_rows"]], Z[f"f{k}_rowdata"])
            and hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest() == Z[f"f{k}_sha"].tobytes())


def segment(data, marker):
    """Offset of the first segment with this marker byte (the 0xFF of the marker)."""
    i = 2
    while data[i + 1] != marker:
        i += 2 + struct.unpack(">H", data[i + 2: i + 4])[0]
    return i


def test_reference_decoder_equals_pillow_over_the_corpus():
    supported = [(k, n) for k, n in enumerate(NAMES) if n["outcome"] == "ok"]
    assert len(supported) >= 30
    for k, n in supported:
        a = jpeg_ref.decode(Z[f"f{k}_jpeg"].tobytes(), n["name"])
        assert a.shape == (n["h"], n["w"], 3) and a.dtype == np.uint8, n
        assert pil_matches(k, a), n["name"]


def test_parser_tables_segments_and_mcu_counts():
    from macaw_llm_b200 import jpeg as J

    _, d = fixture("s224_q75_sub2_rst_rows1")
    f = J.parse(d)
    assert (f.width, f.height, f.hmax, f.vmax, f.mcus_x, f.mcus_y) == (224, 224, 2, 2, 14, 14)
    assert [(c.h, c.v, c.bw, c.bh) for c in f.comps] == [(2, 2, 28, 28), (1, 1, 14, 14), (1, 1, 14, 14)]
    assert f.restart_interval == 14 and len(f.segments) == 14
    assert [s[2:] for s in f.segments] == [(14 * r, 14) for r in range(14)]
    for (s0, s1, _, _), nxt in zip(f.segments, f.segments[1:]):
        assert d[s1] == 0xFF and 0xD0 <= d[s1 + 1] <= 0xD7 and nxt[0] == s1 + 2
    assert f.segments[-1][1] == f.scan[1] and d[f.scan[1]: f.scan[1] + 2] == b"\xff\xd9"
    # Annex K luminance DC table (Pillow's default): code 00 -> category 0, 2 bits; 9-bit codes need maxcode
    dc = f.dc[f.comps[0].td]
    assert dc.look[0] == (2 << 8) | 0 and dc.look[0x3F] == (2 << 8) | 0 and dc.look[0x40] == (3 << 8) | 1
    assert dc.maxcode[2] == 0 and dc.maxcode[3] == 6 and dc.maxcode[9] == 510 and dc.maxcode[17] == 0xFFFFF
    assert f.quant[0][0] == 8 and f.quant[0].dtype == np.uint16   # Annex K luminance 16 at quality 75 -> 8

    _, d = fixture("s224_q75_sub1_rst_blocks1")
    f = J.parse(d)
    assert (f.hmax, f.vmax, f.mcus_x, f.mcus_y, f.restart_interval) == (2, 1, 14, 28, 1)
    assert len(f.segments) == 14 * 28 and all(s[3] == 1 for s in f.segments)
    _, d = fixture("s33x65_q75_gray")
    f = J.parse(d)
    assert len(f.comps) == 1 and (f.mcus_x, f.mcus_y) == (9, 5) and f.segments == [(f.scan[0], f.scan[1], 0, 45)]
    _, d = fixture("s224_qt16_sub2")
    f = J.parse(d)
    assert d[segment(d, 0xC1) + 1] == 0xC1 and int(f.quant[0].max()) == 300 and int(f.quant[1].max()) == 400
    _, d = fixture("s479x641_q50_sub0_opt")
    f = J.parse(d)
    assert (f.mcus_x, f.mcus_y, len(f.segments)) == (81, 60, 1) and f.segments[0][3] == 81 * 60


def test_pack_layout():
    from macaw_llm_b200 import jpeg as J

    infos = [J.parse(fixture(n)[1], n) for n in ("s224_q75_sub2_rst_rows1", "s7x9_q75_gray", "s15x17_q75_sub1")]
    data, desc, z = J.pack(infos)
    im = desc[z["off"]["images"]:z["off"]["images"] + 3 * J.IMAGE_DT.itemsize].view(J.IMAGE_DT)
    sg = desc[z["off"]["segments"]:z["off"]["segments"] + z["n_segments"] * J.SEGMENT_DT.itemsize].view(J.SEGMENT_DT)
    assert z["n_segments"] == 14 + 1 + 1 and list(im["seg0"]) == [0, 14, 15] and list(im["n_seg"]) == [14, 1, 1]
    for k, f in enumerate(infos):
        for j, (s0, s1, m0, nm) in enumerate(f.segments):
            s = sg[im["seg0"][k] + j]
            assert s["image"] == k and (s["mcu0"], s["n_mcu"]) == (m0, nm)
            assert data[s["offset"]: s["offset"] + s["n_bytes"]].tobytes() == f.data[s0:s1]
    assert list(im["n_comp"]) == [3, 1, 3] and list(im["out_ld"]) == [3 * 224, 3 * 9, 3 * 17]
    assert im["coef_off"][1][0] == 64 * (28 * 28 + 2 * 14 * 14) and im["coef_off"][0][1] == 64 * 28 * 28
    assert z["max_blocks"] == 28 * 28 and z["max_pixels"] == 224 * 224 and z["n_huff"] == 4 and z["n_quant"] == 2
    assert all(o % 16 == 0 for o, _, _ in z["outs"])


def _patch(d, off, new):
    return d[:off] + new + d[off + len(new):]


def test_refusals_and_errors_name_the_feature():
    from macaw_llm_b200 import jpeg as J

    for n in NAMES:
        if n["outcome"] != "ok":
            _, d = fixture(n["name"])
            with pytest.raises({"ValueError": ValueError, "NotImplementedError": NotImplementedError}[n["outcome"]]):
                J.parse(d, n["name"])
    with pytest.raises(NotImplementedError, match="progressive"):
        J.parse(fixture("bad_progressive")[1])
    with pytest.raises(NotImplementedError, match="CMYK"):
        J.parse(fixture("bad_cmyk")[1])
    with pytest.raises(ValueError, match="truncated"):
        J.parse(fixture("bad_truncated")[1])
    _, d = fixture("s33x65_q75_sub2")
    sof = segment(d, 0xC0)
    with pytest.raises(NotImplementedError, match="arithmetic"):
        J.parse(_patch(d, sof + 1, b"\xc9"))
    with pytest.raises(NotImplementedError, match="lossless"):
        J.parse(_patch(d, sof + 1, b"\xc3"))
    with pytest.raises(NotImplementedError, match="12-bit"):
        J.parse(_patch(d, sof + 4, b"\x0c"))
    with pytest.raises(NotImplementedError, match="DNL"):
        J.parse(_patch(d, sof + 5, b"\x00\x00"))
    for off, hv in ((11, b"\x41"), (11, b"\x12"), (14, b"\x21")):   # 4:1:1, 4:4:0, chroma 2x1
        with pytest.raises(NotImplementedError, match="sampling factors"):
            J.parse(_patch(d, sof + off, hv))
    with pytest.raises(NotImplementedError, match="RGB"):   # component ids 'R', 'G', 'B' and no JFIF marker
        app0 = segment(d, 0xE0)
        ln = struct.unpack(">H", d[app0 + 2: app0 + 4])[0]
        e = d[:app0] + b"\xff\xe1" + d[app0 + 2:]   # APP0 -> APP1: no JFIF marker
        assert ln == 16
        s = segment(e, 0xC0)
        e = _patch(e, s + 10, b"R")
        e = _patch(e, s + 13, b"G")
        e = _patch(e, s + 16, b"B")
        sos = segment(e, 0xDA)
        e = _patch(_patch(_patch(e, sos + 5, b"R"), sos + 7, b"G"), sos + 9, b"B")
        J.parse(e)
    adobe0 = d[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + d[2:]
    adobe0 = adobe0[:segment(adobe0, 0xE0)] + adobe0[segment(adobe0, 0xE0) + 18:]   # drop the 16-byte JFIF APP0
    with pytest.raises(NotImplementedError, match="Adobe transform 0"):
        J.parse(adobe0)
    assert J.parse(_patch(adobe0, 2 + 4 + 11, b"\x01")).width == 65      # Adobe transform 1 is YCbCr
    assert J.parse(d[:2] + b"\xff\xfe\x00\x05abc" + d[2:]).width == 65   # COM is skipped
    with pytest.raises(NotImplementedError, match="multi-scan"):
        sos = segment(d, 0xDA)
        ln = struct.unpack(">H", d[sos + 2: sos + 4])[0]
        J.parse(d[:-2] + d[sos: sos + 2 + ln] + b"\x00\xff\xd9")
    with pytest.raises(NotImplementedError, match="multi-scan"):   # a scan holding one of three components
        sos = segment(d, 0xDA)
        J.parse(d[:sos] + b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00" + d[sos + 14:])
    with pytest.raises(ValueError, match="not a JPEG"):
        J.parse(b"\x89PNG\r\n\x1a\n" + d)
    _, r = fixture("s224_q75_sub2_rst_rows1")
    dri = segment(r, 0xDD)
    with pytest.raises(ValueError, match="restart markers"):
        J.parse(_patch(r, dri + 4, b"\x00\x1c"))   # 28 MCUs per interval: 7 segments expected, 14 present
    with pytest.raises(ValueError, match="restart markers out of sequence"):
        f = J.parse(r)
        J.parse(_patch(r, f.segments[2][1] + 1, b"\xd5"))
    with pytest.raises(TypeError):
        J.read_item(3.0, 0)


def corrupt(d: bytes) -> bytes:
    """Flip bytes in the middle of the scan without creating or breaking a marker."""
    from macaw_llm_b200 import jpeg as J

    f = J.parse(d)
    s0, s1 = f.segments[0][:2]
    b = bytearray(d)
    for p in range(s0 + (s1 - s0) // 3, s0 + (s1 - s0) // 3 + 40, 5):
        if 0xFF not in b[p - 1: p + 2] and (b[p] ^ 0x5A) != 0xFF:
            b[p] ^= 0x5A
    return bytes(b)


def test_corrupt_scan_is_detected_by_the_reference():
    """The bytes test_jpeg_gpu.py decodes to provoke a status-word error: the reference decoder rejects them too."""
    for name in ("s224_q95_sub2", "s300x400_q75_sub1"):
        bad = corrupt(fixture(name)[1])
        with pytest.raises(ValueError):
            jpeg_ref.decode(bad)


def test_descriptor_structs_match_c_layout():
    from macaw_llm_b200 import _lib

    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "macaw_b200.h"
int main(void){ printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(mm_jpeg_args), offsetof(mm_jpeg_args, status),
  offsetof(mm_jpeg_args, max_pixels), sizeof(mm_jpeg_image), offsetof(mm_jpeg_image, coef_off),
  offsetof(mm_jpeg_image, out_ld), sizeof(mm_jpeg_segment), sizeof(mm_jpeg_huff), offsetof(mm_jpeg_huff, huffval)); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(d, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = list(map(int, subprocess.run([exe], capture_output=True, text=True).stdout.split()))
    want = [ctypes.sizeof(_lib.JpegArgs), _lib.JpegArgs.status.offset, _lib.JpegArgs.max_pixels.offset,
            ctypes.sizeof(_lib.JpegImage), _lib.JpegImage.coef_off.offset, _lib.JpegImage.out_ld.offset,
            ctypes.sizeof(_lib.JpegSegment), ctypes.sizeof(_lib.JpegHuff), _lib.JpegHuff.huffval.offset]
    assert got == want


def test_decode_argument_errors_without_a_gpu():
    from macaw_llm_b200 import _lib

    lib = _lib.load()
    assert lib.mm_jpeg_decode(None, None) != 0 and b"null" in lib.mm_last_error()
    a = _lib.JpegArgs()
    assert lib.mm_jpeg_decode(ctypes.byref(a), None) != 0 and b"null" in lib.mm_last_error()
    for f in ("data", "images", "segments", "huff", "quant", "coef", "planes", "out", "status"):
        setattr(a, f, 4096)
    assert lib.mm_jpeg_decode(ctypes.byref(a), None) != 0 and b"bad sizes" in lib.mm_last_error()
    a.n_images = a.n_segments = a.n_huff = a.n_quant = a.max_blocks = a.max_pixels = 1
    a.coef_elems = a.plane_bytes = a.out_bytes = 64
    a.n_segments = 0
    assert lib.mm_jpeg_decode(ctypes.byref(a), None) != 0 and b"bad sizes" in lib.mm_last_error()
    a.n_segments, a.coef = 1, 4098
    assert lib.mm_jpeg_decode(ctypes.byref(a), None) != 0 and b"misaligned" in lib.mm_last_error()


def test_reference_transform_fixture_follows_from_the_decode():
    """The stored `_transform(224)` crops equal the reference decode resized by the host-side emulation of the resize
    kernels (tests/test_inputs.py), grayscale included: resampling L then converting equals resampling the replicated plane."""
    from macaw_llm_b200 import inputs as I
    from tests.golden.make_jpeg_golden import TF_ROWS
    from tests.test_inputs import _emulate

    for tag in ("color", "gray"):
        k = int(Z[f"tf_{tag}_file"])
        crop = _emulate(jpeg_ref.decode(Z[f"f{k}_jpeg"].tobytes()), I)
        assert hashlib.sha256(np.ascontiguousarray(crop).tobytes()).digest() == Z[f"tf_{tag}_u8_sha"].tobytes(), tag
        assert np.array_equal(crop[TF_ROWS], Z[f"tf_{tag}_u8_rows"]), tag
        mean, std = MEAN_STD
        f32 = ((crop[TF_ROWS].astype(np.float32) / 255.0).transpose(2, 0, 1) - mean[:, None, None]) / std[:, None, None]
        assert np.abs(f32 - Z[f"tf_{tag}_f32_rows"]).max() < 1e-6, tag
