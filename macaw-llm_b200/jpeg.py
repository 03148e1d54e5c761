"""JPEG decoding on the device, bit-exact with Pillow's default decoder (libjpeg-turbo: ISLOW integer IDCT, fancy
upsampling, fixed-point YCbCr -> RGB).

The host side lives here: markers are parsed in Python, entropy-coded segments (restart intervals, or the whole scan) are
found with a vectorised search for RST markers, Huffman tables are expanded into libjpeg's lookahead / maxcode form, and
a batch of files is packed into one page-locked byte buffer plus one descriptor buffer (two host-to-device copies).
`mm_jpeg_decode` (csrc/jpeg.cu) then runs three kernels: entropy decode (one thread per segment), dequantise + IDCT,
upsample + colour convert.  Each image gets a status word; it is read with one synchronise per batch.

Supported: sequential Huffman JPEGs (SOF0 / SOF1), 8-bit samples, one scan; grayscale, or YCbCr with luma sampling 1x1,
2x1 or 2x2 and chroma 1x1; restart intervals; any image size.  Other coding processes, CMYK / RGB colour spaces, other
sampling factors, multi-scan files and DNL raise NotImplementedError naming the feature; malformed or truncated files raise
ValueError.  There is no host fallback: decode such a file on the host and pass the array instead.
"""
from __future__ import annotations

import functools
import os
from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np

from . import _lib

# position in the 8x8 block (row-major) of the k-th coefficient in zigzag order
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39,
                   46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)

_SOF_NAMES = {0xC2: "progressive JPEG", 0xC3: "lossless JPEG", 0xC5: "differential sequential JPEG",
              0xC6: "differential progressive JPEG", 0xC7: "differential lossless JPEG",
              0xC9: "arithmetic-coded JPEG", 0xCA: "arithmetic-coded progressive JPEG",
              0xCB: "arithmetic-coded lossless JPEG", 0xCD: "arithmetic-coded differential JPEG",
              0xCE: "arithmetic-coded differential progressive JPEG",
              0xCF: "arithmetic-coded differential lossless JPEG"}

# status-word bits set by the entropy kernel (csrc/jpeg.cu)
STATUS_BITS = {1: "invalid Huffman code", 2: "coefficient run past 63", 4: "entropy-coded segment ends early",
               8: "bytes left over after the last MCU of a segment", 16: "bad byte stuffing in the scan",
               32: "descriptor out of range"}


@dataclass(frozen=True)
class HuffTable:
    """libjpeg's derived decoding table (jdhuff.c jpeg_make_d_derived_tbl): for codes of up to 8 bits a 256-entry
    lookahead `(length << 8) | symbol` (0 = longer code), for longer codes maxcode[l] / valoffset[l] over huffval."""
    maxcode: np.ndarray    # int32 [18]
    valoffset: np.ndarray  # int32 [18]
    look: np.ndarray       # uint16 [256]
    huffval: np.ndarray    # uint8 [256]


@functools.lru_cache(maxsize=256)
def huff_table(counts: bytes, symbols: bytes, is_dc: bool) -> HuffTable:
    """Expand one DHT table (16 code-length counts and the symbols); raises ValueError on a table libjpeg refuses."""
    bits = [0] + list(counts)
    if sum(bits) > 256 or len(symbols) != sum(bits):
        raise ValueError("bad Huffman table")
    huffsize = [l for l in range(1, 17) for _ in range(bits[l])] + [0]
    huffcode = [0] * len(huffsize)
    code, si, p = 0, huffsize[0], 0
    while huffsize[p]:
        while huffsize[p] == si:
            huffcode[p] = code
            p += 1
            code += 1
        if code >= (1 << si):
            raise ValueError("bad Huffman table")
        code <<= 1
        si += 1
    maxcode = np.full(18, -1, np.int32)
    valoffset = np.zeros(18, np.int32)
    p = 0
    for l in range(1, 17):
        if bits[l]:
            valoffset[l] = p - huffcode[p]
            p += bits[l]
            maxcode[l] = huffcode[p - 1]
    maxcode[17] = 0xFFFFF
    look = np.zeros(256, np.uint16)
    p = 0
    for l in range(1, 9):
        for _ in range(bits[l]):
            lb = huffcode[p] << (8 - l)
            look[lb: lb + (1 << (8 - l))] = (l << 8) | symbols[p]
            p += 1
    if is_dc and any(s > 15 for s in symbols):
        raise ValueError("bad Huffman table")
    hv = np.zeros(256, np.uint8)
    hv[: len(symbols)] = np.frombuffer(symbols, np.uint8)
    return HuffTable(maxcode, valoffset, look, hv)


@dataclass
class Component:
    cid: int
    h: int
    v: int
    tq: int
    td: int = 0     # DC table id (SOS)
    ta: int = 0     # AC table id
    bw: int = 0     # blocks per row / column, whole MCUs
    bh: int = 0


@dataclass
class JpegInfo:
    """One parsed file: geometry, tables, and the entropy-coded segments as (start, end, first MCU, MCU count) byte ranges
    of `data` (markers and trailing fill bytes excluded)."""
    name: str
    data: bytes
    width: int = 0
    height: int = 0
    comps: List[Component] = field(default_factory=list)
    hmax: int = 1
    vmax: int = 1
    mcus_x: int = 0
    mcus_y: int = 0
    restart_interval: int = 0
    quant: dict = field(default_factory=dict)    # id -> uint16 [64], natural order
    dc: dict = field(default_factory=dict)       # id -> HuffTable
    ac: dict = field(default_factory=dict)
    scan: Tuple[int, int] = (0, 0)
    segments: List[Tuple[int, int, int, int]] = field(default_factory=list)

    @property
    def n_mcu(self) -> int:
        return self.mcus_x * self.mcus_y


def _u16(d: bytes, i: int) -> int:
    return (d[i] << 8) | d[i + 1]


def parse(data: bytes, name: str = "<bytes>") -> JpegInfo:
    """Parse the markers of one file and locate its entropy-coded segments."""
    info = JpegInfo(name, bytes(data))
    d = info.data
    n = len(d)

    def bad(msg):
        return ValueError(f"{name}: {msg}")

    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise bad("not a JPEG file (no SOI marker)")
    i, sof, jfif, adobe = 2, None, False, None
    while True:
        if i >= n:
            raise bad("truncated JPEG file (no scan)")
        if d[i] != 0xFF:
            raise bad(f"expected a marker at byte {i}")
        while i < n and d[i] == 0xFF:
            i += 1
        if i >= n:
            raise bad("truncated JPEG file (no scan)")
        m = d[i]
        i += 1
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise bad(f"unexpected marker 0xFF{m:02X} before the scan")
        if i + 2 > n:
            raise bad("truncated JPEG file")
        ln = _u16(d, i)
        if ln < 2 or i + ln > n:
            raise bad(f"truncated JPEG file (segment 0xFF{m:02X})")
        seg = d[i + 2: i + ln]
        i += ln
        if m in _SOF_NAMES:
            raise NotImplementedError(f"{name}: {_SOF_NAMES[m]} is not supported (sequential Huffman JPEG only)")
        if m == 0xCC:
            raise NotImplementedError(f"{name}: arithmetic-coded JPEG is not supported")
        if m == 0xDC:
            raise NotImplementedError(f"{name}: DNL marker is not supported")
        if m in (0xC0, 0xC1):
            if sof is not None:
                raise bad("more than one SOF marker")
            sof = m
            if len(seg) < 6:
                raise bad("short SOF segment")
            prec, info.height, info.width, nc = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if prec == 12:
                raise NotImplementedError(f"{name}: 12-bit samples are not supported")
            if prec != 8:
                raise bad(f"unsupported sample precision {prec}")
            if info.height == 0:
                raise NotImplementedError(f"{name}: DNL (image height defined after the scan) is not supported")
            if info.width == 0:
                raise bad("image width is 0")
            if len(seg) != 6 + 3 * nc:
                raise bad("bad SOF length")
            if nc == 4:
                raise NotImplementedError(f"{name}: CMYK / YCCK JPEG is not supported")
            if nc not in (1, 3):
                raise NotImplementedError(f"{name}: {nc}-component JPEG is not supported")
            for k in range(nc):
                cid, hv, tq = seg[6 + 3 * k], seg[7 + 3 * k], seg[8 + 3 * k]
                h, v = hv >> 4, hv & 15
                if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
                    raise bad("bad component sampling factors or quantisation table")
                info.comps.append(Component(cid, h, v, tq))
        elif m == 0xC4:
            p = 0
            while p < len(seg):
                if p + 17 > len(seg):
                    raise bad("short DHT segment")
                tc, th = seg[p] >> 4, seg[p] & 15
                cnt = bytes(seg[p + 1: p + 17])
                ns = sum(cnt)
                if tc > 1 or th > 3 or p + 17 + ns > len(seg):
                    raise bad("bad DHT segment")
                try:
                    t = huff_table(cnt, bytes(seg[p + 17: p + 17 + ns]), tc == 0)
                except ValueError:
                    raise bad("bad Huffman table") from None
                (info.dc if tc == 0 else info.ac)[th] = t
                p += 17 + ns
        elif m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                sz = 64 * (pq + 1)
                if pq > 1 or tq > 3 or p + 1 + sz > len(seg):
                    raise bad("bad DQT segment")
                raw = np.frombuffer(seg, np.uint8 if pq == 0 else ">u2", count=64, offset=p + 1).astype(np.uint16)
                q = np.zeros(64, np.uint16)
                q[ZIGZAG] = raw
                info.quant[tq] = q
                p += 1 + sz
        elif m == 0xDD:
            if len(seg) != 2:
                raise bad("bad DRI segment")
            info.restart_interval = _u16(seg, 0)
        elif m == 0xE0:
            if len(seg) >= 14 and seg[:5] == b"JFIF\x00":
                jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            break
        else:
            raise bad(f"unknown marker 0xFF{m:02X}")

    # ---- SOS
    if sof is None:
        raise bad("scan before SOF")
    nc = len(info.comps)
    if len(seg) < 1 or len(seg) != 4 + 2 * seg[0]:
        raise bad("bad SOS segment")
    ns = seg[0]
    if ns != nc:
        raise NotImplementedError(f"{name}: multi-scan sequential JPEG is not supported (scan holds {ns} of {nc} components)")
    ids = [c.cid for c in info.comps]
    for k in range(ns):
        cs, t = seg[1 + 2 * k], seg[2 + 2 * k]
        if ids.count(cs) != 1 or ids.index(cs) != k:
            raise bad("scan component selectors do not match the frame")
        info.comps[k].td, info.comps[k].ta = t >> 4, t & 15
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if ss != 0 or se != 63 or ahal != 0:
        raise bad("sequential scan with spectral selection / successive approximation")
    # libjpeg's colour-space guess (jdapimin.c default_decompress_parms): only YCbCr is decoded here
    if nc == 3:
        if not jfif and adobe is not None and adobe == 0:
            raise NotImplementedError(f"{name}: Adobe transform 0 (RGB JPEG) is not supported")
        if not jfif and adobe is None and ids == [82, 71, 66]:
            raise NotImplementedError(f"{name}: RGB JPEG (component ids 'R', 'G', 'B') is not supported")
        y, cb, cr = info.comps
        if (cb.h, cb.v, cr.h, cr.v) != (1, 1, 1, 1) or (y.h, y.v) not in ((1, 1), (2, 1), (2, 2)):
            s = " ".join(f"{c.h}x{c.v}" for c in info.comps)
            raise NotImplementedError(f"{name}: sampling factors {s} are not supported (4:4:4, 4:2:2, 4:2:0 only)")
        info.hmax, info.vmax = y.h, y.v
        info.mcus_x = -(-info.width // (8 * y.h))
        info.mcus_y = -(-info.height // (8 * y.v))
        for c in info.comps:
            c.bw, c.bh = info.mcus_x * c.h, info.mcus_y * c.v
    else:   # one non-interleaved scan: one block per MCU, whatever the declared sampling factors
        c = info.comps[0]
        c.h = c.v = 1
        info.mcus_x, info.mcus_y = -(-info.width // 8), -(-info.height // 8)
        c.bw, c.bh = info.mcus_x, info.mcus_y
    for c in info.comps:
        if c.tq not in info.quant:
            raise bad(f"quantisation table {c.tq} is not defined")
        if c.td not in info.dc or c.ta not in info.ac:
            raise bad("scan uses an undefined Huffman table")

    # ---- entropy-coded data: vectorised search for the markers that end the scan or split it at restarts
    start = i
    b = np.frombuffer(d, np.uint8)
    ff = np.flatnonzero(b[start:-1] == 0xFF) + start
    nxt = b[ff + 1]
    marks = ff[(nxt != 0x00) & (nxt != 0xFF)]
    kinds = b[marks + 1]
    rst = (kinds >= 0xD0) & (kinds <= 0xD7)
    ends = np.flatnonzero(~rst)
    if ends.size == 0:
        raise bad("truncated JPEG file (scan has no end)")
    end_mark = int(marks[ends[0]])
    rsts = marks[: ends[0]]
    got = kinds[: ends[0]]
    if got.size and not np.array_equal(got, 0xD0 + (np.arange(got.size) % 8)):
        raise bad("restart markers out of sequence")
    bounds = [start] + [int(r) + 2 for r in rsts]
    stops = [int(r) for r in rsts] + [end_mark]
    total = info.n_mcu
    ri = info.restart_interval
    want = 1 if ri == 0 else -(-total // ri)
    if len(bounds) != want:
        raise bad(f"{len(bounds) - 1} restart markers in the scan, expected {want - 1}")
    for k, (s0, s1) in enumerate(zip(bounds, stops)):
        while s1 > s0 and d[s1 - 1] == 0xFF:   # fill bytes before a marker
            s1 -= 1
        m0 = k * ri if ri else 0
        info.segments.append((s0, s1, m0, (min(ri, total - m0) if ri else total)))
    info.scan = (start, end_mark)

    # ---- after the scan: only EOI (or tables / APPn / COM) may follow
    i = end_mark
    while True:
        while i < n and d[i] == 0xFF:
            i += 1
        if i >= n:
            raise bad("truncated JPEG file (no EOI marker)")
        m = d[i]
        i += 1
        if m == 0xD9:
            break
        if m == 0xDA:
            raise NotImplementedError(f"{name}: multi-scan sequential JPEG is not supported")
        if m == 0xDC:
            raise NotImplementedError(f"{name}: DNL marker is not supported")
        if m in (0xC4, 0xDB, 0xDD, 0xFE) or 0xE0 <= m <= 0xEF:
            if i + 2 > n or i + _u16(d, i) > n:
                raise bad("truncated JPEG file")
            i += _u16(d, i)
            continue
        raise bad(f"unexpected marker 0xFF{m:02X} after the scan")
    return info


def read_item(item, k: int) -> Tuple[bytes, str]:
    """(bytes, name) of one item: `bytes` / `bytearray` / `memoryview`, or a `str` / `os.PathLike` path."""
    if isinstance(item, (bytes, bytearray, memoryview)):
        return bytes(item), f"<bytes #{k}>"
    if isinstance(item, (str, os.PathLike)):
        with open(item, "rb") as f:
            return f.read(), os.fspath(item)
    raise TypeError(f"JPEG item #{k}: expected bytes, str or os.PathLike, got {type(item).__name__}")


def is_item(x) -> bool:
    return isinstance(x, (bytes, bytearray, memoryview, str, os.PathLike))


# ---------------------------------------------------------------------------------------------------- batch packing
IMAGE_DT = np.dtype(_lib.JpegImage)
SEGMENT_DT = np.dtype(_lib.JpegSegment)
HUFF_DT = np.dtype(_lib.JpegHuff)


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def pack(infos: Sequence[JpegInfo]):
    """Host-side batch layout: (scan bytes uint8, descriptor bytes uint8, sizes dict).  Offsets of the four descriptor
    tables inside the descriptor buffer, the coefficient / plane / output element counts, and each image's output
    (offset, H, W) are in the dict."""
    n_img = len(infos)
    n_seg = sum(len(f.segments) for f in infos)
    images = np.zeros(n_img, IMAGE_DT)
    segs = np.zeros(n_seg, SEGMENT_DT)
    huffs, quants, hkey, qkey = [], [], {}, {}
    scans, data_off, coef_off, plane_off, out_off, s = [], 0, 0, 0, 0, 0
    outs, max_blocks, max_pixels = [], 1, 1
    for k, f in enumerate(infos):
        im = images[k]
        im["width"], im["height"], im["n_comp"] = f.width, f.height, len(f.comps)
        im["hmax"], im["vmax"], im["mcus_x"], im["mcus_y"] = f.hmax, f.vmax, f.mcus_x, f.mcus_y
        im["seg0"], im["n_seg"] = s, len(f.segments)
        for c, comp in enumerate(f.comps):
            for kind, tid, tabs in (("huff_dc", comp.td, f.dc), ("huff_ac", comp.ta, f.ac)):
                t = tabs[tid]
                if id(t) not in hkey:
                    hkey[id(t)] = len(huffs)
                    huffs.append(t)
                im[kind][c] = hkey[id(t)]
            q = f.quant[comp.tq].tobytes()
            if q not in qkey:
                qkey[q] = len(quants)
                quants.append(q)
            im["quant"][c] = qkey[q]
            im["bw"][c], im["bh"][c] = comp.bw, comp.bh
            im["coef_off"][c] = coef_off
            im["plane_off"][c] = plane_off
            nb = comp.bw * comp.bh
            coef_off += nb * 64
            plane_off += nb * 64
            max_blocks = max(max_blocks, nb)
        im["out_off"], im["out_ld"] = out_off, 3 * f.width
        outs.append((out_off, f.height, f.width))
        out_off += _align(3 * f.width * f.height, 16)
        max_pixels = max(max_pixels, f.width * f.height)
        a, b = f.scan
        scans.append(np.frombuffer(f.data, np.uint8, count=b - a, offset=a))
        for (s0, s1, m0, nm) in f.segments:
            segs[s] = (data_off + s0 - a, s1 - s0, k, m0, nm)
            s += 1
        data_off += b - a
    huff = np.zeros(len(huffs), HUFF_DT)
    for j, t in enumerate(huffs):
        huff[j] = (t.maxcode, t.valoffset, t.look, t.huffval)
    quant = np.frombuffer(b"".join(quants), np.uint16)
    parts, off = [], {}
    pos = 0
    for key, arr in (("images", images), ("segments", segs), ("huff", huff), ("quant", quant)):
        pos = _align(pos, 16)
        off[key] = pos
        raw = arr.view(np.uint8).reshape(-1)
        parts.append((pos, raw))
        pos += raw.size
    desc = np.zeros(_align(pos, 16), np.uint8)
    for p, raw in parts:
        desc[p: p + raw.size] = raw
    data = np.concatenate(scans)
    sizes = dict(off=off, data_bytes=int(data.size), n_images=n_img, n_segments=n_seg, n_huff=len(huffs), n_quant=len(quants), coef=coef_off,
                 planes=plane_off, out=max(out_off, 16), max_blocks=max_blocks, max_pixels=max_pixels, outs=outs)
    return data, desc, sizes


MAX_BATCH = 4096   # images per mm_jpeg_decode call (its IDCT grid has 3 rows per image)


def decode(items: Sequence, device) -> list:
    """Decode a batch of JPEG files on `device`: a list of uint8 (H, W, 3) device tensors (grayscale files have their
    plane replicated).  One host-to-device copy of the scan bytes, one of the descriptors, one `mm_jpeg_decode` call and
    one synchronise to read the per-image status words (per 4096 files)."""
    infos = []
    for k, it in enumerate(items):
        raw, name = read_item(it, k)
        infos.append(parse(raw, name))
    out = []
    for c0 in range(0, len(infos), MAX_BATCH):
        out += _decode_parsed(infos[c0: c0 + MAX_BATCH], device)
    return out


def _decode_parsed(infos: Sequence[JpegInfo], device) -> list:
    import torch

    from . import ops

    dev = torch.device(device)
    data, desc, z = pack(infos)
    h_data = torch.empty(max(data.size, 16), dtype=torch.uint8, pin_memory=True)
    h_data[: data.size].numpy()[:] = data
    h_desc = torch.empty(desc.size, dtype=torch.uint8, pin_memory=True)
    h_desc.numpy()[:] = desc
    with torch.cuda.device(dev):
        out, status = ops.jpeg_decode(h_data.to(dev, non_blocking=True), h_desc.to(dev, non_blocking=True), z)
        st = status.cpu().numpy()   # the batch's one synchronise; the page-locked sources stay alive until here
    bad = np.flatnonzero(st)
    if bad.size:
        k = int(bad[0])
        why = ", ".join(v for b, v in STATUS_BITS.items() if st[k] & b)
        raise ValueError(f"{infos[k].name}: corrupt JPEG data ({why})")
    return [out[o: o + h * w * 3].view(h, w, 3) for (o, h, w) in z["outs"]]
