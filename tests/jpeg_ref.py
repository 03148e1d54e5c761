"""numpy restatement of libjpeg-turbo's default decode, the arithmetic the device decoder (csrc/jpeg.cu) reproduces:

  entropy decode   jdhuff.c: derived tables (lookahead + maxcode), DC prediction reset at each restart, EOB / ZRL
  IDCT             jidctint.c jpeg_idct_islow: CONST_BITS 13, PASS1_BITS 2, the range_limit table on a 10-bit masked index
  upsampling       jdsample.c h2v1 / h2v2 fancy (triangle) filters, edges replicated at the downsampled size; box
                   replication when the downsampled width is <= 2 (jinit_upsampler)
  colour           jdcolor.c ycc_rgb_convert, 16-bit fixed point

The marker parser is the package's (macaw_llm_b200.jpeg.parse).  numpy only: no Pillow, so the GPU tier can use it too.
decode(bytes) -> uint8 (H, W, 3).
"""
from __future__ import annotations

import numpy as np

from macaw_llm_b200 import jpeg as J


def _bits16(seg: bytes):
    """Unstuffed segment -> (peek16 list: the 16 bits starting at every bit position, number of real bits)."""
    b = np.frombuffer(seg, np.uint8)
    if b.size:
        stuffed = np.zeros(b.size, bool)
        stuffed[1:] = (b[1:] == 0) & (b[:-1] == 0xFF)
        b = b[~stuffed]
    nbits = 8 * b.size
    p = np.concatenate([b, np.zeros(10, np.uint8)]).astype(np.int64)
    w = (p[:-2] << 16) | (p[1:-1] << 8) | p[2:]                # 24-bit window at each byte
    i = np.arange(nbits + 64)
    peek = (w[i >> 3] >> (8 - (i & 7))) & 0xFFFF
    return peek.tolist(), nbits


def entropy_decode(info: J.JpegInfo):
    """-> per component int16 (bh, bw, 8, 8) natural-order coefficients."""
    coefs = [np.zeros((c.bh, c.bw, 64), np.int32) for c in info.comps]
    zz = J.ZIGZAG.tolist()
    tabs = [(info.dc[c.td], info.ac[c.ta]) for c in info.comps]
    tabs = [tuple((t.look.tolist(), t.maxcode.tolist(), t.valoffset.tolist(), t.huffval.tolist()) for t in pair)
            for pair in tabs]
    for (s0, s1, m0, nm) in info.segments:
        peek, nbits = _bits16(info.data[s0:s1])
        pos = 0
        pred = [0] * len(info.comps)

        def sym(tab):
            nonlocal pos
            look, maxcode, valoff, hv = tab
            v = peek[pos]
            e = look[v >> 8]
            if e:
                pos += e >> 8
                return e & 255
            l = 9
            code = v >> 7
            while l <= 16 and code > maxcode[l]:
                l += 1
                code = v >> (16 - l)
            if l > 16:
                raise ValueError("invalid Huffman code")
            pos += l
            return hv[(code + valoff[l]) & 255]

        def recv(s):
            nonlocal pos
            r = peek[pos] >> (16 - s)
            pos += s
            return r - ((1 << s) - 1) if r < (1 << (s - 1)) else r

        for m in range(m0, m0 + nm):
            my, mx = divmod(m, info.mcus_x)
            for ci, c in enumerate(info.comps):
                dct, act = tabs[ci]
                out = coefs[ci]
                for v in range(c.v):
                    for h in range(c.h):
                        blk = out[my * c.v + v, mx * c.h + h]
                        s = sym(dct)
                        pred[ci] += recv(s) if s else 0
                        blk[0] = ((pred[ci] + 32768) & 0xFFFF) - 32768    # stored as JCOEF (int16)
                        k = 1
                        while k < 64:
                            rs = sym(act)
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                if k > 63:
                                    raise ValueError("coefficient run past 63")
                                blk[zz[k]] = recv(s)
                                k += 1
                            elif r == 15:
                                k += 16
                                if k > 64:
                                    raise ValueError("coefficient run past 63")
                            else:
                                break
            if pos > nbits:
                raise ValueError("entropy-coded segment ends early")
        if nbits - pos >= 8:
            raise ValueError("bytes left over after the last MCU of a segment")
    return [c.reshape(c.shape[0], c.shape[1], 8, 8).astype(np.int16) for c in coefs]


FIX = dict(f0_298=2446, f0_390=3196, f0_541=4433, f0_765=6270, f0_899=7373, f1_175=9633, f1_501=12299, f1_847=15137,
           f1_961=16069, f2_053=16819, f2_562=20995, f3_072=25172)


def _idct_1d(x, shift):
    """One 8-point pass of jpeg_idct_islow over the last-but-one axis of x (int64): returns the 8 outputs DESCALEd."""
    F = FIX
    z2, z3 = x[2], x[6]
    z1 = (z2 + z3) * F["f0_541"]
    tmp2 = z1 + z3 * -F["f1_847"]
    tmp3 = z1 + z2 * F["f0_765"]
    z2, z3 = x[0], x[4]
    tmp0 = (z2 + z3) << 13
    tmp1 = (z2 - z3) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x[7], x[5], x[3], x[1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * F["f1_175"]
    tmp0 = tmp0 * F["f0_298"]
    tmp1 = tmp1 * F["f2_053"]
    tmp2 = tmp2 * F["f3_072"]
    tmp3 = tmp3 * F["f1_501"]
    z1 = z1 * -F["f0_899"]
    z2 = z2 * -F["f2_562"]
    z3 = z3 * -F["f1_961"] + z5
    z4 = z4 * -F["f0_390"] + z5
    tmp0 += z1 + z3
    tmp1 += z2 + z4
    tmp2 += z2 + z3
    tmp3 += z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + tmp3 + r) >> shift, (tmp11 + tmp2 + r) >> shift, (tmp12 + tmp1 + r) >> shift,
            (tmp13 + tmp0 + r) >> shift, (tmp13 - tmp0 + r) >> shift, (tmp12 - tmp1 + r) >> shift,
            (tmp11 - tmp2 + r) >> shift, (tmp10 - tmp3 + r) >> shift]


def range_limit(x):
    """jdmaster.c prepare_range_limit_table as the IDCT indexes it: table[(x) & 1023] of the post-IDCT half."""
    x = x & 1023
    return np.where(x < 128, x + 128, np.where(x < 512, 255, np.where(x < 896, 0, x - 896))).astype(np.uint8)


def idct_islow(coef, q):
    """coef int16 (..., 8, 8), q uint16 (64,) natural order -> uint8 samples (..., 8, 8)."""
    x = coef.astype(np.int64) * q.reshape(8, 8).astype(np.int64)
    cols = _idct_1d([x[..., k, :] for k in range(8)], 13 - 2)            # pass 1: columns, workspace[row][col]
    ws = np.stack(cols, axis=-2)
    rows = _idct_1d([ws[..., :, k] for k in range(8)], 13 + 2 + 3)       # pass 2: rows
    return range_limit(np.stack(rows, axis=-1))


def _plane(coef, q):
    bh, bw = coef.shape[:2]
    return idct_islow(coef, q).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(c, H, W, h, v):
    """Fancy upsampling (jdsample.c) of a chroma plane whose real size is (ceil(H / v), ceil(W / h)) -> (H, W) int64."""
    cw, ch = -(-W // h), -(-H // v)
    c = c[:ch, :cw].astype(np.int64)
    if h == 1 and v == 1:
        return c
    if cw <= 2:                                   # jinit_upsampler: box replication
        return np.repeat(np.repeat(c, v, 0), h, 1)[:H, :W]
    if v == 1:
        left = np.concatenate([c[:, :1], c[:, :-1]], 1)
        right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * c + left + 1) >> 2
        out[:, 1::2] = (3 * c + right + 2) >> 2
        return out[:H, :W]
    up = np.concatenate([c[:1], c[:-1]], 0)
    dn = np.concatenate([c[1:], c[-1:]], 0)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    for r0, nb in ((0, up), (1, dn)):
        s = 3 * c + nb
        left = np.concatenate([s[:, :1], s[:, :-1]], 1)
        right = np.concatenate([s[:, 1:], s[:, -1:]], 1)
        out[r0::2, 0::2] = (3 * s + left + 8) >> 4
        out[r0::2, 1::2] = (3 * s + right + 7) >> 4
    return out[:H, :W]


def ycc_to_rgb(y, cb, cr):
    cb = cb - 128
    cr = cr - 128
    r = y + ((91881 * cr + 32768) >> 16)
    g = y + ((-46802 * cr + -22554 * cb + 32768) >> 16)
    b = y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode_info(info: J.JpegInfo) -> np.ndarray:
    coefs = entropy_decode(info)
    H, W = info.height, info.width
    planes = [_plane(k, info.quant[c.tq]) for k, c in zip(coefs, info.comps)]
    y = planes[0][:H, :W].astype(np.int64)
    if len(planes) == 1:
        return np.repeat(y[..., None], 3, -1).astype(np.uint8)
    cb = upsample(planes[1], H, W, info.hmax, info.vmax)
    cr = upsample(planes[2], H, W, info.hmax, info.vmax)
    return ycc_to_rgb(y, cb, cr)


def decode(data: bytes, name: str = "<bytes>") -> np.ndarray:
    return decode_info(J.parse(data, name))
