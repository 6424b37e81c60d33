"""A numpy model of libjpeg-turbo's baseline encoder as cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) drives it
(3-channel BGR uint8, 4:2:0, Annex K Huffman tables, JFIF 1.01, no restart markers), stage by stage, so that the host
build of csrc/jpeg.cuh and the device can be held to each stage and the whole can be held to cv2's bytes.  Shared by
tests/test_jpeg_on_host.py, tests/test_gpu_jpeg.py and tests/golden/make_golden_jpeg.py; the test images are made here
from seeds."""
import os

import numpy as np

# ---------------------------------------------------------------------------------------------- tables (Annex K)
QUANT_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
QUANT_CHROMA = np.full(64, 99, np.int64)
QUANT_CHROMA[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 19, 24, 25, 26, 27]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 99, 47, 66, 99, 99]

DC_BITS = [[0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]]
DC_VALS = [list(range(12)), list(range(12))]
AC_BITS = [[0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]]
AC_VALS = [[
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
    0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
    0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
    0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa]]


def zigzag_order():
    """natural index of zigzag position k (jpeg_natural_order), walked along the anti-diagonals"""
    out = []
    for s in range(15):
        cells = [(i, s - i) for i in range(8) if 0 <= s - i < 8]
        if s % 2 == 0:
            cells = cells[::-1]          # even diagonals run from bottom-left to top-right
        out += [r * 8 + c for r, c in cells]
    return np.array(out, np.int64)


ZIGZAG = zigzag_order()


def huff_codes(bits, vals):
    """canonical Huffman codes (Annex C): symbol -> (code, length); length 0 = not in the table"""
    code, length = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            code[vals[k]], length[vals[k]] = c, ln
            c += 1
            k += 1
        c <<= 1
    return code, length


DC_CODES = [huff_codes(DC_BITS[t], DC_VALS[t]) for t in range(2)]
AC_CODES = [huff_codes(AC_BITS[t], AC_VALS[t]) for t in range(2)]


def quant_tables(quality):
    """jpeg_set_quality(cinfo, quality, force_baseline=TRUE): natural-order tables [2][64]"""
    q = 5000 // quality if quality < 50 else 200 - quality * 2
    out = []
    for base in (QUANT_LUMA, QUANT_CHROMA):
        t = (base * q + 50) // 100
        out.append(np.clip(t, 1, 255))
    return np.stack(out)


# ---------------------------------------------------------------------------------------------- header
def header(width, height, quality):
    """SOI, APP0 (JFIF 1.01, aspect 1:1), DQT x2, SOF0 (4:2:0), DHT x4 (DC0, AC0, DC1, AC1), SOS: libjpeg's order"""
    b = bytearray(b"\xff\xd8")
    b += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    for t, tab in enumerate(quant_tables(quality)):
        b += b"\xff\xdb\x00\x43" + bytes([t]) + bytes(int(v) for v in tab[ZIGZAG])
    b += b"\xff\xc0\x00\x11\x08" + height.to_bytes(2, "big") + width.to_bytes(2, "big")
    b += b"\x03\x01\x22\x00\x02\x11\x01\x03\x11\x01"
    for t in range(2):
        for cls, bits, vals in ((0, DC_BITS[t], DC_VALS[t]), (1, AC_BITS[t], AC_VALS[t])):
            b += b"\xff\xc4" + (3 + 16 + len(vals)).to_bytes(2, "big") + bytes([cls << 4 | t]) + bytes(bits) + bytes(vals)
    b += b"\xff\xda\x00\x0c\x03\x01\x00\x02\x11\x03\x11\x00\x3f\x00"
    return bytes(b)


# ---------------------------------------------------------------------------------------------- pixels -> samples
def _fix(x):
    return int(x * 65536 + 0.5)


def rgb_ycc(img):
    """jccolor.c rgb_ycc_convert on BGR uint8 [..., 3] -> Y, Cb, Cr int64 (16-bit fixed point, ONE_HALF - 1 on Cb/Cr)"""
    b, g, r = (img[..., i].astype(np.int64) for i in range(3))
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def downsample_h2v2(c):
    """h2v2_downsample on an even-sized plane: (sum of 2 x 2 + bias) >> 2, bias 1, 2, 1, 2, ... along each output row"""
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    bias = np.tile([1, 2], s.shape[1] // 2 + 1)[:s.shape[1]]
    return (s + bias) >> 2


def planes(img):
    """The three component planes the DCT reads, padded as jcprepct.c / jcsample.c pad them: Y [16 mh][16 mw] (edge
    replicated; blocks past ceil(w/8) x ceil(h/8) are never read), Cb / Cr [8 mh][8 mw]: colour rows padded to an even
    count and columns to 16 mw by replication, downsampled, then the last downsampled row replicated."""
    h, w = img.shape[:2]
    mh, mw = -(-h // 16), -(-w // 16)
    y, cb, cr = rgb_ycc(img)
    Y = np.pad(y, ((0, 16 * mh - h), (0, 16 * mw - w)), mode="edge")
    out = [Y]
    for c in (cb, cr):
        c = np.pad(c, ((0, h % 2), (0, 16 * mw - w)), mode="edge")
        d = downsample_h2v2(c)
        out.append(np.pad(d, ((0, 8 * mh - d.shape[0]), (0, 0)), mode="edge"))
    return out


def blocks_of(plane):
    """[H][W] -> [H/8][W/8][8][8]"""
    H, W = plane.shape
    return plane.reshape(H // 8, 8, W // 8, 8).transpose(0, 2, 1, 3)


# ---------------------------------------------------------------------------------------------- DCT and quantisation
C13 = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
           f2053=16819, f2562=20995, f3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    """one pass of jfdctint.c (libjpeg 6b islow) along the last axis; first: the row pass"""
    k = C13
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(d)
    n = 13 - 2 if first else 13 + 2
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        o[..., 0], o[..., 4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    z1 = (t12 + t13) * k["f0541"]
    o[..., 2] = _descale(z1 + t13 * k["f0765"], n)
    o[..., 6] = _descale(z1 - t12 * k["f1847"], n)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * k["f1175"]
    t4, t5, t6, t7 = t4 * k["f0298"], t5 * k["f2053"], t6 * k["f3072"], t7 * k["f1501"]
    z1, z2 = -z1 * k["f0899"], -z2 * k["f2562"]
    z3, z4 = -z3 * k["f1961"] + z5, -z4 * k["f0390"] + z5
    o[..., 7] = _descale(t4 + z1 + z3, n)
    o[..., 5] = _descale(t5 + z2 + z4, n)
    o[..., 3] = _descale(t6 + z2 + z3, n)
    o[..., 1] = _descale(t7 + z1 + z4, n)
    return o


def fdct_islow(blk):
    """samples [..., 8, 8] (0..255) -> jpeg_fdct_islow output (scaled by 8), int64"""
    d = blk.astype(np.int64) - 128
    d = _fdct_1d(d, True)
    d = _fdct_1d(np.swapaxes(d, -1, -2), False)
    return np.swapaxes(d, -1, -2)


def reciprocal(divisor):
    """compute_reciprocal (jcdctmgr.c, 16-bit DCTELEM): (reciprocal, correction, shift r) with
    q = ((|x| + correction) * reciprocal) >> r.  Divisors here are 8 * table >= 8."""
    divisor = np.asarray(divisor, np.int64)
    b = np.floor(np.log2(divisor)).astype(np.int64)
    r = 16 + b
    fq, fr = (np.int64(1) << r) // divisor, (np.int64(1) << r) % divisor
    c = divisor // 2
    pow2 = fr == 0
    fq = np.where(pow2, fq >> 1, np.where(fr <= divisor // 2, fq, fq + 1))
    r = np.where(pow2, r - 1, r)
    c = np.where(~pow2 & (fr <= divisor // 2), c + 1, c)
    return fq, c, r


def quantize(coef, table):
    """coef [..., 64] natural order (fdct output), table [64] natural order -> quantised, natural order"""
    fq, c, r = reciprocal(table * 8)
    a = np.abs(coef)
    q = ((a + c) * fq) >> r
    return np.where(coef < 0, -q, q)


# ---------------------------------------------------------------------------------------------- coefficients
def coefficients(img, quality):
    """Quantised coefficients in zigzag order, in scan order: int64 [n_mcu][6][64] (Y00, Y01, Y10, Y11, Cb, Cr), the
    dummy blocks past ceil(w/8) x ceil(h/8) included (AC 0, DC of the block before it in the MCU)."""
    h, w = img.shape[:2]
    mh, mw = -(-h // 16), -(-w // 16)
    Y, Cb, Cr = planes(img)
    qt = quant_tables(quality)
    out = np.empty((mh, mw, 6, 64), np.int64)
    yb = quantize(fdct_islow(blocks_of(Y)).reshape(2 * mh, 2 * mw, 64), qt[0])[..., ZIGZAG]
    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        out[:, :, i] = yb[dy::2, dx::2]
    out[:, :, 4] = quantize(fdct_islow(blocks_of(Cb)).reshape(mh, mw, 64), qt[1])[..., ZIGZAG]
    out[:, :, 5] = quantize(fdct_islow(blocks_of(Cr)).reshape(mh, mw, 64), qt[1])[..., ZIGZAG]
    hb, wb = -(-h // 8), -(-w // 8)
    if wb % 2:                          # right dummies: block (r, 1) of the last MCU column
        for i in (1, 3):
            out[:, -1, i] = 0
            out[:, -1, i, 0] = out[:, -1, i - 1, 0]
    if hb % 2:                          # bottom dummies: blocks (1, *) of the last MCU row take block (0, 1)'s DC
        out[-1, :, 2:4] = 0
        out[-1, :, 2, 0] = out[-1, :, 1, 0]
        out[-1, :, 3, 0] = out[-1, :, 1, 0]
    return out.reshape(mh * mw, 6, 64)


# ---------------------------------------------------------------------------------------------- entropy coding
def nbits(v):
    """magnitude category: bit length of |v|"""
    a = np.abs(np.asarray(v, np.int64))
    out = np.zeros(a.shape, np.int64)
    while np.any(a):
        out += a > 0
        a = a >> 1
    return out


def _extra(v, s):
    return np.where(v < 0, v + (np.int64(1) << s) - 1, v) & ((np.int64(1) << s) - 1)


COMP_TABLE = np.array([0, 0, 0, 0, 1, 1])


def dc_diffs(coef):
    """coef [n_mcu][6][64] -> DC differences in scan order [n_mcu][6] (predictor per component, starting at 0)"""
    dc = coef[:, :, 0]
    ys = dc[:, :4].reshape(-1)
    dy = np.diff(ys, prepend=0).reshape(-1, 4)
    dcb = np.diff(dc[:, 4], prepend=0)
    dcr = np.diff(dc[:, 5], prepend=0)
    return np.concatenate([dy, dcb[:, None], dcr[:, None]], axis=1)


def tokens(coef):
    """(value, nbits, block) of every Huffman code with its extra bits, in stream order; block = scan-order block index"""
    return block_tokens(coef.reshape(-1, 64), dc_diffs(coef).reshape(-1), np.tile(COMP_TABLE, coef.shape[0]))


def block_tokens(flat, diffs, tab):
    """the same for blocks [n][64] (zigzag) with their DC differences [n] and tables [n] (0 luma, 1 chroma)"""
    flat, diffs, tab = np.asarray(flat, np.int64), np.asarray(diffs, np.int64), np.asarray(tab, np.int64)
    nb = flat.shape[0]
    keys, vals, lens = [], [], []
    # DC
    s = nbits(diffs)
    code = np.where(tab == 0, DC_CODES[0][0][s], DC_CODES[1][0][s])
    cl = np.where(tab == 0, DC_CODES[0][1][s], DC_CODES[1][1][s])
    keys.append(np.arange(nb) * 65 * 4)
    vals.append((code << s) | _extra(diffs, s))
    lens.append(cl + s)
    # AC
    bi, k = np.nonzero(flat[:, 1:])
    k = k + 1
    v = flat[bi, k]
    same = np.r_[False, bi[1:] == bi[:-1]]
    prev = np.where(same, np.r_[0, k[:-1]], 0)        # the previous non-zero position of the block, 0 = the DC
    run = k - prev - 1
    s = nbits(v)
    sym = ((run & 15) << 4) | s
    t = tab[bi]
    acode = np.where(t == 0, AC_CODES[0][0][sym], AC_CODES[1][0][sym])
    alen = np.where(t == 0, AC_CODES[0][1][sym], AC_CODES[1][1][sym])
    assert np.all(alen > 0)
    nz = run >> 4
    for j in range(3):                  # ZRLs: 16 zeros each, only before a non-zero coefficient
        m = nz > j
        keys.append(((bi[m] * 65 + k[m]) * 4 + j))
        vals.append(np.where(t[m] == 0, AC_CODES[0][0][0xF0], AC_CODES[1][0][0xF0]))
        lens.append(np.where(t[m] == 0, AC_CODES[0][1][0xF0], AC_CODES[1][1][0xF0]))
    keys.append((bi * 65 + k) * 4 + 3)
    vals.append((acode << s) | _extra(v, s))
    lens.append(alen + s)
    # EOB unless coefficient 63 is non-zero
    eob = flat[:, 63] == 0
    b = np.flatnonzero(eob)
    keys.append((b * 65 + 64) * 4)
    vals.append(np.where(tab[b] == 0, AC_CODES[0][0][0], AC_CODES[1][0][0]))
    lens.append(np.where(tab[b] == 0, AC_CODES[0][1][0], AC_CODES[1][1][0]))
    keys, vals, lens = (np.concatenate(x) for x in (keys, vals, lens))
    o = np.argsort(keys, kind="stable")
    return vals[o], lens[o], keys[o] // (65 * 4)


def block_bits(coef):
    """bits of each block's codes [n_mcu][6] (DC difference included)"""
    _, lens, blk = tokens(coef)
    return np.bincount(blk, weights=lens, minlength=coef.shape[0] * 6).astype(np.int64).reshape(-1, 6)


def pack(vals, lens):
    """MSB-first bit stream of the tokens, the tail padded with 1-bits to a byte -> bytes (unstuffed)"""
    total = int(lens.sum())
    start = np.cumsum(lens) - lens
    idx = np.repeat(np.arange(len(lens)), lens)
    pos = np.arange(total) - start[idx]
    bits = ((vals[idx] >> (lens[idx] - 1 - pos)) & 1).astype(np.uint8)
    pad = (-total) % 8
    bits = np.concatenate([bits, np.ones(pad, np.uint8)])
    return np.packbits(bits)


def stuff(data):
    """a 0x00 after every 0xFF byte"""
    data = np.asarray(data, np.uint8)
    ff = np.flatnonzero(data == 0xFF)
    return np.insert(data, ff + 1, 0)


def entropy(coef):
    vals, lens, _ = tokens(coef)
    return stuff(pack(vals, lens))


def encode(img, quality=95):
    """cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality])[1] of a BGR uint8 [h][w][3] image"""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    body = entropy(coefficients(img, quality))
    return np.concatenate([np.frombuffer(header(w, h, quality), np.uint8), body, np.array([0xFF, 0xD9], np.uint8)])


def cv2_encode(img, quality=95):
    import cv2
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(img, np.uint8), [cv2.IMWRITE_JPEG_QUALITY, int(quality)])
    assert ok
    return buf.reshape(-1)


# ---------------------------------------------------------------------------------------------- test images
SIZES = [(1, 1), (8, 8), (16, 16), (17, 23), (33, 47), (240, 320), (320, 1280), (480, 2560)]     # (h, w)
QUALITIES = [1, 10, 50, 75, 95, 100]
CONTENTS = ["constant", "gradient", "noise", "dots", "frames"]


def _dots(h, w, rng):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = rng.integers(0, 12, (h, w, 3)).astype(np.float64)
    for _ in range(max(1, h * w // 4000)):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(1.5, 4)
        img += rng.uniform(150, 255) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))[..., None]
    return np.clip(img, 0, 255).astype(np.uint8)


_FRAMES = None


def live_frames():
    """The processed frames of a few reads of the live loop's golden scene through the oracle chain (RefPort
    preprocessing -> find_dot dots), as the stream sees them: np.hstack of the 4 cameras, uint8 [reads][320][1280][3]."""
    global _FRAMES
    if _FRAMES is None:
        from oracle.ref_port import RefPort
        from tests.live_util import CAPTURE, K, golden_scene, load_golden, oracle_read, render_read
        g = load_golden()
        scene = golden_scene(g)
        port = RefPort([K] * 4)
        out = []
        for k in (0, 20, 33):
            res = oracle_read(port, scene, render_read(scene, k, dark=(k == 33)), CAPTURE, None, None, [0.0])
            out.append(np.hstack(list(res["frames"])))
        _FRAMES = np.stack(out)
    return _FRAMES


def make_image(content, h, w, seed=0):
    rng = np.random.default_rng([seed, h, w, CONTENTS.index(content)])
    if content == "constant":
        return np.broadcast_to(rng.integers(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()
    if content == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(xx * 255 // max(1, w - 1)), (yy * 255 // max(1, h - 1)), ((xx + yy) * 7) % 256], -1).astype(np.uint8)
    if content == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if content == "dots":
        return _dots(h, w, rng)
    f = live_frames()[seed % 3]
    reps = (-(-h // f.shape[0]), -(-w // f.shape[1]), 1)
    return np.ascontiguousarray(np.tile(f, reps)[:h, :w])


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_cv2.npz")


def load_golden():
    """tests/golden/jpeg_cv2.npz as a list of (name, image, quality, cv2's bytes); the images are made again from
    their seeds and checked against the recorded SHA-256"""
    import hashlib
    z = np.load(GOLDEN)
    ends = np.cumsum(z["jpeg_len"])
    out = []
    for i, ((h, w), q, content, digest) in enumerate(zip(z["shapes"], z["quality"], z["content"], z["sha256"])):
        img = make_image(str(content), int(h), int(w), seed=5)
        assert hashlib.sha256(img.tobytes()).hexdigest() == str(digest), f"golden image {i} is not what made it"
        out.append((f"{content}_{h}x{w}_q{q}", img, int(q), z["jpeg"][ends[i] - z["jpeg_len"][i]:ends[i]]))
    return out
