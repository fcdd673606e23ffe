"""Baseline JPEG exactly as cv2.imwrite / cv2.imencode writes it (OpenCV 4.13, libjpeg-turbo 3.1), restated from the
algorithm in integer numpy.  The GPU encoder (csrc/jpeg.cu) is pinned to this, and this to cv2.

cv2's settings: 4:2:0 (luma h2v2, chroma h1v1), the integer ("islow") forward DCT, the quantisation and Huffman tables of
ITU-T T.81 Annex K scaled by the quality, no Huffman optimisation, no restart markers, a JFIF 1.01 APP0 with density 1:1
and unit 0.  Stages, each exposed for the tests:

  ycc()            BGR -> YCbCr in 16-bit fixed point (FIX(x) = int(x * 65536 + 0.5))
  planes()         edge replication + h2v2 chroma downsampling -> Y, Cb, Cr sample planes covering whole blocks
  fdct_islow()     8x8 integer forward DCT (13-bit constants, 2 extra bits in the row pass), output scaled by 8
  quantize()       round-half-away division by 8 * table entry
  blocks()         quantised coefficients of every 8x8 block in MCU scan order (Y0 Y1 Y2 Y3 Cb Cr), dummy blocks included,
                   in zigzag order
  entropy()        Huffman-coded scan data with 0xFF byte stuffing and the final byte padded with 1-bits
  headers()        SOI, APP0, DQT 0, DQT 1, SOF0, DHT DC0 / AC0 / DC1 / AC1, SOS
  encode()         the whole file

Edges, as libjpeg's pre-processing does them (and not the "pad everything to 16" shortcut, which differs whenever H is even
and not a multiple of 16): columns are replicated from the last pixel before downsampling (Y to ceil(W/8)*8 columns, the
chroma input to ceil(ceil(W/2)/8)*16); rows only to the 2-row group before downsampling, and the downsampled chroma rows
are then replicated to the MCU height.  Luma blocks past the image (right of ceil(W/8) or below ceil(H/8) block columns /
rows) are dummies: all zero, with the DC of the block to their left (right edge) or of the last block of the row above in
the same MCU (bottom edge)."""
from __future__ import annotations

import numpy as np

# ---------------------------------------------------------------------------------------------------------- tables
# ITU-T T.81 Annex K, natural (row-major) order
STD_LUMA_QT = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_QT = np.full(64, 99, np.int64)
STD_CHROMA_QT[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# Huffman tables (BITS: codes of each length 1..16, HUFFVAL), Annex K.3
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16,
    0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6,
    0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8,
    0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34,
    0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4,
    0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6,
    0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])


def _zigzag():
    """ZIGZAG[k] = natural index of the k-th coefficient in zigzag order (walk the anti-diagonals, alternating direction)."""
    order = []
    for s in range(15):
        cells = [(r, s - r) for r in range(8) if 0 <= s - r < 8]
        order += cells if s % 2 else cells[::-1]
    return np.array([r * 8 + c for r, c in order], np.int64)


ZIGZAG = _zigzag()


def huff_codes(spec):
    """(BITS, HUFFVAL) -> {symbol: (code, length)}, canonical code assignment (T.81 Annex C)."""
    bits, vals = spec
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def clamp_quality(quality: int) -> int:
    """cv2: IMWRITE_JPEG_QUALITY is clamped to [0, 100]; libjpeg then treats 0 as 1."""
    return min(max(int(quality), 1), 100)


def quant_tables(quality: int):
    """-> (luma, chroma) int64 [64] in natural order, libjpeg's quality scaling clamped to baseline (1..255)."""
    q = clamp_quality(quality)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    f = lambda t: np.clip((t * scale + 50) // 100, 1, 255)   # noqa: E731
    return f(STD_LUMA_QT), f(STD_CHROMA_QT)


# ---------------------------------------------------------------------------------------------------------- transform
def _fix(x):
    return int(x * 65536 + 0.5)


def ycc(bgr):
    """uint8 [h,w,3] BGR -> (Y, Cb, Cr) int64 [h,w]."""
    b, g, r = (bgr[..., c].astype(np.int64) for c in range(3))
    half = 1 << 15
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + (128 << 16) + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + (128 << 16) + half - 1) >> 16
    return y, cb, cr


def geometry(w: int, h: int) -> dict:
    """Block counts: luma blocks per row / column, MCUs per row / column (= chroma blocks)."""
    return {"bw": -(-w // 8), "bh": -(-h // 8), "mw": -(-w // 16), "mh": -(-h // 16)}


def _rep(a, rows, cols):
    """Replicate the last row / column of a up to rows x cols."""
    return np.pad(a, ((0, rows - a.shape[0]), (0, cols - a.shape[1])), mode="edge")


def downsample_h2v2(c):
    """[2r, 2c] -> [r, c]: (a + b + c + d + bias) >> 2, bias 1, 2, 1, 2, ... along the output row."""
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return (s + bias[None, :]) >> 2


def planes(bgr, pad16_rows: bool = False, cols_after: bool = False):
    """uint8 [h,w,3] BGR -> (Y [mh*16, mw*16], Cb, Cr [mh*8, mw*8]) int64 sample planes.  Y is replicated to whole MCUs
    here for convenience; blocks outside ceil(w/8) x ceil(h/8) are replaced by dummies in blocks().
    pad16_rows / cols_after: the two wrong edge treatments (input rows padded to 16 before downsampling; columns
    replicated after downsampling instead of before), kept for the tests that show they change the bytes."""
    h, w = bgr.shape[:2]
    g = geometry(w, h)
    y, cb, cr = ycc(bgr)
    Y = _rep(y, g["mh"] * 16, g["mw"] * 16)
    rows_in = g["mh"] * 16 if pad16_rows else -(-h // 2) * 2
    cols_in = -(-w // 2) * 2 if cols_after else g["mw"] * 16
    chroma = []
    for c in (cb, cr):
        d = downsample_h2v2(_rep(c, rows_in, cols_in))
        chroma.append(_rep(d, g["mh"] * 8, g["mw"] * 8))
    return Y, chroma[0], chroma[1]


# jfdctint constants, 13 fractional bits
C_0_298631336, C_0_390180644, C_0_541196100, C_0_765366865 = 2446, 3196, 4433, 6270
C_0_899976223, C_1_175875602, C_1_501321110, C_1_847759065 = 7373, 9633, 12299, 15137
C_1_961570560, C_2_053119869, C_2_562915447, C_3_072711026 = 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, last):
    """One 8-point pass along the last axis of d [..., 8]; last: the column pass (different scaling)."""
    tmp0, tmp7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    tmp1, tmp6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    tmp2, tmp5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    tmp3, tmp4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    out = np.empty_like(d)
    sh = CONST_BITS + PASS1_BITS if last else CONST_BITS - PASS1_BITS
    if last:
        out[..., 0] = _descale(tmp10 + tmp11, PASS1_BITS)
        out[..., 4] = _descale(tmp10 - tmp11, PASS1_BITS)
    else:
        out[..., 0] = (tmp10 + tmp11) << PASS1_BITS
        out[..., 4] = (tmp10 - tmp11) << PASS1_BITS
    z1 = (tmp12 + tmp13) * C_0_541196100
    out[..., 2] = _descale(z1 + tmp13 * C_0_765366865, sh)
    out[..., 6] = _descale(z1 - tmp12 * C_1_847759065, sh)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * C_1_175875602
    tmp4, tmp5 = tmp4 * C_0_298631336, tmp5 * C_2_053119869
    tmp6, tmp7 = tmp6 * C_3_072711026, tmp7 * C_1_501321110
    z1, z2 = -z1 * C_0_899976223, -z2 * C_2_562915447
    z3, z4 = -z3 * C_1_961570560 + z5, -z4 * C_0_390180644 + z5
    out[..., 7] = _descale(tmp4 + z1 + z3, sh)
    out[..., 5] = _descale(tmp5 + z2 + z4, sh)
    out[..., 3] = _descale(tmp6 + z2 + z3, sh)
    out[..., 1] = _descale(tmp7 + z1 + z4, sh)
    return out


def fdct_islow(samples):
    """[..., 8, 8] samples 0..255 -> [..., 8, 8] DCT coefficients scaled by 8 (rows first, then columns)."""
    d = samples.astype(np.int64) - 128
    d = _fdct_1d(d, last=False)
    return np.swapaxes(_fdct_1d(np.swapaxes(d, -1, -2), last=True), -1, -2)


def quantize(coef, table):
    """[..., 64] natural order / [64] table -> round(|x| / (8 q)) half away from zero, sign restored."""
    d = (table * 8).astype(np.int64)
    a = np.abs(coef)
    return np.sign(coef) * ((a + d // 2) // d)


def _tiles(p):
    """[R*8, C*8] -> [R, C, 8, 8]"""
    R, C = p.shape[0] // 8, p.shape[1] // 8
    return p.reshape(R, 8, C, 8).transpose(0, 2, 1, 3)


def blocks(bgr, quality: int = 95, dummy_dc: bool = True, **plane_kw):
    """uint8 [h,w,3] BGR -> int64 [mh*mw*6, 64]: the quantised coefficients of every block in scan order (MCU by MCU,
    Y0 Y1 Y2 Y3 Cb Cr), zigzag order, dummy blocks included.  dummy_dc=False: dummies keep DC 0 (a wrong variant)."""
    h, w = bgr.shape[:2]
    g = geometry(w, h)
    ql, qc = quant_tables(quality)
    Y, Cb, Cr = planes(bgr, **plane_kw)
    qy = quantize(fdct_islow(_tiles(Y)).reshape(2 * g["mh"], 2 * g["mw"], 64), ql)
    qb = quantize(fdct_islow(_tiles(Cb)).reshape(g["mh"], g["mw"], 64), qc)
    qr = quantize(fdct_islow(_tiles(Cr)).reshape(g["mh"], g["mw"], 64), qc)
    out = np.zeros((g["mh"], g["mw"], 6, 64), np.int64)
    for j in range(4):
        out[:, :, j] = qy[(j >> 1)::2, (j & 1)::2]
    out[:, :, 4], out[:, :, 5] = qb, qr
    bx = 2 * np.arange(g["mw"])[None, :, None] + np.array([0, 1, 0, 1])[None, None, :]
    by = 2 * np.arange(g["mh"])[:, None, None] + np.array([0, 0, 1, 1])[None, None, :]
    right, bottom = bx >= g["bw"], by >= g["bh"]            # [mh, mw, 4]
    dummy = right | bottom
    ydc = out[:, :, :4, 0].copy()
    out[:, :, :4][dummy] = 0
    if dummy_dc:
        # right edge: the DC of the block to the left; bottom dummy row: the DC of the last block of the row above (Y1)
        y1 = np.where(right[:, :, 1], ydc[:, :, 0], ydc[:, :, 1])
        y3_right = np.where(right[:, :, 3], ydc[:, :, 2], ydc[:, :, 3])
        out[:, :, 1, 0] = y1
        out[:, :, 2, 0] = np.where(bottom[:, :, 2], y1, ydc[:, :, 2])
        out[:, :, 3, 0] = np.where(bottom[:, :, 3], y1, y3_right)
    return out.reshape(-1, 64)[:, ZIGZAG]


# ---------------------------------------------------------------------------------------------------------- bitstream
_CODES = {name: huff_codes(spec) for name, spec in
          (("dc0", DC_LUMA), ("ac0", AC_LUMA), ("dc1", DC_CHROMA), ("ac1", AC_CHROMA))}


def _nbits(v):
    return int(abs(int(v))).bit_length()


def _vbits(v, n):
    return (int(v) if v >= 0 else int(v) - 1) & ((1 << n) - 1)


def tokens(blk, stats=None):
    """[nblk, 64] zigzag coefficients in scan order -> (values, lengths) of every Huffman code / amplitude field."""
    vals, lens = [], []
    pred = [0, 0, 0]
    for i, b in enumerate(blk):
        j = i % 6
        comp = 0 if j < 4 else j - 3
        dc, ac = (_CODES["dc0"], _CODES["ac0"]) if comp == 0 else (_CODES["dc1"], _CODES["ac1"])
        diff = int(b[0]) - pred[comp]
        pred[comp] = int(b[0])
        n = _nbits(diff)
        c, l = dc[n]
        vals.append(c); lens.append(l)
        if n:
            vals.append(_vbits(diff, n)); lens.append(n)
        if stats is not None:
            stats["max_dc_cat"] = max(stats.get("max_dc_cat", 0), n)
        last = 0
        for k in np.flatnonzero(b[1:]) + 1:
            run = k - last - 1
            while run > 15:
                c, l = ac[0xF0]
                vals.append(c); lens.append(l)
                run -= 16
                if stats is not None:
                    stats["zrl"] = stats.get("zrl", 0) + 1
            n = _nbits(b[k])
            c, l = ac[(run << 4) | n]
            vals.append(c); lens.append(l)
            vals.append(_vbits(b[k], n)); lens.append(n)
            last = k
        if last < 63:
            c, l = ac[0x00]
            vals.append(c); lens.append(l)
    return np.array(vals, np.uint64), np.array(lens, np.int64)


def pack_bits(vals, lens):
    """MSB-first concatenation of the fields, the last byte padded with 1-bits -> uint8 array (not yet stuffed)."""
    total = int(lens.sum())
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    idx = np.repeat(np.arange(len(lens)), lens)
    pos = np.arange(total) - np.repeat(starts, lens)
    bits = ((vals[idx] >> (lens[idx] - 1 - pos).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
    bits = np.concatenate([bits, np.ones((-total) % 8, np.uint8)])
    return np.packbits(bits)


def stuff(data):
    """0xFF -> 0xFF 0x00."""
    ff = np.flatnonzero(data == 0xFF)
    return np.insert(data, ff + 1, 0)


def entropy(blk, stuffing: bool = True, stats=None):
    raw = pack_bits(*tokens(blk, stats))
    if stats is not None:
        stats["ff"] = stats.get("ff", 0) + int((raw == 0xFF).sum())
    return (stuff(raw) if stuffing else raw).tobytes()


# ---------------------------------------------------------------------------------------------------------- markers
def _marker(code, payload: bytes) -> bytes:
    return bytes([0xFF, code]) + (len(payload) + 2).to_bytes(2, "big") + payload


def headers(w: int, h: int, quality: int = 95) -> bytes:
    ql, qc = quant_tables(quality)
    out = b"\xff\xd8"
    out += _marker(0xE0, b"JFIF\x00" + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
    for t, q in enumerate((ql, qc)):
        out += _marker(0xDB, bytes([t]) + bytes(q[ZIGZAG].astype(np.uint8).tolist()))
    out += _marker(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls, t, spec in ((0, 0, DC_LUMA), (1, 0, AC_LUMA), (0, 1, DC_CHROMA), (1, 1, AC_CHROMA)):
        out += _marker(0xC4, bytes([(cls << 4) | t]) + bytes(spec[0]) + bytes(spec[1]))
    out += _marker(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    return out


HEADER_BYTES = 623      # len(headers(...)): the same for every size and quality


def encode(bgr, quality: int = 95, stats=None, **variant) -> bytes:
    """uint8 [h,w,3] BGR -> the bytes cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, quality]) returns.
    variant (tests only): pad16_rows / cols_after (planes), dummy_dc (blocks), stuffing (entropy)."""
    bgr = np.ascontiguousarray(bgr, np.uint8)
    if bgr.ndim == 2:
        raise ValueError("greyscale is not supported")
    h, w = bgr.shape[:2]
    stuffing = variant.pop("stuffing", True)
    dummy_dc = variant.pop("dummy_dc", True)
    blk = blocks(bgr, quality, dummy_dc=dummy_dc, **variant)
    if stats is not None:
        g = geometry(w, h)
        stats["right_dummies"] = stats.get("right_dummies", 0) + int(g["bw"] % 2) * g["mh"]
        stats["bottom_dummies"] = stats.get("bottom_dummies", 0) + int(g["bh"] % 2) * g["mw"]
        stats["even_h_chroma_pad"] = stats.get("even_h_chroma_pad", 0) + int(h % 2 == 0 and h % 16 != 0)
    return headers(w, h, quality) + entropy(blk, stuffing, stats) + b"\xff\xd9"


def bound(w: int, h: int) -> int:
    """Worst-case size of one encoded w x h image: every block at its longest code (DC 22 bits, 63 AC fields of 26 bits),
    every byte stuffed, plus the headers, the padding byte and EOI.  Equals cc_jpeg_bound."""
    g = geometry(w, h)
    data = -(-(g["mw"] * g["mh"] * 6 * MAX_BLOCK_BITS) // 8) + 1
    return HEADER_BYTES + 2 * data + 2


MAX_BLOCK_BITS = 22 + 63 * 26
