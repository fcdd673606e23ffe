"""Baseline / extended-sequential Huffman JPEG decoded exactly as cv2.imdecode(buf, IMREAD_COLOR) decodes it (OpenCV 4.13
with libjpeg-turbo 3.1), restated from the algorithm in integer numpy.  The GPU decoder (csrc/jpeg_decode.cu) is pinned to
this, and this to cv2.

Stages, each exposed for the tests, with the libjpeg-turbo module each one restates:

  parse()           markers (jdmarker.c: get_sof / get_dqt / get_dht / get_dri / get_sos, examine_app0 / examine_app14, the
                    colour-space guess of jdapimin.c) -> a per-image table, or a status: UNSUPPORTED for anything the device
                    decoder leaves to the host, CORRUPT for a malformed header.  Never raises, never reads past the buffer.
  huff_table()      canonical code assignment and its validity check (jdhuff.c jpeg_make_d_derived_tbl) -> a 16-bit lookup
  intervals()       the scan split at its RSTn markers with the FF 00 stuffing removed (what jdhuff.c's bit reader sees)
  decode_coeffs()   sequential Huffman decode (jdhuff.c decode_mcu): DC differences, AC run/size symbols, ZRL, EOB; the
                    coefficients of a position past 63 land on 63 (jpeg_natural_order's 16 extra entries); DC prediction per
                    component, reset at every restart
  decode_coeffs_selfsync()  the same coefficients by self-synchronising parallel decoding (Weissenberger & Schmidt, ICPP
                    2018 / HiPC 2021): every restart interval is cut into subsequences of a fixed number of bits, each decoded
                    from a guessed state until all agree, then written from the synchronised states
  idct_islow()      dequantisation and the integer inverse DCT (jidctint.c), range limit of jdmaster.c
  upsample()        fancy upsampling (jdsample.c h2v1 / h1v2 / h2v2_fancy_upsample, with the row context of jdmainct.c:
                    rows above the image repeat its first row, rows below it its last), box replication (h2v1 / h2v2_upsample)
                    where the downsampled width is 2 or less
  ycc_to_bgr()      the table-driven YCbCr -> BGR conversion (jdcolor.c build_ycc_rgb_table / ycc_rgb_convert)
  decode()          the whole file -> (status, BGR uint8 [h, w, 3] or None)

libjpeg-turbo's SIMD inverse DCT (the one cv2 runs) agrees with jidctint.c while the dequantised coefficients and the
first-pass outputs fit comfortably in 16 bits and the final values lie in [-512, 511]; outside that range the two differ,
and such an image is reported UNSUPPORTED (decoded by cv2 on the host) rather than guessed."""
from __future__ import annotations

import numpy as np

OK, UNSUPPORTED, CORRUPT = 0, 1, 2

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46,
                   53, 60, 61, 54, 47, 55, 62, 63], np.int64)
# Limits inside which every libjpeg-turbo inverse DCT gives the same samples (see the module docstring)
IDCT_IN_LIMIT = 16383
IDCT_OUT_LO, IDCT_OUT_HI = -512, 511


class _Bad(Exception):
    def __init__(self, status):
        self.status = status


def _be16(b, i):
    return (b[i] << 8) | b[i + 1]


# ---------------------------------------------------------------------------------------------------------- markers
def huff_table(counts, vals, dc: bool):
    """(BITS[16], HUFFVAL) -> (length [65536], symbol [65536]) indexed by the next 16 bits; length 0 = no code.
    Raises _Bad(CORRUPT) where jpeg_make_d_derived_tbl raises JERR_BAD_HUFF_TABLE."""
    length = np.zeros(65536, np.int64)
    symbol = np.zeros(65536, np.int64)
    code, k = 0, 0
    for L in range(1, 17):
        for _ in range(counts[L - 1]):
            if code + 1 >= (1 << L):                    # codes must fit in L bits and never be all ones
                raise _Bad(CORRUPT)
            lo = code << (16 - L)
            length[lo:lo + (1 << (16 - L))] = L
            symbol[lo:lo + (1 << (16 - L))] = vals[k]
            code += 1
            k += 1
        code <<= 1
    if dc and any(v > 15 for v in vals):
        raise _Bad(CORRUPT)
    return length, symbol


def _exif_orientation(seg: bytes):
    """Orientation tag of an APP1 Exif payload (after "Exif\\0\\0"): 1..8, or None when absent; raises on a layout that
    cannot be read (the image then goes to cv2)."""
    t = seg[6:]
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        raise _Bad(UNSUPPORTED)
    big = t[:2] == b"MM"
    rd = lambda o, n: int.from_bytes(t[o:o + n], "big" if big else "little")   # noqa: E731
    ifd = rd(4, 4)
    if ifd + 2 > len(t):
        raise _Bad(UNSUPPORTED)
    for i in range(rd(ifd, 2)):
        e = ifd + 2 + 12 * i
        if e + 12 > len(t):
            raise _Bad(UNSUPPORTED)
        if rd(e, 2) == 0x0112:
            return rd(e + 8, 2)
    return None


_SOF_OTHER = {0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF}


def parse(data: bytes):
    """-> (status, info).  info (status OK): w, h, ncomp, comps [(id, H, V, tq)], qt {id: int64 [64] natural order},
    dc / ac {id: (length, symbol)}, td / ta per component, ri (restart interval in MCUs), scan (offset, length) of the
    entropy-coded data between SOS and the marker that ends it."""
    try:
        return OK, _parse(bytes(data))
    except _Bad as e:
        return e.status, None


def _parse(b: bytes):
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise _Bad(CORRUPT)
    pos = 2
    qt, dct, act = {}, {}, {}
    sof = None
    ri = 0
    jfif, adobe = False, None
    while True:
        if pos + 2 > n or b[pos] != 0xFF:
            raise _Bad(CORRUPT)
        while pos < n and b[pos] == 0xFF:
            pos += 1
        if pos + 3 > n:
            raise _Bad(CORRUPT)
        code = b[pos]
        pos += 1
        if code in (0xD8, 0xD9, 0x01) or 0xD0 <= code <= 0xD7:
            raise _Bad(CORRUPT)                         # no standalone marker belongs before the scan
        if code < 0xC0 or code in (0xC8, 0xDE, 0xDF) or 0xF0 <= code <= 0xFD:
            raise _Bad(CORRUPT)                         # a marker libjpeg's read_markers does not know: cv2 fails
        ln = _be16(b, pos)
        if ln < 2 or pos + ln > n:
            raise _Bad(CORRUPT)
        seg = b[pos + 2:pos + ln]
        pos += ln
        if code in (0xC0, 0xC1):
            if sof is not None or len(seg) < 6:
                raise _Bad(CORRUPT)
            P, h, w, nf = seg[0], _be16(seg, 1), _be16(seg, 3), seg[5]
            if len(seg) != 6 + 3 * nf or nf == 0 or h == 0 or w == 0:
                raise _Bad(CORRUPT)
            if P != 8:
                raise _Bad(UNSUPPORTED)
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
            if any(not (1 <= H <= 4 and 1 <= V <= 4) or tq > 3 for _, H, V, tq in comps):
                raise _Bad(CORRUPT)
            if len({c[0] for c in comps}) != nf:
                raise _Bad(UNSUPPORTED)
            if nf == 3:
                if comps[0][1] > 2 or comps[0][2] > 2 or any((H, V) != (1, 1) for _, H, V, _ in comps[1:]):
                    raise _Bad(UNSUPPORTED)
            elif nf != 1:
                raise _Bad(UNSUPPORTED)
            sof = {"w": w, "h": h, "ncomp": nf, "comps": comps}
        elif code in _SOF_OTHER or code == 0xCC:
            raise _Bad(UNSUPPORTED)                     # progressive, lossless, hierarchical, arithmetic
        elif code == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                nb = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + nb > len(seg):
                    raise _Bad(CORRUPT)
                v = np.frombuffer(seg[i + 1:i + 1 + nb], ">u2" if pq else np.uint8).astype(np.int64)
                if v.max() > 32767:
                    raise _Bad(UNSUPPORTED)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = v
                qt[tq] = t
                i += 1 + nb
        elif code == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise _Bad(CORRUPT)
                tc, th = seg[i] >> 4, seg[i] & 15
                counts = list(seg[i + 1:i + 17])
                tot = sum(counts)
                if tc > 1 or th > 3 or tot > 256 or i + 17 + tot > len(seg):
                    raise _Bad(CORRUPT)
                vals = list(seg[i + 17:i + 17 + tot])
                (act if tc else dct)[th] = (counts, vals)
                i += 17 + tot
        elif code == 0xDD:
            if len(seg) != 2:
                raise _Bad(CORRUPT)
            ri = _be16(seg, 0)
        elif code == 0xE0:
            jfif = jfif or (len(seg) >= 14 and seg[:5] == b"JFIF\x00")
        elif code == 0xE1:
            if seg[:6] == b"Exif\x00\x00":
                o = _exif_orientation(seg)
                if o is not None and o != 1:
                    raise _Bad(UNSUPPORTED)
        elif code == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif code == 0xDA:
            if sof is None or len(seg) < 1:
                raise _Bad(CORRUPT)
            ns = seg[0]
            if len(seg) != 4 + 2 * ns or ns == 0:
                raise _Bad(CORRUPT)
            ids = [c[0] for c in sof["comps"]]
            sc = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
            if any(c not in ids for c, _, _ in sc) or any(td > 3 or ta > 3 for _, td, ta in sc):
                raise _Bad(CORRUPT)
            Ss, Se, A = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if [c for c, _, _ in sc] != ids or (Ss, Se, A) != (0, 63, 0):
                raise _Bad(UNSUPPORTED)                 # more than one scan, or not a full sequential scan
            break
        # APPn, COM and the rest: skipped
    if sof["ncomp"] == 3 and not jfif and ((adobe is not None and adobe == 0) or (adobe is None and ids == [82, 71, 66])):
        raise _Bad(UNSUPPORTED)                         # stored as RGB, not YCbCr
    # the scan ends at the first marker that is not RSTn (FF FF is fill before a marker)
    start, end = pos, n
    i = pos
    while True:
        i = b.find(b"\xff", i)
        if i < 0 or i + 1 >= n:
            break
        m = b[i + 1]
        if m == 0x00 or 0xD0 <= m <= 0xD7 or m == 0xFF:
            i += 1 if m == 0xFF else 2
            continue
        end = i
        if m != 0xD9:
            raise _Bad(UNSUPPORTED)                     # another scan (or DNL) follows
        break
    info = dict(sof)
    tables = {}
    try:
        for cid, td, ta in sc:
            tables[("dc", td)] = huff_table(*dct[td], dc=True)
            tables[("ac", ta)] = huff_table(*act[ta], dc=False)
    except KeyError:
        raise _Bad(UNSUPPORTED) from None               # libjpeg would substitute its default tables
    for _, _, _, tq in sof["comps"]:
        if tq not in qt:
            raise _Bad(CORRUPT)
    info.update(qt={c[3]: qt[c[3]] for c in sof["comps"]}, huff=tables, td=[s[1] for s in sc], ta=[s[2] for s in sc], ri=ri,
                scan=(start, end - start))
    info.update(geometry(info))
    return info


def geometry(info) -> dict:
    """MCU layout: mcux, mcuy, the component of each block of an MCU with its (h, v) offset, block planes per component
    (bw, bh in blocks) and downsampled sizes (dw, dh in samples)."""
    w, h, comps = info["w"], info["h"], info["comps"]
    if info["ncomp"] == 1:
        bw, bh = -(-w // 8), -(-h // 8)
        return {"mcux": bw, "mcuy": bh, "blocks": [(0, 0, 0)], "planes": [(bw, bh, w, h)], "hmax": 1, "vmax": 1}
    Hm, Vm = comps[0][1], comps[0][2]
    mcux, mcuy = -(-w // (8 * Hm)), -(-h // (8 * Vm))
    blocks, planes = [], []
    for ci, (_, H, V, _) in enumerate(comps):
        blocks += [(ci, bx, by) for by in range(V) for bx in range(H)]
        planes.append((mcux * H, mcuy * V, -(-w * H // Hm), -(-h * V // Vm)))
    return {"mcux": mcux, "mcuy": mcuy, "blocks": blocks, "planes": planes, "hmax": Hm, "vmax": Vm}


# ---------------------------------------------------------------------------------------------------------- entropy
def intervals(data: bytes, info):
    """The scan's entropy-coded bytes with the stuffing removed, split at its RSTn markers -> list of bytes.  Raises
    _Bad(CORRUPT) unless the markers run D0, D1, ... and there is one interval per restart interval."""
    off, ln = info["scan"]
    s = data[off:off + ln]
    out, cur, i, want = [], bytearray(), 0, 0
    while i < len(s):
        c = s[i]
        if c != 0xFF:
            cur.append(c)
            i += 1
            continue
        nx = s[i + 1] if i + 1 < len(s) else None
        if nx == 0x00:
            cur.append(0xFF)
            i += 2
        elif nx == 0xFF or nx is None:
            i += 1                                      # fill byte
        else:                                           # RSTn
            if nx != 0xD0 + want:
                raise _Bad(CORRUPT)
            want = (want + 1) & 7
            out.append(bytes(cur))
            cur = bytearray()
            i += 2
    out.append(bytes(cur))
    nmcu = info["mcux"] * info["mcuy"]
    nint = -(-nmcu // info["ri"]) if info["ri"] else 1
    if len(out) != nint:
        raise _Bad(CORRUPT)
    return out


def _windows(buf: bytes):
    """16-bit big-endian windows at every bit position of buf (zeros past its end) -> (int64 [nbits + 1], nbits)."""
    bits = np.unpackbits(np.frombuffer(buf, np.uint8)).astype(np.int64)
    nb = len(bits)
    bits = np.concatenate([bits, np.zeros(16, np.int64)])
    win = np.zeros(nb + 1, np.int64)
    for i in range(16):
        win += bits[i:i + nb + 1] << (15 - i)
    return win, nb


def _extend(v, s):
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


class _Decoder:
    """Symbol-by-symbol decoding of one interval.  A state is (pos, blk, zz): the bit position, the block of the MCU and
    the next zigzag index (0 = the DC difference comes next)."""

    def __init__(self, info, buf):
        self.win, self.nbits = _windows(buf)
        self.bpm = len(info["blocks"])
        self.dc = [info["huff"][("dc", info["td"][c])] for c, _, _ in info["blocks"]]
        self.ac = [info["huff"][("ac", info["ta"][c])] for c, _, _ in info["blocks"]]

    def run(self, state, end, limit=None, out=None):
        """Decode from state while the position is below `end` (or until `limit` blocks are complete) -> (state, blocks
        completed, blocks completed before the first invalid code or None).  A symbol that would run past the interval
        stops the decode at the interval's end; after an invalid code decoding goes on one bit later from block 0, zigzag 0
        (a guessed state meets invalid codes; on the true chain one is corruption).  out: callback(block, zz, value)."""
        pos, blk, zz = state
        done, err = 0, None
        win, nbits = self.win, self.nbits
        while pos < end and (limit is None or done < limit):
            w = int(win[pos]) if pos <= nbits else 0
            tab = self.dc[blk] if zz == 0 else self.ac[blk]
            L = int(tab[0][w])
            if L == 0:
                err = done if err is None else err
                pos, blk, zz = pos + 1, 0, 0
                continue
            sym = int(tab[1][w])
            s = sym if zz == 0 else sym & 15
            r = 0 if zz == 0 else sym >> 4
            if pos + L + s > nbits:
                return (nbits, blk, zz), done, err
            v = 0
            if s:
                v = _extend((int(win[pos + L]) >> (16 - s)) & ((1 << s) - 1), s)
            pos += L + s
            if zz == 0:
                if out is not None:
                    out(done, 0, v)
                zz = 1
            elif s:
                zz += r
                if out is not None:
                    out(done, min(zz, 63), v)
                zz += 1
            elif r == 15:
                zz += 16
            else:
                zz = 64
            if zz >= 64:
                zz = 0
                blk = blk + 1 if blk + 1 < self.bpm else 0
                done += 1
        return (pos, blk, zz), done, err


def _expected_blocks(info, j, nint):
    nmcu = info["mcux"] * info["mcuy"]
    ri = info["ri"] or nmcu
    return (min(ri, nmcu - j * ri) if nint > 1 else nmcu) * len(info["blocks"])


def _dc_values(info, coef, starts):
    """DC differences -> DC values: running sums per component, reset at each interval start (int16 as JCOEF stores)."""
    comp = np.array([c for c, _, _ in info["blocks"]])
    bpm = len(comp)
    bcomp = comp[np.arange(len(coef)) % bpm]
    seg = np.zeros(len(coef), np.int64)
    seg[np.asarray(starts[1:], np.int64)] = 1
    seg = np.cumsum(seg)
    dc = coef[:, 0].astype(np.int64)
    out = np.zeros(len(coef), np.int64)
    for c in range(comp.max() + 1):
        for sgi in np.unique(seg):
            m = np.flatnonzero((bcomp == c) & (seg == sgi))
            out[m] = np.cumsum(dc[m])
    coef[:, 0] = out.astype(np.int16)
    return coef


def decode_coeffs(data: bytes, info):
    """Sequential decode -> int16 [n_blocks, 64] zigzag coefficients in scan order (the dequantisation input).
    Raises _Bad(CORRUPT) on an invalid code or a scan that ends early."""
    ivs = intervals(data, info)
    total = info["mcux"] * info["mcuy"] * len(info["blocks"])
    coef = np.zeros((total, 64), np.int64)
    starts, base = [], 0
    for j, buf in enumerate(ivs):
        want = _expected_blocks(info, j, len(ivs))
        d = _Decoder(info, buf)

        def put(b, zz, v, base=base):
            coef[base + b, zz] = v
        _, done, err = d.run((0, 0, 0), d.nbits + 1, limit=want, out=put)
        if done < want or err is not None:
            raise _Bad(CORRUPT)
        starts.append(base)
        base += want
    return _dc_values(info, coef, starts)


def decode_coeffs_selfsync(data: bytes, info, sub_bits: int = 256, stats=None):
    """decode_coeffs by self-synchronisation.  Each interval of n bits is cut into ceil(n / sub_bits) subsequences.
    Subsequence q starts from a guessed state (its first bit, block 0, zigzag 0; the exact state for q = 0) and decodes every
    symbol that starts before its end; its end state is the start state of q + 1.  Rounds then replace each start state by
    the previous subsequence's end state and decode again where it changed, until nothing changes (after round r the first
    r + 1 subsequences are exact, and in practice a guess falls into step within a few codes).  A prefix sum of the blocks
    completed per subsequence gives each subsequence's first block; a second pass writes the coefficients from the
    synchronised states, and the DC differences are summed per component and interval."""
    ivs = intervals(data, info)
    total = info["mcux"] * info["mcuy"] * len(info["blocks"])
    coef = np.zeros((total, 64), np.int64)
    starts, base, rounds = [], 0, 0
    for j, buf in enumerate(ivs):
        want = _expected_blocks(info, j, len(ivs))
        d = _Decoder(info, buf)
        nsub = max(1, -(-d.nbits // sub_bits))
        ends_at = [min((q + 1) * sub_bits, d.nbits) for q in range(nsub)]
        ends_at[-1] = d.nbits + 1                      # the last subsequence runs to the interval's end
        start = [(0, 0, 0)] + [(q * sub_bits, 0, 0) for q in range(1, nsub)]
        res = [d.run(start[q], ends_at[q]) for q in range(nsub)]
        r = 0
        while True:
            new = [start[0]] + [res[q - 1][0] for q in range(1, nsub)]
            changed = [q for q in range(nsub) if new[q] != start[q]]
            if not changed:
                break
            r += 1
            start = new
            for q in changed:
                res[q] = d.run(start[q], ends_at[q])
        rounds = max(rounds, r)
        counts = np.array([c for _, c, _ in res], np.int64)
        first = np.concatenate([[0], np.cumsum(counts)[:-1]])
        if counts.sum() < want or any(e is not None and f + e < want for (_, _, e), f in zip(res, first)):
            raise _Bad(CORRUPT)             # too few blocks, or an invalid code on the synchronised chain before the last
        for q in range(nsub):
            if first[q] >= want:
                break

            def put(b, zz, v, off=base + int(first[q])):
                if off + b < base + want:
                    coef[off + b, zz] = v
            d.run(start[q], ends_at[q], out=put)
        starts.append(base)
        base += want
    if stats is not None:
        stats["rounds"] = max(stats.get("rounds", 0), rounds)
    return _dc_values(info, coef, starts)


# ---------------------------------------------------------------------------------------------------------- pixels
C_0_298631336, C_0_390180644, C_0_541196100, C_0_765366865 = 2446, 3196, 4433, 6270
C_0_899976223, C_1_175875602, C_1_501321110, C_1_847759065 = 7373, 9633, 12299, 15137
C_1_961570560, C_2_053119869, C_2_562915447, C_3_072711026 = 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2


def _idct_1d(d, shift):
    """One 8-point pass of jidctint.c along the last axis, descaled by `shift`."""
    z2, z3 = d[..., 2], d[..., 6]
    z1 = (z2 + z3) * C_0_541196100
    tmp2 = z1 - z3 * C_1_847759065
    tmp3 = z1 + z2 * C_0_765366865
    tmp0 = (d[..., 0] + d[..., 4]) << CONST_BITS
    tmp1 = (d[..., 0] - d[..., 4]) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d[..., 7], d[..., 5], d[..., 3], d[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * C_1_175875602
    t0, t1, t2, t3 = t0 * C_0_298631336, t1 * C_2_053119869, t2 * C_3_072711026, t3 * C_1_501321110
    z1, z2 = -z1 * C_0_899976223, -z2 * C_2_562915447
    z3, z4 = -z3 * C_1_961570560 + z5, -z4 * C_0_390180644 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    out = np.empty_like(d)
    out[..., 0], out[..., 7] = (tmp10 + t3 + r) >> shift, (tmp10 - t3 + r) >> shift
    out[..., 1], out[..., 6] = (tmp11 + t2 + r) >> shift, (tmp11 - t2 + r) >> shift
    out[..., 2], out[..., 5] = (tmp12 + t1 + r) >> shift, (tmp12 - t1 + r) >> shift
    out[..., 3], out[..., 4] = (tmp13 + t0 + r) >> shift, (tmp13 - t0 + r) >> shift
    return out


def range_limit(x):
    """jdmaster.c's post-IDCT table indexed by x & 1023: x + 128 clamped to 0..255 for x in [-512, 511], wrapping outside."""
    j = x & 1023
    return np.where(j < 128, j + 128, np.where(j < 512, 255, np.where(j < 896, 0, j - 896))).astype(np.uint8)


def idct_islow(coef_zz, qtab):
    """int [..., 64] zigzag coefficients, int [64] natural-order table (or [..., 64]) -> (uint8 [..., 8, 8] samples, in
    range: the values stay where every libjpeg-turbo IDCT agrees)."""
    nat = np.zeros(coef_zz.shape, np.int64)
    nat[..., ZIGZAG] = coef_zz
    deq = (nat * qtab).reshape(coef_zz.shape[:-1] + (8, 8))
    ok = np.abs(deq).max(initial=0) <= IDCT_IN_LIMIT
    ws = np.swapaxes(_idct_1d(np.swapaxes(deq, -1, -2), CONST_BITS - PASS1_BITS), -1, -2)     # columns
    ok = ok and np.abs(ws).max(initial=0) <= IDCT_IN_LIMIT
    out = _idct_1d(ws, CONST_BITS + PASS1_BITS + 3)                                            # rows
    ok = ok and out.min(initial=0) >= IDCT_OUT_LO and out.max(initial=0) <= IDCT_OUT_HI
    return range_limit(out), bool(ok)


def planes(info, coef):
    """Coefficients in scan order -> per component the sample plane [bh*8, bw*8] (uint8) and whether the IDCT stayed in
    range."""
    qt = info["qt"]
    out, ok = [], True
    nb = len(info["blocks"])
    mcux, mcuy = info["mcux"], info["mcuy"]
    cm = coef.reshape(mcuy, mcux, nb, 64)
    for ci, (_, H, V, tq) in enumerate(info["comps"]):
        idx = [k for k, (c, _, _) in enumerate(info["blocks"]) if c == ci]
        smp, good = idct_islow(cm[:, :, idx].astype(np.int64), qt[tq])        # [mcuy, mcux, V*H, 8, 8]
        ok = ok and good
        smp = smp.reshape(mcuy, mcux, V, H, 8, 8).transpose(0, 2, 4, 1, 3, 5)
        out.append(smp.reshape(mcuy * V * 8, mcux * H * 8))
    return out, ok


def upsample(plane, dw, dh, hx, vy, w, h):
    """A downsampled plane (valid dw x dh) -> full resolution [h, w] int64; hx, vy in {1, 2}: the horizontal / vertical
    factors.  Fancy (triangle) filters with context rows clamped to the plane, box replication when dw <= 2 for h2."""
    c = plane[:dh, :dw].astype(np.int64)
    if hx == 1 and vy == 1:
        return c[:h, :w]
    y = np.arange(h)
    x = np.arange(w)
    if hx == 2 and dw <= 2:                            # h2v1_upsample / h2v2_upsample: plain replication
        return c[(y // vy)[:, None], (x // 2)[None, :]]
    if vy == 2:
        near = c[y // 2]
        far = c[np.clip(np.where(y % 2 == 0, y // 2 - 1, y // 2 + 1), 0, dh - 1)]
        if hx == 1:                                    # h1v2
            bias = np.where(y % 2 == 0, 1, 2)[:, None]
            return (3 * near[:, x] + far[:, x] + bias) >> 2
        cs = 3 * near + far                            # h2v2: column sums of the two rows
        col = x // 2
        odd = (x % 2 == 1)
        other = np.clip(np.where(odd, col + 1, col - 1), 0, dw - 1)
        return (3 * cs[:, col] + cs[:, other] + np.where(odd, 7, 8)[None, :]) >> 4
    near = c[y]                                        # h2v1
    col = x // 2
    odd = (x % 2 == 1)
    other = np.clip(np.where(odd, col + 1, col - 1), 0, dw - 1)
    return (3 * near[:, col] + near[:, other] + np.where(odd, 2, 1)[None, :]) >> 2


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_bgr(Y, Cb, Cr):
    """jdcolor.c ycc_rgb_convert with its tables -> uint8 [h, w, 3] BGR."""
    cb, cr = Cb.astype(np.int64) - 128, Cr.astype(np.int64) - 128
    half = 1 << 15
    r = Y + ((_fix(1.40200) * cr + half) >> 16)
    g = Y + ((-_fix(0.71414) * cr + (-_fix(0.34414) * cb + half)) >> 16)
    b = Y + ((_fix(1.77200) * cb + half) >> 16)
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def pixels(info, coef):
    """Coefficients -> (BGR uint8 [h, w, 3], in range)."""
    w, h = info["w"], info["h"]
    pl, ok = planes(info, coef)
    if info["ncomp"] == 1:
        g = pl[0][:h, :w]
        return np.repeat(g[:, :, None], 3, 2), ok
    Hm, Vm = info["hmax"], info["vmax"]
    Y = pl[0][:h, :w].astype(np.int64)
    ch = [upsample(pl[c], info["planes"][c][2], info["planes"][c][3], Hm, Vm, w, h) for c in (1, 2)]
    return ycc_to_bgr(Y, ch[0], ch[1]), ok


def decode(data: bytes, selfsync_bits: int = 0):
    """The whole file -> (status, BGR uint8 [h, w, 3] or None): what cv2.imdecode(buf, IMREAD_COLOR) returns, for every
    file whose status is OK."""
    status, info = parse(data)
    if status:
        return status, None
    try:
        coef = decode_coeffs_selfsync(data, info, selfsync_bits) if selfsync_bits else decode_coeffs(data, info)
    except _Bad as e:
        return e.status, None
    img, ok = pixels(info, coef)
    return (OK, img) if ok else (UNSUPPORTED, None)


def coeffs(data: bytes):
    """-> int16 [n_blocks, 64] zigzag coefficients in scan order (the device's coefficient tap), or None if not OK."""
    status, info = parse(data)
    if status:
        return None
    try:
        return decode_coeffs(data, info).astype(np.int16)
    except _Bad:
        return None
