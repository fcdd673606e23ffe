"""oracle/jpeg_decode.py against cv2.imdecode, byte for byte, over a generated sweep of sizes, qualities, sampling modes,
restart intervals and optimised tables; its self-synchronising decode against its sequential decode; its header parser
against unsupported and malformed files (a status every time, never an exception)."""
import os

import numpy as np
import pytest

from oracle import jpeg as oj
from oracle import jpeg_decode as od

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_decode_cv2.npz")
SAMPLING = {444: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 422: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            440: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, 420: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
MODES = (420, 422, 440, 444, "grey")


def _img(h, w, seed, sigma=10):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, sigma, (h, w, 3)), 0, 255).astype(np.uint8)


def _enc(img, q=95, samp=420, rst=0, opt=False, luma=None, chroma=None):
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if samp == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[samp]]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if opt:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if luma is not None:
        p += [cv2.IMWRITE_JPEG_LUMA_QUALITY, luma, cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma]
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def _same_as_cv2(f):
    st, got = od.decode(f)
    want = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
    return st == od.OK and got.shape == want.shape and np.array_equal(got, want)


def _sweep():
    cases = []
    for w in range(1, 34):
        for h in range(1, 34):
            i = w * 34 + h
            cases.append((h, w, i, dict(q=(95, 50, 10, 100, 75)[i % 5], samp=MODES[i % 5], rst=(0, 1, 3, 0, 5)[i % 4],
                                        opt=i % 7 == 0)))
    for q in range(1, 101):
        cases.append((19 + q % 13, 23 + q % 11, 5000 + q, dict(q=q, samp=MODES[q % 5], luma=(q * 37) % 100 + 1,
                                                                  chroma=(q * 53) % 100 + 1)))
    for i, (h, w) in enumerate([(77, 121), (135, 241), (333, 199), (481, 271), (1079, 1919)]):
        cases.append((h, w, 6000 + i, dict(q=(85, 30, 95, 60, 20)[i], samp=MODES[i % 5], rst=(0, 7, 0, 11, 0)[i],
                                           opt=i % 2 == 1)))
    return cases


def test_oracle_equals_cv2_on_the_generated_sweep():
    n = 0
    for h, w, seed, kw in _sweep():
        assert _same_as_cv2(_enc(_img(h, w, seed), **kw)), (h, w, kw)
        n += 1
    assert n >= 1000


@pytest.mark.parametrize("samp", MODES)
def test_restart_intervals_and_optimised_tables(samp):
    img = _img(70, 101, 7)
    mcus = {420: 5 * 7, 422: 9 * 7, 440: 5 * 13, 444: 9 * 13, "grey": 9 * 13}[samp]
    for rst in (1, 3, mcus - 1, mcus + 4):
        for opt in (False, True):
            assert _same_as_cv2(_enc(img, 80, samp, rst, opt)), (rst, opt)


def test_the_projects_encoder_output():
    for i, (h, w) in enumerate([(1, 1), (17, 33), (64, 48), (101, 77)]):
        img = _img(h, w, 40 + i)
        for q in (95, 50):
            f = oj.encode(img, q)
            assert _same_as_cv2(f)
            assert np.array_equal(od.coeffs(f), oj.blocks(img, q)), (h, w, q)


def _fixture():
    g = np.load(GOLDEN)
    k = 0
    while f"file{k}" in g:
        yield k, g[f"file{k}"].tobytes(), g.get(f"want{k}"), int(g[f"status{k}"])
        k += 1


def test_fixture():
    n = 0
    for k, f, want, status in _fixture():
        st, got = od.decode(f)
        assert st == status, k
        if st == od.OK:
            assert np.array_equal(got, want), k
        n += 1
    assert n >= 30


@pytest.mark.parametrize("bits", [32, 64, 256, 1024])
def test_selfsync_equals_sequential(bits):
    stats = {}
    for k, f, _, status in _fixture():
        if status != od.OK:
            continue
        _, info = od.parse(f)
        seq = od.decode_coeffs(f, info)
        assert np.array_equal(od.decode_coeffs_selfsync(f, info, bits, stats), seq), (k, bits)
    big = _enc(_img(240, 320, 3), 95)
    _, info = od.parse(big)
    assert np.array_equal(od.decode_coeffs_selfsync(big, info, bits, stats), od.decode_coeffs(big, info))
    assert stats["rounds"] >= 1                      # some guess was wrong and had to be synchronised


def _segments(f):
    """[(marker, offset of FF, length field)] up to SOS."""
    out, pos = [], 2
    while True:
        m = f[pos + 1]
        ln = int.from_bytes(f[pos + 2:pos + 4], "big")
        out.append((m, pos, ln))
        if m == 0xDA:
            return out
        pos += 2 + ln


def _seg(f, marker):
    return next((p, ln) for m, p, ln in _segments(f) if m == marker)


def test_unsupported_files_are_classified():
    img = _img(40, 56, 1)
    base = _enc(img, 90)
    prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    assert od.parse(prog)[0] == od.UNSUPPORTED
    p, _ = _seg(base, 0xC0)
    sof = bytearray(base)
    sof[p + 1] = 0xC3                                                       # lossless
    assert od.parse(bytes(sof))[0] == od.UNSUPPORTED
    sof[p + 1] = 0xC9                                                       # arithmetic
    assert od.parse(bytes(sof))[0] == od.UNSUPPORTED
    b12 = bytearray(base)
    b12[p + 4] = 12                                                         # 12-bit
    assert od.parse(bytes(b12))[0] == od.UNSUPPORTED
    s411 = bytearray(base)
    s411[p + 4 + 6 + 1] = 0x41                                              # luma 4x1: 4:1:1
    assert od.parse(bytes(s411))[0] == od.UNSUPPORTED
    for orient, status in ((6, od.UNSUPPORTED), (1, od.OK)):
        exif = b"Exif\x00\x00MM\x00\x2a\x00\x00\x00\x08\x00\x01\x01\x12\x00\x03\x00\x00\x00\x01" + bytes([0, orient, 0, 0]) + b"\x00" * 4
        f = base[:2] + b"\xff\xe1" + (len(exif) + 2).to_bytes(2, "big") + exif + base[2:]
        assert od.parse(f)[0] == status
    two_scans = base[:-2] + base[base.find(b"\xff\xda"):]                   # a second SOS after the first scan
    assert od.parse(two_scans)[0] == od.UNSUPPORTED
    # every one of them still decodes through cv2 on the host
    for f in (prog, two_scans):
        assert cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) is not None


def _marker_after_soi(f, code, payload=b"\x00\x00"):
    return f[:2] + bytes([0xFF, code]) + (len(payload) + 2).to_bytes(2, "big") + payload + f[2:]


def _malformed():
    """(name, file, status) of malformed headers: every one is CORRUPT."""
    base = _enc(_img(40, 56, 2), 90)
    out = []
    sos, sos_len = _seg(base, 0xDA)
    for cut in range(0, sos + 2 + sos_len, 7):                              # truncated anywhere in the headers
        out.append((f"cut at {cut}", base[:cut]))
    p, _ = _seg(base, 0xC0)
    zero = bytearray(base)
    zero[p + 5:p + 7] = b"\x00\x00"
    out.append(("zero height", bytes(zero)))
    zero = bytearray(base)
    zero[p + 7:p + 9] = b"\x00\x00"
    out.append(("zero width", bytes(zero)))
    p, _ = _seg(base, 0xC4)
    many = bytearray(base)
    many[p + 5:p + 21] = bytes([0, 0, 0, 0, 0, 0, 0, 0, 255, 255, 0, 0, 0, 0, 0, 0])
    out.append(("510 codes: more than 256", bytes(many)))
    over = bytearray(base)
    over[p + 5:p + 21] = bytes([3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 9])
    out.append(("3 codes of 1 bit", bytes(over)))
    tables = _segments(base)
    ac0 = next(q for m, q, _ in tables if m == 0xC4 and base[q + 4] == 0x10)    # the luma AC table: 162 codes
    short = bytearray(base)
    short[ac0 + 5:ac0 + 21] = bytes([162] + [0] * 15)
    out.append(("162 codes of 1 bit", bytes(short)))
    p, _ = _seg(base, 0xDB)
    undefined = bytearray(base)
    undefined[p + 4] = 3                                                    # DQT 0 becomes 3: table 0 never defined
    out.append(("DQT id never defined", bytes(undefined)))
    seglen = bytearray(base)
    seglen[p + 2:p + 4] = (0xFFF0).to_bytes(2, "big")
    out.append(("segment runs past the end", bytes(seglen)))
    for code in (0x02, 0xBF, 0xC8, 0xDE, 0xDF, 0xF0, 0xFD):
        out.append((f"unknown marker {code:02X}", _marker_after_soi(base, code)))
    out += [("empty", b""), ("one byte", b"\xff"), ("SOI only", b"\xff\xd8"), ("SOI EOI", b"\xff\xd8\xff\xd9"),
            ("GIF", b"GIF89a"), ("fill bytes only", b"\xff\xd8" + b"\xff" * 50)]
    return out


def test_malformed_headers_give_a_status():
    for name, f in _malformed():
        assert od.parse(f) == (od.CORRUPT, None), name
        assert od.decode(f) == (od.CORRUPT, None), name
    # where libjpeg fails outright, cv2 returns None: the host fallback gives the caller the same None
    for name, f in _malformed():
        if name.startswith(("unknown marker", "zero", "510", "162", "3 codes", "DQT", "SOI", "GIF", "fill")):
            assert cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) is None, name


def _native_parse(files):
    """cc_jpeg_parse (host code of the library) on `files`, its table followed by 1 MB of guard bytes -> status [K]."""
    from clearcam_b200._lib import lib
    L = lib()
    K = len(files)
    lengths = np.array([len(f) for f in files], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    data = np.frombuffer(b"".join(files) + b"\0", np.uint8).copy()
    tb, guard = int(L.cc_jpeg_table_bytes()), 1 << 20
    raw = np.full(16 + K * tb + guard, 0xA5, np.uint8)
    off = (-raw.ctypes.data) % 16
    sizes, status, blocks = np.zeros((K, 2), np.int32), np.zeros(K, np.int32), np.zeros(K, np.int64)
    assert L.cc_jpeg_parse(data.ctypes.data, int(lengths.sum()), offsets.ctypes.data, lengths.ctypes.data, K,
                           raw.ctypes.data + off, sizes.ctypes.data, status.ctypes.data, blocks.ctypes.data) == 0
    assert (raw[:off] == 0xA5).all() and (raw[off + K * tb:] == 0xA5).all(), "the parser wrote outside its table"
    return status


def test_native_parser_classifies_as_the_oracle_and_stays_in_its_table():
    """The library's own marker parser (host code, no GPU needed) on every malformed, unsupported and fixture file: the
    oracle's status, and not one byte written past the table."""
    files = [f for _, f in _malformed()]
    img = _img(40, 56, 1)
    base = _enc(img, 90)
    files.append(cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes())
    exif = b"Exif\x00\x00MM\x00\x2a\x00\x00\x00\x08\x00\x01\x01\x12\x00\x03\x00\x00\x00\x01\x00\x06\x00\x00" + b"\x00" * 4
    files.append(_marker_after_soi(base, 0xE1, exif))
    files.append(base[:-2] + base[base.find(b"\xff\xda"):])
    files += [f for _, f, _, _ in _fixture()]
    want = np.array([od.parse(f)[0] for f in files], np.int32)
    assert np.array_equal(_native_parse(files), want)
    for f, w in zip(files, want):
        assert _native_parse([f])[0] == w


def test_corrupt_scans():
    base = _enc(_img(64, 80, 3), 90)
    _, info = od.parse(base)
    off, ln = info["scan"]
    assert od.decode(base[:off + ln // 2])[0] == od.CORRUPT                 # ends before the last MCU
    inv = bytearray(base)
    inv[off + ln // 3:off + ln // 3 + 8] = b"\xff\x00" * 4
    assert od.decode(bytes(inv))[0] == od.CORRUPT                           # no code of any table is all ones
    rst = _enc(_img(64, 80, 3), 90, rst=1)
    i = rst.find(b"\xff\xd2")
    wrong = rst[:i + 1] + b"\xd6" + rst[i + 2:]
    assert od.decode(wrong)[0] == od.CORRUPT                                # RSTn out of order


def test_coefficients_out_of_range_are_left_to_the_host():
    """A DC so large that libjpeg-turbo's SIMD and C inverse DCTs disagree: reported, not guessed."""
    base = _enc(np.full((8, 8, 3), 128, np.uint8), 100, 444)
    p, _ = _seg(base, 0xDB)
    f = bytearray(base)
    f[p + 5] = 255                                                          # DC quantiser 255 instead of 1
    st, info = od.parse(bytes(f))
    assert st == od.OK
    big = _enc(np.full((8, 8, 3), 255, np.uint8), 100, 444)
    g = bytearray(big)
    g[p + 5] = 255
    assert od.decode(bytes(g))[0] == od.UNSUPPORTED
