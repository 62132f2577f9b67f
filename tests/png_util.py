"""PNG fixtures for the decoder tests: a small PNG writer for what cv2.imencode cannot write (palette and sub-byte depths, Adam7, fixed
per-row filters, IDAT splits, zlib strategies / window sizes / flush points, eXIf, ancillary chunks), files cv2.imencode writes, and the
refused files with the status the decoder gives them."""
import os
import struct
import zlib

import numpy as np

try:
    import cv2
except ImportError:                                   # the tests that need cv2 skip themselves
    cv2 = None

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIG = b"\x89PNG\r\n\x1a\n"
INVALID, UNSUPPORTED = 1, 5
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
A7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]   # x0, y0, dx, dy


def chunk(t, d):
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)


def ihdr(w, h, bd, ct, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bd, ct, 0, 0, interlace))


def exif(orientation, little=False):
    if little:
        return b"II\x2a\x00\x08\x00\x00\x00" + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, orientation, 0) + b"\x00" * 4
    return b"MM\x00\x2a\x00\x00\x00\x08" + struct.pack(">H", 1) + struct.pack(">HHIHH", 0x0112, 3, 1, orientation, 0) + b"\x00" * 4


def pack_row(samples, bd):
    """samples: 1-D array of sample values of one row -> bytes"""
    s = np.asarray(samples, np.int64)
    if bd == 16:
        return s.astype(">u2").tobytes()
    if bd == 8:
        return s.astype(np.uint8).tobytes()
    per = 8 // bd
    pad = (-len(s)) % per
    s = np.r_[s, np.zeros(pad, np.int64)].reshape(-1, per)
    b = np.zeros(len(s), np.int64)
    for k in range(per):
        b |= s[:, k] << (8 - bd * (k + 1))
    return b.astype(np.uint8).tobytes()


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def filter_rows(rows, bpp, filters):
    """rows: list of raw row bytes; filters: per row filter type (0-4) -> the filtered data with filter bytes"""
    out = bytearray()
    prev = bytes(len(rows[0])) if rows else b""
    for r, row in enumerate(rows):
        f = filters[r % len(filters)]
        out.append(f)
        for x in range(len(row)):
            a = row[x - bpp] if x >= bpp else 0
            b = prev[x]
            c = prev[x - bpp] if x >= bpp else 0
            pred = (0, a, b, (a + b) >> 1, _paeth(a, b, c))[f]
            out.append((row[x] - pred) & 255)
        prev = row
    return bytes(out)


def raw_data(samples, ct, bd, interlace=0, filters=(0,)):
    """samples: [h, w, channels] ints -> filtered data of every pass"""
    h, w, c = samples.shape
    bpp = max(1, c * bd // 8)
    passes = A7 if interlace else [(0, 0, 1, 1)]
    out = b""
    for x0, y0, dx, dy in passes:
        sub = samples[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        rows = [pack_row(sub[r].reshape(-1), bd) for r in range(sub.shape[0])]
        out += filter_rows(rows, bpp, filters)
    return out


def compress(raw, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, strategy)
    if not flush_every:
        return co.compress(raw) + co.flush()
    out = b""
    for k in range(0, len(raw), flush_every):
        out += co.compress(raw[k:k + flush_every]) + co.flush(flush)
    return out + co.flush()


def make_png(samples, ct, bd, interlace=0, filters=(0,), zdata=None, split=None, pre=b"", post=b"", palette=None, **zkw):
    samples = np.asarray(samples)
    if samples.ndim == 2:
        samples = samples[:, :, None]
    h, w = samples.shape[:2]
    z = zdata if zdata is not None else compress(raw_data(samples, ct, bd, interlace, filters), **zkw)
    if split is None:
        idat = chunk(b"IDAT", z)
    else:
        idat, k, i = b"", 0, 0
        while k < len(z) or i == 0:
            n = split[i % len(split)]
            idat += chunk(b"IDAT", z[k:k + n]); k += n; i += 1
    plte = chunk(b"PLTE", bytes(palette)) if palette is not None else b""
    return SIG + ihdr(w, h, bd, ct, interlace) + plte + pre + idat + post + chunk(b"IEND", b"")


def idat_stream(png):
    """the concatenated IDAT payloads of a PNG file (its zlib stream)"""
    i, z = 8, b""
    while i + 8 <= len(png):
        n = struct.unpack(">I", png[i:i + 4])[0]
        if png[i + 4:i + 8] == b"IDAT":
            z += png[i + 8:i + 8 + n]
        i += 12 + n
    return z


def _rs(seed):
    return np.random.RandomState(seed)


def picture(h, w, seed, channels=3):
    """seeded smooth picture with some texture, uint8 [h, w, channels]"""
    rs = _rs(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * (3 + k) + yy * (5 - k) + rs.randint(0, 50)) % 256 for k in range(channels)], -1)
    noise = rs.randint(0, 24, (h, w, channels))
    return ((base + noise) % 256).astype(np.uint8)


def crazyhorse():
    return cv2.imread(os.path.join(ROOT, "tests", "golden", "crazyhorse_0.jpg"))


def imencode(img, params=()):
    ok, e = cv2.imencode(".png", img, list(params))
    assert ok
    return e.tobytes()


def hand_matrix():
    """files from the hand-written writer: (name, bytes)"""
    out = []
    rs = _rs(5)
    for ct, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for bd in depths:
            for il in (0, 1):
                h, w = (13, 19) if il == 0 else (11, 9)
                c = CHANNELS[ct]
                hi = (1 << bd) - 1
                s = rs.randint(0, hi + 1, (h, w, c))
                pal = None
                if ct == 3:
                    npal = min(1 << bd, 200)
                    pal = rs.randint(0, 256, 3 * npal).astype(np.uint8).tolist()
                    s = rs.randint(0, 1 << bd, (h, w, 1))            # indices past PLTE included when 2^bd > npal
                out.append((f"ct{ct}_bd{bd}_il{il}", make_png(s, ct, bd, il, filters=(0, 1, 2, 3, 4), palette=pal)))
    pic = picture(17, 23, 1)
    for f in range(5):
        out.append((f"filter{f}", make_png(pic, 2, 8, filters=(f,))))
    out.append(("filters_mixed_adam7", make_png(pic, 2, 8, 1, filters=(4, 0, 3, 1, 2))))
    for w, h in ((1, 1), (2, 3), (5, 1), (7, 7), (3, 9)):
        out.append((f"adam7_{w}x{h}", make_png(picture(h, w, w * 10 + h), 2, 8, 1, filters=(4, 1))))
    big = picture(64, 80, 2)
    for split in ((1,), (0, 7, 1), (100, 3, 2000)):
        out.append((f"split_{'_'.join(map(str, split))}", make_png(big, 2, 8, filters=(1, 4), split=split)))
    for st, nm in ((zlib.Z_DEFAULT_STRATEGY, "default"), (zlib.Z_FILTERED, "filtered"), (zlib.Z_HUFFMAN_ONLY, "huffman"),
                   (zlib.Z_RLE, "rle"), (zlib.Z_FIXED, "fixed")):
        out.append((f"strategy_{nm}", make_png(big, 2, 8, filters=(0, 4), strategy=st)))
    for wb in (8, 9, 12, 15):
        out.append((f"wbits{wb}", make_png(big, 2, 8, filters=(2,), wbits=wb)))
    for lvl in (0, 1, 9):
        out.append((f"level{lvl}", make_png(big, 2, 8, filters=(1,), level=lvl)))
    out.append(("sync_flush", make_png(big, 2, 8, filters=(4,), flush_every=1000)))
    out.append(("full_flush", make_png(big, 2, 8, filters=(4,), flush_every=777, flush=zlib.Z_FULL_FLUSH)))
    small = picture(6, 10, 3)
    for o in range(1, 9):
        out.append((f"exif{o}_before", make_png(small, 2, 8, pre=chunk(b"eXIf", exif(o)))))
        out.append((f"exif{o}_after_le", make_png(small, 2, 8, post=chunk(b"eXIf", exif(o, little=True)))))
    bad = bytearray(chunk(b"eXIf", exif(6))); bad[-1] ^= 1
    out.append(("exif_bad_crc", make_png(small, 2, 8, pre=bytes(bad))))
    anc = (chunk(b"tRNS", b"\x00\x01\x00\x02\x00\x03") + chunk(b"gAMA", struct.pack(">I", 100000)) + chunk(b"sRGB", b"\x00")
           + chunk(b"sBIT", b"\x05\x06\x05") + chunk(b"cHRM", bytes(32)) + chunk(b"zzZz", b"unknown") + chunk(b"tEXt", b"k\x00v"))
    out.append(("ancillary", make_png(small, 2, 8, pre=anc)))
    badtext = bytearray(chunk(b"tEXt", b"a\x00b")); badtext[-1] ^= 1
    out.append(("ancillary_bad_crc", make_png(small, 2, 8, pre=bytes(badtext))))
    out.append(("palette_trns", make_png(rs.randint(0, 4, (5, 6, 1)), 3, 8, palette=[9, 8, 7, 6, 5, 4, 3, 2, 1, 0, 0, 0],
                                         pre=chunk(b"tRNS", b"\x00\x80"))))
    out.append(("grey_trns_gama", make_png(rs.randint(0, 256, (5, 6, 1)), 0, 8, pre=chunk(b"tRNS", b"\x00\x07") + chunk(b"gAMA", struct.pack(">I", 45455)))))
    out.append(("rgba_alpha0", make_png(np.array([[[1, 2, 3, 0], [200, 100, 50, 255]]]), 6, 8)))
    out.append(("grey16_highbyte", make_png(np.array([[[0x12ff], [0x1280], [0xfe80], [0x0080]]]), 0, 16)))
    raw = raw_data(picture(9, 12, 4), 2, 8)
    out.append(("extra_compressed_data", make_png(picture(9, 12, 4), 2, 8, zdata=zlib.compress(raw + b"\x00" * 50))))
    out.append(("extra_idat_bytes", make_png(picture(9, 12, 4), 2, 8, zdata=zlib.compress(raw) + b"garbage")))
    return out


def cv2_matrix(big=False):
    """files cv2.imencode writes: (name, bytes)"""
    out = []
    ch = crazyhorse()
    out.append(("crazyhorse_default", imencode(ch)))
    for lvl in range(10):
        out.append((f"synthetic_level{lvl}", imencode(picture(61, 83, 10 + lvl), [cv2.IMWRITE_PNG_COMPRESSION, lvl])))
    for st in (cv2.IMWRITE_PNG_STRATEGY_DEFAULT, cv2.IMWRITE_PNG_STRATEGY_FILTERED, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY,
               cv2.IMWRITE_PNG_STRATEGY_RLE, cv2.IMWRITE_PNG_STRATEGY_FIXED):
        out.append((f"synthetic_strategy{st}", imencode(picture(70, 90, 30 + st), [cv2.IMWRITE_PNG_STRATEGY, st])))
    out.append(("grey", imencode(cv2.cvtColor(picture(50, 70, 40), cv2.COLOR_BGR2GRAY))))
    out.append(("rgb16", imencode(picture(40, 50, 41).astype(np.uint16) * 257 + 3)))
    out.append(("rgba", imencode(np.dstack([picture(40, 50, 42), picture(40, 50, 43, 1)]))))
    out.append(("bilevel", imencode(cv2.cvtColor(picture(33, 65, 44), cv2.COLOR_BGR2GRAY), [cv2.IMWRITE_PNG_BILEVEL, 1])))
    if big:
        out.append(("crazyhorse_level1", imencode(ch, [cv2.IMWRITE_PNG_COMPRESSION, 1])))
        out.append(("crazyhorse_level9", imencode(ch, [cv2.IMWRITE_PNG_COMPRESSION, 9])))
        out.append(("crazyhorse_fixed", imencode(ch, [cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_STRATEGY_FIXED])))
    return out


def matrix(big=False):
    return hand_matrix() + cv2_matrix(big)


def refused():
    """(name, bytes, status) of files every decode refuses"""
    pic = picture(9, 12, 6)
    raw = raw_data(pic, 2, 8)
    good = make_png(pic, 2, 8)
    out = []
    out.append(("truncated", good[:len(good) // 2], INVALID))
    out.append(("no_iend", good[:-12], INVALID))
    out.append(("not_png", b"\x89PNG\r\n\x1a\x0b" + good[8:], INVALID))
    b = bytearray(good); b[8 + 8 + 3] ^= 1
    out.append(("ihdr_crc", bytes(b), INVALID))
    b = bytearray(good); b[-12 - 5] ^= 1
    out.append(("idat_crc", bytes(b), INVALID))
    out.append(("not_enough_data", make_png(pic, 2, 8, zdata=zlib.compress(raw[:-20])), INVALID))
    out.append(("filter5", make_png(pic, 2, 8, zdata=zlib.compress(bytes([5]) + raw[1:])), INVALID))
    z = bytearray(zlib.compress(raw)); z[-1] ^= 1
    out.append(("adler", make_png(pic, 2, 8, zdata=bytes(z)), INVALID))
    out.append(("btype3", make_png(pic, 2, 8, zdata=b"\x78\x9c\x07" + bytes(40)), INVALID))
    out.append(("stored_nlen", make_png(pic, 2, 8, zdata=b"\x78\x01\x01\x05\x00\xfb\xff" + bytes(5)), INVALID))
    # dynamic headers zlib refuses: HLIT 287+, an over-subscribed code-length code
    out.append(("hlit_287", make_png(pic, 2, 8, zdata=b"\x78\x9c" + bytes([0b11111101, 0xff, 0xff, 0xff] + [0] * 40)), INVALID))
    out.append(("cl_oversubscribed", make_png(pic, 2, 8, zdata=b"\x78\x9c" + bytes([0b00000101, 0, 0x90, 0x24] + [0] * 40)), INVALID))
    out.append(("distance_too_far", make_png(pic, 2, 8, zdata=b"\x78\x01" + _fixed_far()), INVALID))
    out.append(("zlib_header", make_png(pic, 2, 8, zdata=b"\x79\x9c" + zlib.compress(raw)[2:]), INVALID))
    out.append(("fdict", make_png(pic, 2, 8, zdata=b"\x78\xbb" + zlib.compress(raw)[2:]), INVALID))
    out.append(("bad_colour_type", SIG + ihdr(4, 4, 8, 5) + chunk(b"IDAT", zlib.compress(bytes(20))) + chunk(b"IEND", b""), INVALID))
    out.append(("palette_no_plte", SIG + ihdr(4, 1, 8, 3) + chunk(b"IDAT", zlib.compress(bytes(5))) + chunk(b"IEND", b""), INVALID))
    out.append(("unknown_critical", make_png(pic, 2, 8, pre=chunk(b"ABCD", b"x")), INVALID))
    actl = chunk(b"acTL", struct.pack(">II", 1, 0))
    out.append(("apng", make_png(pic, 2, 8, pre=actl), UNSUPPORTED))
    return out


def _fixed_far():
    """a fixed-Huffman block whose first symbol is a copy at distance 1: nothing precedes it"""
    bits = []

    def put(v, n, rev=False):
        for k in range(n):
            bits.append((v >> (n - 1 - k)) & 1 if rev else (v >> k) & 1)
    put(1, 1); put(1, 2)                 # BFINAL, fixed
    put(0b0000001, 7, rev=True)          # length code 257 (length 3)
    put(0b00000, 5, rev=True)            # distance code 0 (distance 1)
    put(0, 7, rev=True)                  # end of block
    bits += [0] * ((-len(bits)) % 8)
    return bytes(sum(bits[i + k] << k for k in range(8)) for i in range(0, len(bits), 8)) + b"\x00\x00\x00\x01"
