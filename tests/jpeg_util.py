"""Test inputs of the JPEG decoder: a seeded synthetic matrix encoded with cv2.imencode (quality, sampling, restart interval,
optimised tables, sizes and EXIF orientation, each varied around a 1023x767 q95 4:2:0 base; every sampling x restart combination at
1023x767 and 17x9), the committed crazyhorse JPEG, and the files the decoder must refuse."""
import os
import struct

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def crazyhorse():
    with open(os.path.join(GOLDEN, "crazyhorse_0.jpg"), "rb") as f:
        return f.read()


def picture(w, h, seed):
    """Smooth noise with gradients and hard edges: every coefficient band and plenty of 0xFF stuffing at high quality."""
    import cv2
    rs = np.random.RandomState(seed)
    im = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if min(w, h) > 4:
        im = cv2.GaussianBlur(im, (0, 0), 1.5)
    yy, xx = np.mgrid[0:h, 0:w]
    im[..., 0] = np.clip(im[..., 0].astype(int) + xx * 200 // w - 100, 0, 255)
    im[..., 2] = np.clip(im[..., 2].astype(int) + yy * 200 // h - 100, 0, 255)
    for _ in range(max(1, w * h // 20000)):
        x, y, s = rs.randint(0, w), rs.randint(0, h), rs.randint(1, 60)
        im[y:y + s, x:x + s] = rs.randint(0, 256, 3)
    return im


def exif_app1(orientation):
    """An APP1 segment holding a little-endian TIFF block whose IFD0 has one entry: Orientation (0x0112, SHORT)."""
    tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack("<I", 0)
    body = b"Exif\x00\x00" + tiff
    return b"\xff\xe1" + struct.pack(">H", len(body) + 2) + body


def encode(w, h, q=95, sampling="420", rst=0, optimize=False, grey=False, orientation=None, seed=0):
    import cv2
    im = picture(w, h, seed)
    if grey:
        im = np.ascontiguousarray(im[..., 1])
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)]
    if not grey:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    ok, buf = cv2.imencode(".jpg", im, params)
    assert ok
    b = buf.tobytes()
    if orientation is not None:
        b = b[:2] + exif_app1(orientation) + b[2:]
    return b


def matrix(big=True):
    """[(name, bytes)]: the synthetic matrix.  big=False leaves out the 4000x3000 file."""
    cases = []
    seed = 0
    def add(name, **kw):
        nonlocal seed
        seed += 1
        cases.append((name, encode(seed=seed, **kw)))
    for w, h in ((1023, 767), (17, 9)):
        for s in SAMPLING:
            for rst in (0, 1, 7):
                add(f"{w}x{h}_q95_{s}_rst{rst}", w=w, h=h, sampling=s, rst=rst)
        add(f"{w}x{h}_grey", w=w, h=h, grey=True)
        add(f"{w}x{h}_grey_rst7", w=w, h=h, grey=True, rst=7)
    for q in (50, 75, 100):
        add(f"1023x767_q{q}_420", w=1023, h=767, q=q)
    add("1023x767_q95_420_optimized", w=1023, h=767, optimize=True)
    add("1023x767_q75_422_optimized_rst7", w=1023, h=767, q=75, sampling="422", optimize=True, rst=7)
    for w, h in ((1, 1), (7, 5)):
        add(f"{w}x{h}_q95_420", w=w, h=h)
        add(f"{w}x{h}_q95_444", w=w, h=h, sampling="444")
    for o in range(1, 9):
        add(f"1023x767_q95_420_orientation{o}", w=1023, h=767, orientation=o)
    add("17x9_q95_422_orientation6", w=17, h=9, sampling="422", orientation=6)
    if big:
        add("4000x3000_q95_420", w=4000, h=3000)
    return cases


def entropy_start(b):
    """Offset of the first entropy-coded byte (just after the SOS segment)."""
    i = b.index(b"\xff\xda")
    return i + 2 + struct.unpack(">H", b[i + 2:i + 4])[0]


def refused():
    """[(name, bytes, expected status)]: files the decoder must refuse.  1 = SFMB200_ERR_INVALID, 5 = SFMB200_ERR_UNSUPPORTED."""
    import cv2
    im = picture(64, 48, 99)
    base = encode(64, 48, seed=99)
    ok, prog = cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    sof = base.index(b"\xff\xc0")
    p12 = bytearray(base); p12[sof + 4] = 12
    c4 = bytearray(base); c4[sof + 9] = 4
    s = entropy_start(base)
    undefined = bytearray(base); undefined[s:s + 8] = b"\xff\x00" * 4          # 32 one-bits: no Huffman code is all ones
    flipped = bytearray(base); flipped[1] ^= 0xFF                              # SOI destroyed
    return [("progressive", prog.tobytes(), 5), ("12bit_header", bytes(p12), 5), ("4_components", bytes(c4), 5),
            ("truncated", base[:len(base) // 2], 1), ("truncated_headers", base[:s - 20], 1), ("undefined_code", bytes(undefined), 1),
            ("soi_flipped", bytes(flipped), 1)]
