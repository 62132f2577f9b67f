"""The PNG decoder without a GPU: its parser (csrc/png_parse.h) and arithmetic (csrc/png_math.cuh) compiled with g++ by the harness
tests/host_png.cpp.  The serial inflate equals zlib.decompress; the dynamic-header test accepts exactly the headers zlib accepts; the
block-parallel schedule of csrc/png.cu (chain, per-block word decode, pointer-jumping rounds, Adler-32, unfilter, colour, orientation)
gives cv2.imdecode's bytes; sfmb200_image_info reports cv2's shapes and the right statuses; and truncated and corrupted files run
under AddressSanitizer / UndefinedBehaviorSanitizer without a report."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
import png_util as P  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _compile(name, flags):
    so = os.path.join(ROOT, "tests", "_build", name)
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.run([CXX, "-std=c++17", "-shared", "-fPIC", *flags, "-x", "c++", os.path.join(ROOT, "tests", "host_png.cpp"), "-o", so], check=True)
    return so


@pytest.fixture(scope="module")
def hp():
    return C.CDLL(_compile("libhost_png.so", ["-O2"]))


@pytest.fixture(scope="module")
def files():
    return P.matrix()


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _inflate(hp, z):
    a = np.frombuffer(z, np.uint8)
    cap = 64 << 20
    out = np.zeros(cap, np.uint8); n = C.c_size_t(0); nb = C.c_int64(0)
    rc = hp.hp_inflate(_vp(a), C.c_size_t(len(z)), _vp(out), C.c_size_t(cap), C.byref(n), C.byref(nb))
    return rc, out[:n.value].tobytes(), nb.value


def _decode(hp, b):
    a = np.frombuffer(b, np.uint8)
    info = np.zeros(8, np.int64)
    rc = hp.hp_info(_vp(a), C.c_size_t(len(b)), _vp(info))
    if rc:
        return rc, None, None
    out = np.zeros((info[2], info[1], 3), np.uint8); st = np.zeros(5, np.int64)
    rc = hp.hp_decode(_vp(a), C.c_size_t(len(b)), _vp(out), _vp(st))
    return rc, out, st


def _zlib_streams():
    rs = np.random.RandomState(3)
    data = [bytes(rs.randint(0, 256, 5000).astype(np.uint8)), bytes(20000), P.raw_data(P.picture(50, 60, 9), 2, 8, filters=(1, 4)),
            b"abc" * 3000 + bytes(rs.randint(0, 4, 7000).astype(np.uint8))]
    out = []
    for k, d in enumerate(data):
        for st in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
            for wb in (8, 11, 15):
                out.append((f"d{k}_s{st}_w{wb}", P.compress(d, 6, wb, st)))
        for lvl in range(10):
            out.append((f"d{k}_l{lvl}", P.compress(d, lvl)))
        out.append((f"d{k}_sync", P.compress(d, flush_every=999)))
        out.append((f"d{k}_full", P.compress(d, flush_every=1234, flush=zlib.Z_FULL_FLUSH)))
    return out


def test_serial_inflate_equals_zlib(hp, files):
    streams = _zlib_streams() + [(n, P.idat_stream(b)) for n, b in files]
    for name, z in streams:
        rc, out, _ = _inflate(hp, z)
        d = zlib.decompressobj()
        ref = d.decompress(z)
        assert rc == 0 and out == ref, name


def _zlib_header_verdict(z):
    """False if zlib refuses the stream in its first dynamic header, True if the header passed (whatever happens after it)"""
    try:
        zlib.decompressobj().decompress(z)
    except zlib.error as e:
        msg = str(e)
        header = ("too many length or distance symbols", "invalid code lengths set", "invalid bit length repeat",
                  "invalid literal/lengths set", "invalid distances set", "invalid code -- missing end-of-block")
        return not any(h in msg for h in header)
    return True


def test_dynamic_header_accepts_what_zlib_accepts(hp):
    base = P.compress(P.raw_data(P.picture(40, 50, 11), 2, 8, filters=(4,)), 9)
    assert (base[2] >> 1) & 3 == 2                              # the first block is dynamic
    rs = np.random.RandomState(7)
    acc = rej = 0
    for t in range(3000):
        b = bytearray(base)
        for _ in range(1 + t % 3):
            bit = 16 + 3 + rs.randint(0, 14 + 19 * 3 + 80)      # inside HLIT .. the first code lengths
            b[bit >> 3] ^= 1 << (bit & 7)
        b = bytes(b)
        a = np.frombuffer(b[2:], np.uint8)
        ours = bool(hp.hp_dynamic_header(_vp(a), C.c_size_t(len(b) - 2), C.c_uint64(3)))
        assert ours == _zlib_header_verdict(b), t
        acc += ours; rej += not ours
    assert acc > 0 and rej > 500, (acc, rej)            # a flipped header bit almost always breaks a code


def test_block_parallel_decode_equals_cv2(hp, files):
    chained = spec = 0
    for name, b in files:
        rc, out, st = _decode(hp, b)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert rc == 0 and out.shape == ref.shape and np.array_equal(out, ref), name
        chained += st[0] > 1
        spec += st[4]
        if not name.startswith(("ct", "adam7", "filter", "exif", "strategy_fixed", "level0", "split", "sync", "full")):
            assert st[4] == st[0] - st[1] - st[2], (name, st)    # the scan found every dynamic block start
    assert chained >= 4 and spec > 60                   # crazyhorse, the flushed and the large-window streams


def test_image_info_matches_cv2_and_refuses(files):
    from sfm_toy_library_b200 import capi
    import jpeg_util as J
    for name, b in files:
        rc, f, w, h = capi.image_info(b)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert rc == 0 and f == capi.FORMAT_PNG and (h, w, 3) == ref.shape, name
    rc, f, w, h = capi.image_info(J.crazyhorse())
    assert (rc, f, w, h) == (0, capi.FORMAT_JPEG, 1024, 768)
    assert capi.image_info(b"GIF89a" + bytes(30))[0] == 1
    assert capi.image_info(b"")[0] == 1
    deferred = {"not_enough_data", "filter5", "adler", "btype3", "stored_nlen", "hlit_287", "cl_oversubscribed", "distance_too_far"}
    for name, b, status in P.refused():
        assert capi.image_info(b)[0] == (0 if name in deferred else status), name    # stream errors are only found by decoding


def test_refused_files(hp):
    for name, b, status in P.refused():
        assert _decode(hp, b)[0] == status, name
        if status == P.INVALID:
            assert cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) is None, name


def test_sanitizers_on_truncated_and_corrupted_files(tmp_path):
    so = _compile("libhost_png_san.so", ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"])
    base = P.make_png(P.picture(20, 24, 8), 2, 8, 1, filters=(4, 1))
    fixed = P.make_png(P.picture(16, 20, 9), 2, 8, filters=(2,), strategy=zlib.Z_FIXED)
    rs = np.random.RandomState(1234)
    cases = [base[:k] for k in (3, 20, 40, len(base) // 2, len(base) - 3)]
    for i in range(300):
        src = bytearray(base if i % 2 == 0 else fixed)
        idat = src.find(b"IDAT")
        for _ in range(1 + i % 3):
            src[rs.randint(idat + 4, len(src) - 16)] = rs.randint(0, 256)
        # re-seal the IDAT CRC so that the corruption reaches the inflate
        n = int.from_bytes(src[idat - 4:idat], "big")
        src[idat + 4 + n:idat + 8 + n] = (zlib.crc32(bytes(src[idat:idat + 4 + n])) & 0xffffffff).to_bytes(4, "big")
        cases.append(bytes(src))
    blob = tmp_path / "cases.bin"
    with open(blob, "wb") as f:
        for b in cases:
            f.write(len(b).to_bytes(4, "little") + b)
    driver = (
        "import ctypes as C, numpy as np\n"
        f"L = C.CDLL({so!r})\n"
        f"d = open({str(blob)!r}, 'rb').read(); i = 0; res = []\n"
        "while i < len(d):\n"
        "    n = int.from_bytes(d[i:i + 4], 'little'); b = d[i + 4:i + 4 + n]; i += 4 + n\n"
        "    a = np.frombuffer(b, np.uint8); info = np.zeros(8, np.int64); st = np.zeros(4, np.int64)\n"
        "    rc = L.hp_info(a.ctypes.data_as(C.c_void_p), C.c_size_t(n), info.ctypes.data_as(C.c_void_p))\n"
        "    if rc == 0:\n"
        "        out = np.zeros(int(info[1] * info[2] * 3), np.uint8)\n"
        "        rc = L.hp_decode(a.ctypes.data_as(C.c_void_p), C.c_size_t(n), out.ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p))\n"
        "    res.append(rc)\n"
        "print(' '.join(map(str, res)))\n")
    env = dict(os.environ, LD_PRELOAD=subprocess.run([CXX, "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip(),
               ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")
    r = subprocess.run(["python3", "-c", driver], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-3000:]
    res = [int(x) for x in r.stdout.split()]
    assert len(res) == len(cases)
    assert all(x == 1 for x in res[:5]), res[:5]
    assert all(x in (0, 1) for x in res[5:])
    print("300 corruptions: %d decoded, %d invalid" % (res[5:].count(0), res[5:].count(1)))
