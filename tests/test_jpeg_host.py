"""The JPEG decoder without a GPU: its parser (csrc/jpeg_parse.h) and arithmetic (csrc/jpeg_math.cuh) compiled with g++ by the harness
tests/host_jpeg.cpp decode the synthetic matrix and the crazyhorse file byte-identically to cv2.imdecode; the self-synchronising
subsequence decode gives the serial decode's coefficient blocks; sfmb200_jpeg_info reports cv2's shapes and the right statuses; and
under AddressSanitizer / UndefinedBehaviorSanitizer truncated and corrupted files decode without a report."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_util as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _compile(name, flags):
    so = os.path.join(ROOT, "tests", "_build", name)
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.run([CXX, "-std=c++17", "-shared", "-fPIC", *flags, "-x", "c++", os.path.join(ROOT, "tests", "host_jpeg.cpp"), "-o", so], check=True)
    return so


@pytest.fixture(scope="module")
def hj():
    return C.CDLL(_compile("libhost_jpeg.so", ["-O2"]))


@pytest.fixture(scope="module")
def files():
    return J.matrix() + [("crazyhorse_0", J.crazyhorse())]


def _decode(hj, b, S=0):
    info = np.zeros(6, np.int64)
    a = np.frombuffer(b, np.uint8)
    rc = hj.hj_info(a.ctypes.data_as(C.c_void_p), C.c_size_t(len(b)), info.ctypes.data_as(C.c_void_p))
    if rc:
        return rc, None, None, None
    out = np.zeros((info[3], info[2], 3), np.uint8); coef = np.zeros(info[5] * 64, np.int16); st = np.zeros(6, np.int64)
    rc = hj.hj_decode(a.ctypes.data_as(C.c_void_p), C.c_size_t(len(b)), C.c_uint32(S), out.ctypes.data_as(C.c_void_p),
                      coef.ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p))
    return rc, out, coef, st


def test_serial_decode_equals_cv2(hj, files):
    for name, b in files:
        rc, out, _, _ = _decode(hj, b)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert rc == 0 and out.shape == ref.shape and np.array_equal(out, ref), name


def test_subsequence_decode_equals_serial(hj, files):
    extra, first, subs = 0, 0, 0
    for name, b in files:
        if name.startswith("4000x3000"):
            continue
        rc0, out0, c0, _ = _decode(hj, b)
        rc1, out1, c1, st = _decode(hj, b, 64)
        assert rc0 == rc1 == 0 and np.array_equal(c0, c1) and np.array_equal(out0, out1), name
        first += st[0]; extra += st[1]; subs += st[2]
    print(f"64-bit subsequences: {subs}, codewords of the first pass {first}, decoded again to synchronise {extra} "
          f"({extra / subs:.1f} per subsequence)")
    rc, _, c0, _ = _decode(hj, J.crazyhorse())
    for S in (256, 1024):
        rc, _, c1, st = _decode(hj, J.crazyhorse(), S)
        assert rc == 0 and np.array_equal(c0, c1)
        print(f"crazyhorse, {S}-bit subsequences: {st[2]}, exits moved in round 1 / 2: {st[3]} / {st[4]}, "
              f"extra codewords per subsequence {st[1] / st[2]:.1f}")


def test_jpeg_info_matches_cv2_and_refuses(files):
    from sfm_toy_library_b200 import capi
    for name, b in files:
        rc, w, h, c = capi.jpeg_info(b)
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        assert rc == 0 and (h, w, 3) == ref.shape and c == (1 if "grey" in name else 3), name
    for name, b, status in J.refused():
        rc = capi.jpeg_info(b)[0]
        assert rc == (0 if name == "undefined_code" else status), name       # a bad code is only found by decoding


def test_refused_files_in_the_harness(hj):
    for name, b, status in J.refused():
        assert _decode(hj, b)[0] == status, name
        assert _decode(hj, b, 64)[0] == status, name


def test_sanitizers_on_truncated_and_corrupted_files(tmp_path):
    so = _compile("libhost_jpeg_san.so", ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"])
    base = J.encode(96, 64, q=90, sampling="422", rst=3, seed=7)
    plain = J.encode(80, 56, q=75, sampling="420", seed=8)
    s0, s1 = J.entropy_start(base), J.entropy_start(plain)
    rs = np.random.RandomState(1234)
    cases = [base[:k] for k in (3, s0 - 5, s0 + 10, len(base) // 2, len(base) - 3)]
    for i in range(200):
        src, s = (base, s0) if i % 2 == 0 else (plain, s1)
        b = bytearray(src)
        for _ in range(1 + i % 3):
            b[rs.randint(s, len(b) - 2)] = rs.randint(0, 256)
        cases.append(bytes(b))
    blob = tmp_path / "cases.bin"
    with open(blob, "wb") as f:
        for b in cases:
            f.write(len(b).to_bytes(4, "little") + b)
    driver = (
        "import ctypes as C, numpy as np, sys\n"
        f"L = C.CDLL({so!r})\n"
        f"d = open({str(blob)!r}, 'rb').read(); i = 0; res = []\n"
        "while i < len(d):\n"
        "    n = int.from_bytes(d[i:i + 4], 'little'); b = d[i + 4:i + 4 + n]; i += 4 + n\n"
        "    a = np.frombuffer(b, np.uint8); info = np.zeros(6, np.int64); st = np.zeros(6, np.int64)\n"
        "    rc = L.hj_info(a.ctypes.data_as(C.c_void_p), C.c_size_t(n), info.ctypes.data_as(C.c_void_p))\n"
        "    if rc == 0:\n"
        "        out = np.zeros(int(info[2] * info[3] * 3), np.uint8)\n"
        "        rc = max(L.hj_decode(a.ctypes.data_as(C.c_void_p), C.c_size_t(n), C.c_uint32(S), out.ctypes.data_as(C.c_void_p), None,\n"
        "                             st.ctypes.data_as(C.c_void_p)) for S in (0, 64))\n"
        "    res.append(rc)\n"
        "print(' '.join(map(str, res)))\n")
    env = dict(os.environ, LD_PRELOAD=subprocess.run([CXX, "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip(),
               ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")
    r = subprocess.run(["python3", "-c", driver], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-3000:]
    res = [int(x) for x in r.stdout.split()]
    assert len(res) == len(cases)
    assert all(x == 1 for x in res[:5]), res[:5]                    # truncated files are INVALID
    assert all(x in (0, 1, 5) for x in res[5:])
    print("200 corruptions: %d decoded, %d invalid, %d unsupported" % (res[5:].count(0), res[5:].count(1), res[5:].count(5)))
