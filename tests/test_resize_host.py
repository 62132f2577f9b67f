"""The image downscale without a GPU: the numpy oracle (tests/resize_oracle.py) equals cv2.resize on random B,G,R images over the
factors and sizes the reference can meet; the arithmetic of csrc/resize_math.cuh, compiled with g++ through tests/host_resize.cpp,
equals the oracle, including the 2x2 area path's edge blocks at odd sizes; sfmb200_resize_size gives cv2's shapes and refuses what
cv::resize asserts on."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import resize_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

FACTORS = [float(np.float32(s)) for s in (0.2, 0.25, 0.3, 0.45, 0.5, 0.6, 0.7, 0.75, 0.8, 0.9, 1.25, 1.5, 2.0)]
SIZES = [(1, 37), (37, 1), (1, 1), (2, 3), (9, 9), (173, 99), (175, 101), (64, 48), (333, 221), (1024, 768)]


def _image(w, h, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _cases():
    for k, (w, h) in enumerate(SIZES):
        img = _image(w, h, k)
        for s in FACTORS:
            if R.resize_size(w, h, s) is not None:
                yield f"{w}x{h}@{s:g}", img, s


@pytest.fixture(scope="module")
def hr():
    so = os.path.join(ROOT, "tests", "_build", "libhost_resize.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.run([CXX, "-std=c++17", "-shared", "-fPIC", "-O2", "-x", "c++", os.path.join(ROOT, "tests", "host_resize.cpp"), "-o", so],
                   check=True)
    return C.CDLL(so)


def _harness(hr, img, s):
    h, w = img.shape[:2]
    dw = C.c_int(0); dh = C.c_int(0)
    assert hr.hr_size(w, h, C.c_double(s), C.byref(dw), C.byref(dh)) == 0
    out = np.zeros((dh.value, dw.value, 3), np.uint8)
    src = np.ascontiguousarray(img)
    assert hr.hr_resize(src.ctypes.data_as(C.c_void_p), w, h, C.c_double(s), out.ctypes.data_as(C.c_void_p)) == 0
    return out


def test_oracle_equals_cv2():
    n = 0
    for name, img, s in _cases():
        ref = cv2.resize(img, None, fx=s, fy=s)
        got = R.resize(img, s)
        assert got.shape == ref.shape and np.array_equal(got, ref), name
        n += 1
    assert n > 100


def test_oracle_equals_cv2_4000x3000():
    img = _image(4000, 3000, 99)
    for s in (0.25, 0.5, float(np.float32(0.3))):
        assert np.array_equal(R.resize(img, s), cv2.resize(img, None, fx=s, fy=s)), s


def test_oracle_same_size_is_a_copy():
    img = _image(9, 9, 5)
    for s in (1.0, 1.01, 0.98):                      # 9 * s rounds to 9: cv::resize copies
        assert np.array_equal(R.resize(img, s), img) and np.array_equal(cv2.resize(img, None, fx=s, fy=s), img), s


def test_header_arithmetic_equals_oracle(hr):
    for name, img, s in _cases():
        assert np.array_equal(_harness(hr, img, s), R.resize(img, s)), name
    for s in (1.01, float(np.float32(0.3))):
        img = _image(9, 9, 6) if s > 1 else _image(4000, 3000, 7)
        assert np.array_equal(_harness(hr, img, s), R.resize(img, s)), s


def test_area_path_edge_blocks_at_odd_sizes(hr):
    """Factor 0.5 on odd sizes that round up (175 -> 88, 3 -> 2): the last column / row averages only its in-bounds pixels."""
    for k, (w, h) in enumerate(((175, 101), (3, 3), (5, 175), (175, 4), (7, 9), (1, 3), (3, 1))):
        img = _image(w, h, 40 + k)
        if R.resize_size(w, h, 0.5) is None:
            continue
        ref = cv2.resize(img, None, fx=0.5, fy=0.5)
        assert np.array_equal(R.resize(img, 0.5), ref) and np.array_equal(_harness(hr, img, 0.5), ref), (w, h)
    # the edge mean of two pixels rounds half to even: (5 + 6) / 2 -> 6, (6 + 7) / 2 -> 6, (1 + 2) / 2 -> 2
    img = np.zeros((2, 3, 3), np.uint8)
    img[:, 2, 0] = (5, 6); img[:, 2, 1] = (6, 7); img[:, 2, 2] = (1, 2)
    ref = cv2.resize(img, None, fx=0.5, fy=0.5)
    assert ref[0, 1].tolist() == [6, 6, 2] and np.array_equal(_harness(hr, img, 0.5), ref)


def test_resize_size_matches_cv2_and_refuses():
    from sfm_toy_library_b200 import capi
    f06 = float(np.float32(0.6))
    for w, h, s, want in ((173, 173, 0.5, (86, 86)), (175, 175, 0.5, (88, 88)), (1024, 768, f06, (614, 461)),
                          (4000, 3000, 0.25, (1000, 750)), (9, 9, 1.01, (9, 9))):
        assert capi.resize_size(w, h, s) == want, (w, h, s)
        assert cv2.resize(np.zeros((h, w, 3), np.uint8), None, fx=s, fy=s).shape[:2] == want[::-1]
    for w, h in SIZES:
        for s in FACTORS:
            got = capi.resize_size(w, h, s)
            assert got == R.resize_size(w, h, s), (w, h, s)
            if got is not None:
                assert cv2.resize(np.zeros((h, w, 3), np.uint8), None, fx=s, fy=s).shape[:2] == got[::-1]
    for s in (0.0, -0.5, float("nan"), float("inf"), -float("inf")):
        assert capi.resize_size(640, 480, s) is None, s
    assert capi.resize_size(1, 1, 0.4) is None and capi.resize_size(3, 100, 0.1) is None      # no pixels left
    for w, h, s in ((1, 1, 0.4), (3, 100, 0.1)):
        with pytest.raises(cv2.error):
            cv2.resize(np.zeros((h, w, 3), np.uint8), None, fx=s, fy=s)
