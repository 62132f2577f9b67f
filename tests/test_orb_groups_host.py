"""How ORB extraction cuts a batch into groups that share one launch sequence, without a GPU: csrc/orb_groups.h compiled with g++ through
tests/host_orb_groups.cpp.  Every image lands in exactly one group, in order; a group's device bytes and staging stay within their
budgets and its image count within grid z, unless a single image exceeds a budget on its own, which then gets a group of its own; the
flat FAST and blur grids of a group stay within grid x; and equally sized images give the equal-size batch rule
max(1, min(n, 2 GB / device bytes per image, 96 MB / staging per image)) images per group."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
LL = C.c_longlong


@pytest.fixture(scope="module")
def hg():
    so = os.path.join(ROOT, "tests", "_build", "libhost_orb_groups.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.run([CXX, "-std=c++17", "-shared", "-fPIC", "-O2", "-Wall", "-Werror", "-x", "c++",
                    os.path.join(ROOT, "tests", "host_orb_groups.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.hog_image_bytes.restype = LL
    L.hog_image_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.hog_groups.argtypes = [C.POINTER(LL), C.POINTER(LL), C.c_int, LL, LL, C.c_int, C.POINTER(C.c_int)]
    L.hog_dev_budget.restype = LL
    L.hog_stage_budget.restype = LL
    return L


def image_bytes(hg, w, h, raw=True):
    rows = C.c_int()
    return int(hg.hog_image_bytes(w, h, 5000, int(raw), C.byref(rows))), rows.value


def groups(hg, dev, stage=None, dev_budget=None, stage_budget=None, max_images=None):
    n = len(dev)
    d = (LL * max(n, 1))(*dev)
    s = (LL * max(n, 1))(*stage) if stage is not None else None
    out = (C.c_int * (n + 1))()
    g = hg.hog_groups(d, s, n, dev_budget or hg.hog_dev_budget(), stage_budget or hg.hog_stage_budget(),
                      max_images or hg.hog_max_group(), out)
    return list(out[:g + 1]) if n else [0]


def check(starts, dev, stage, dev_budget, stage_budget, max_images):
    n = len(dev)
    assert starts[0] == 0 and starts[-1] == n and all(a < b for a, b in zip(starts, starts[1:]))   # each image in exactly one group
    for a, b in zip(starts, starts[1:]):
        if b - a == 1:
            continue                                       # a single image may exceed a budget on its own
        assert sum(dev[a:b]) <= dev_budget and b - a <= max_images
        if stage is not None:
            assert sum(stage[a:b]) <= stage_budget
        # greedy: the next image would not have fitted
        if b < n:
            assert (sum(dev[a:b + 1]) > dev_budget or b + 1 - a > max_images or
                    (stage is not None and sum(stage[a:b + 1]) > stage_budget))


@pytest.mark.parametrize("w,h,n", [(1024, 768, 7), (1024, 768, 50), (4032, 3024, 50), (3024, 4032, 9), (8, 8, 100000),
                                   (16384, 16384, 3), (640, 480, 1)])
def test_equal_sizes_give_the_equal_size_batch_rule(hg, w, h, n):
    per, _ = image_bytes(hg, w, h)
    img = w * h * 3
    slots = max(1, min(n, (2 << 30) // per, (96 << 20) // img, hg.hog_max_group()))
    want = list(range(0, n, slots)) + [n]
    assert groups(hg, [per] * n, [img] * n) == want


def test_mixed_sizes_respect_budgets_and_grids(hg):
    rs = np.random.RandomState(7)
    sizes = [(4032, 3024), (3024, 4032), (1023, 767), (767, 1023), (1001, 333), (64, 48), (8, 8), (16384, 16384), (8000, 6000)]
    for trial in range(30):
        pick = [sizes[i] for i in rs.randint(0, len(sizes), rs.randint(1, 200))]
        for raw in (True, False):
            info = [image_bytes(hg, w, h, raw) for w, h in pick]
            dev = [b for b, _ in info]
            stage = [w * h * 3 for w, h in pick] if raw else None
            budget = int(rs.choice([hg.hog_dev_budget(), 1 << 28, 1 << 26]))
            st = groups(hg, dev, stage, dev_budget=budget)
            check(st, dev, stage, budget, hg.hog_stage_budget(), hg.hog_max_group())
            for a, b in zip(st, st[1:]):
                # flat FAST (32x32) and blur (64x16) grids: tile rows of the group x words of its widest image < 2^31
                wmax = max(w for w, _ in pick[a:b])
                rows = sum(r for _, r in info[a:b])
                assert (rows // 16 + 8 * (b - a)) * ((wmax + 31) // 32) < 2 ** 31


def test_an_image_over_budget_gets_its_own_group(hg):
    dev = [10, 10, 500, 10, 10, 10]
    assert groups(hg, dev, None, dev_budget=100) == [0, 2, 3, 6]
    assert groups(hg, [500], None, dev_budget=100) == [0, 1]
    assert groups(hg, [10] * 5, [60, 60, 60, 60, 60], dev_budget=100, stage_budget=100) == [0, 1, 2, 3, 4, 5]
    assert groups(hg, [1] * 10, None, max_images=4) == [0, 4, 8, 10]
    assert groups(hg, [], None) == [0]
