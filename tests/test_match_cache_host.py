"""The per-call matcher's resident-image arena without a GPU: csrc/match_cache.h, compiled with g++ through tests/host_match_cache.cpp,
is driven the way sfmb200_match_knn2_ratio drives it, with the device buffers modelled by DevBuf::reserve's growth rule.  After every
call the capacity rule holds (rows_cap * width + 16 <= desc capacity, blk_cap * block bytes <= exp capacity), every resident image
lies inside both buffers, and no placement reaches the guard in cache_acquire.  Covers the width switches that once let the arena
take rows sized for a narrower width (32 -> 64 bytes over 9000-row images, 16 -> 128 bytes) and seeded random call sequences."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
HIT, MISS, REFUSED = 0, 1, 2


@pytest.fixture(scope="module")
def hm():
    so = os.path.join(ROOT, "tests", "_build", "libhost_match_cache.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.run([CXX, "-std=c++17", "-shared", "-fPIC", "-O2", "-Wall", "-Werror", "-x", "c++",
                    os.path.join(ROOT, "tests", "host_match_cache.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.hmc_new.restype = C.c_void_p
    L.hmc_free.argtypes = [C.c_void_p]
    L.hmc_call.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_int, C.c_uint64, C.c_int, C.c_int,
                           C.POINTER(C.c_longlong)]
    L.hmc_entries.argtypes = [C.c_void_p, C.POINTER(C.c_longlong), C.c_int]
    L.hmc_set_rows_cap.argtypes = [C.c_void_p, C.c_longlong]
    L.hmc_block_bytes.restype = C.c_longlong
    return L


def _width(desc_bytes):
    return next(w for w in (16, 32, 64, 128) if desc_bytes <= w)


class Arena:
    """One context's arena.  Images are named by small integers standing for host pointers."""

    def __init__(self, L):
        self.L = L; self.h = L.hmc_new()
        self.br = L.hmc_block_rows(); self.bb = L.hmc_block_bytes()

    def close(self):
        self.L.hmc_free(self.h)

    def entries(self):
        buf = (C.c_longlong * (6 * 4096))()
        n = self.L.hmc_entries(self.h, buf, 4096)
        assert n <= 4096
        e = np.frombuffer(buf, np.int64)[:6 * n].reshape(n, 6)
        return [(int(h), int(r), int(b), int(x) & (2 ** 64 - 1), int(r0), int(b0)) for h, r, b, x, r0, b0 in e]

    def call(self, q, nq, hq, t, nt, ht, desc_bytes, keep=True):
        """-> None when the call returns before the arena, else a dict of the state after it."""
        out = (C.c_longlong * 14)()
        if self.L.hmc_call(self.h, q, nq, hq, t, nt, ht, desc_bytes, int(keep), out):
            return None
        k = ("flushed", "q", "t", "width", "rows_cap", "rows_used", "blk_cap", "blk_used", "desc_cap", "exp_cap", "hits", "misses",
             "desc_req", "exp_req")
        return dict(zip(k, list(out)))

    def check(self, s):
        """The capacity rule, and every resident image inside both buffers, packed from row 0 without overlap."""
        w = s["width"]
        assert s["q"] != REFUSED and s["t"] != REFUSED, s
        assert s["rows_cap"] * w + 16 <= s["desc_cap"], s
        assert s["blk_cap"] * self.bb <= s["exp_cap"], s
        assert s["rows_used"] <= s["rows_cap"] and s["blk_used"] <= s["blk_cap"], s
        row, blk = 0, 0
        for host, rows, db, _, row0, blk0 in self.entries():
            nblk = -(-rows // self.br) if w == 32 else 0
            assert _width(db) == w and row0 == row and blk0 == blk, (host, rows, db, row0, blk0, s)
            row += rows; blk += nblk
            assert row * w <= s["desc_cap"] and blk * self.bb <= s["exp_cap"], (host, rows, row, blk, s)
        assert (row, blk) == (s["rows_used"], s["blk_used"]), s

    def resident(self, host, rows, db, h):
        return any(e[:4] == (host, rows, db, h) for e in self.entries())


@pytest.fixture
def arena(hm):
    a = Arena(hm)
    yield a
    a.close()


def test_32_then_64_bytes_on_9000_row_images(arena):
    """One 32-byte call sizes the buffer for 131 072 rows of 32 bytes, 81 924 rows of 64.  Then 64-byte calls on consecutive pairs
    of 9000-row images each add one new image: the arena must flush before its rows pass the buffer, not at 131 072 rows."""
    s = arena.call(1, 300, 11, 2, 280, 12, 32)
    arena.check(s)
    assert s["rows_cap"] == 131072 and s["desc_cap"] == 5243156
    flushes = 0
    for i in range(1, 15):
        s = arena.call(100 + i, 9000, i, 100 + i - 1, 9000, i - 1, 64)
        arena.check(s)
        assert s["t"] == (MISS if i == 1 or s["flushed"] else HIT), (i, s)
        flushes += s["flushed"] and i > 1
    assert flushes >= 1 and s["rows_cap"] * 64 + 16 <= s["desc_cap"]


def test_16_then_128_bytes(arena):
    """A buffer sized by a 16-byte call (2.6 MB) holds 20 482 rows of 128 bytes, not 131 072."""
    arena.check(arena.call(1, 300, 1, 2, 280, 2, 16))
    for i in range(1, 4):
        s = arena.call(10 + i, 11000, i, 10 + i - 1, 11000, i - 1, 128)
        arena.check(s)
    assert s["desc_cap"] >= s["rows_used"] * 128 >= 2 * 11000 * 128


def test_16_bytes_grown_in_place_then_32(arena):
    """A 32-byte call, then a 16-byte pair of more rows than 32-byte rows fit in the buffer, placed without enlarging it, then
    32-byte images."""
    s = arena.call(1, 300, 1, 2, 280, 2, 32)
    arena.check(s)
    cap = s["desc_cap"]
    s = arena.call(3, 150000, 3, 4, 150000, 4, 16)
    arena.check(s)
    assert s["desc_cap"] == cap and s["rows_used"] * 32 > cap
    for i in range(1, 12):
        arena.check(arena.call(10 + i, 9000, i, 10 + i - 1, 9000, i - 1, 32))


def test_every_width_switch(arena):
    """32 -> 64 -> 128 -> 16 -> 61 -> 32, enough rows at each width to pass the previous width's capacity."""
    k = 0
    for db, rows, calls in ((32, 300, 1), (64, 9000, 14), (128, 11000, 3), (16, 40000, 6), (61, 20000, 8), (32, 9000, 20)):
        for _ in range(calls):
            k += 1
            arena.check(arena.call(k, rows, k, k - 1, rows, k - 1, db))


def test_repeated_image_is_a_hit_and_changed_content_a_miss(arena):
    s = arena.call(1, 900, 7, 2, 800, 8, 32)
    assert (s["q"], s["t"]) == (MISS, MISS)
    s = arena.call(1, 900, 7, 2, 800, 8, 32)
    assert (s["q"], s["t"], s["flushed"], s["desc_req"], s["exp_req"]) == (HIT, HIT, 0, 0, 0)
    s = arena.call(2, 800, 8, 1, 900, 99, 32)                                  # buffer 1 reused with new content
    assert (s["q"], s["t"]) == (HIT, MISS)
    s = arena.call(1, 500, 99, 1, 900, 99, 32)                                 # a prefix view of the same buffer is another image
    assert (s["q"], s["t"]) == (MISS, HIT)
    s = arena.call(3, 700, 5, 3, 700, 5, 32)                                   # q is t: placed once
    assert (s["q"], s["t"]) == (MISS, HIT) and s["rows_used"] == 900 + 800 + 900 + 500 + 700
    arena.check(s)
    s = arena.call(3, 700, 5, 3, 700, 5, 61)                                   # same rows at another width: a miss
    assert (s["q"], s["t"], s["flushed"]) == (MISS, HIT, 1)
    s = arena.call(3, 700, 5, 3, 700, 5, 61, keep=False)                       # the arena switched off: every call starts empty
    assert (s["q"], s["t"], s["flushed"], s["rows_used"]) == (MISS, HIT, 1, 700)
    arena.check(s)


def test_guard_refuses_a_placement_past_the_buffer(arena):
    """A plan that overstated the row capacity is caught before any copy: the arena is reset and the next call plans afresh."""
    arena.check(arena.call(1, 300, 1, 2, 280, 2, 64))
    arena.L.hmc_set_rows_cap(arena.h, 10 ** 7)
    s = arena.call(3, 90000, 3, 4, 90000, 4, 64)
    assert s["q"] == MISS and s["t"] == REFUSED and arena.entries() == []
    s = arena.call(3, 90000, 3, 4, 90000, 4, 64)
    arena.check(s)
    assert (s["q"], s["t"]) == (MISS, MISS)


@pytest.mark.parametrize("seed", range(12))
def test_random_call_sequences(arena, seed):
    """Widths 1..128 bytes, 0..20 000 rows, reused buffers with new content, prefix views, q is t and the arena switched off."""
    rs = np.random.RandomState(seed)
    size = {b: int(rs.randint(0, 20001)) for b in range(1, 13)}               # host buffer -> its rows
    content = {b: int(rs.randint(1, 2 ** 62)) for b in size}
    widths = [int(x) for x in rs.randint(1, 129, 4)] + [32, 61]
    db = int(rs.choice(widths))
    for _ in range(160):
        if rs.rand() < 0.15:
            db = int(rs.choice(widths)) if rs.rand() < 0.7 else int(rs.randint(1, 129))
        if rs.rand() < 0.1:                                                    # the caller refills a buffer
            b = int(rs.randint(1, 13)); content[b] = int(rs.randint(1, 2 ** 62))
            if rs.rand() < 0.3:
                size[b] = int(rs.randint(0, 20001))
        q = int(rs.randint(1, 13)); t = q if rs.rand() < 0.15 else int(rs.randint(1, 13))
        nq, nt = size[q], size[t]
        if rs.rand() < 0.2:
            nq = int(rs.randint(0, nq + 1))                                    # a prefix view: same pointer, fewer rows
        hq = content[q] ^ nq; ht = content[t] ^ nt                             # the hash covers exactly the rows passed
        keep = rs.rand() > 0.08
        before = arena.entries()
        width_before = before and _width(before[0][2])
        s = arena.call(q, nq, hq, t, nt, ht, db, keep)
        if s is None:
            assert nq == 0 or nt < 2
            continue
        arena.check(s)
        was = lambda h, n, x: any(e[:4] == (h, n, db, x) for e in before)
        reuse = keep and width_before == _width(db)
        if was(q, nq, hq) and (q, nq, hq) == (t, nt, ht) or was(q, nq, hq) and was(t, nt, ht):
            if reuse:                                                          # nothing to place: no flush, no growth, two hits
                assert (s["q"], s["t"], s["flushed"], s["desc_req"], s["exp_req"]) == (HIT, HIT, 0, 0, 0), s
        if not was(q, nq, hq) or not reuse:
            assert s["q"] == MISS, s
        if not s["flushed"] and was(q, nq, hq):
            assert s["q"] == HIT, s
        if (t, nt, ht) == (q, nq, hq):
            assert s["t"] == HIT, s
        assert arena.resident(q, nq, db, hq) and arena.resident(t, nt, db, ht)
