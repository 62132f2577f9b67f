"""Descriptor matching off its common path, every result compared exactly with the oracle (oracle/match_oracle.c):
  * the per-call matcher's resident-image arena across descriptor-width switches (32 -> 64 -> 128 -> 16 -> 61 -> 32), prefix views,
    q is t, refilled buffers and SFMB200_MATCH_CACHE=0;
  * eight host threads on one context (Hamming at two widths and L2 interleaved) beside a thread running a descriptor set;
  * pair batches over images of 0, 1, 2 and 127..383 rows: self, repeated and reversed pairs, pairs without query rows or with fewer
    than two train rows, on every kernel (wgmma and XOR/POPC Hamming, 64 and 61 bytes, L2 at dims 128 and 100);
  * ties at a nonzero distance at every boundary where the wgmma kernel merges candidates: lanes, column halves, tiles and splits;
  * L2 at its value extremes (rows of 0 and 255) on the tensor cores, and the fp32 SIMT kernel at dims above 128;
  * sfmb200_match_pairs_device: the dense survivors, d_pair_start and *d_total against sfmb200_match_pairs."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from sfm_toy_library_b200 import capi

pytestmark = pytest.mark.gpu
RATIO = capi.RATIO_REFERENCE


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _same(got, ref):
    for x, y in zip(got, ref):
        np.testing.assert_array_equal(x, y)


def _hamming_images(seed, sizes, nbytes=32, world=6000):
    """Half of each image's rows are rows of a shared `world` with up to 4 bits flipped, so every pair has matches (and exact
    duplicates, i.e. ties); the rest are random."""
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (world, nbytes), dtype=np.uint8)
    out = []
    for n in sizes:
        d = rs.randint(0, 256, (n, nbytes), dtype=np.uint8)
        k = np.flatnonzero(rs.rand(n) < 0.5)
        rows = base[rs.randint(0, world, len(k))]
        for bit in rs.randint(0, nbytes * 8, (4, len(k))):
            rows[np.arange(len(k)), bit >> 3] ^= (1 << (bit & 7)).astype(np.uint8)
        d[k] = rows
        out.append(d)
    return out


def _sift_images(seed, sizes, dim=128, world=3000):
    """Integer-valued float rows in [0, 255] (SIFT-like); half of each image's rows are rows of a shared `world` moved by +-3."""
    rs = np.random.RandomState(seed)
    base = np.minimum(rs.exponential(25.0, (world, dim)), 255).astype(np.int32)
    out = []
    for n in sizes:
        d = np.minimum(rs.exponential(25.0, (n, dim)), 255).astype(np.int32)
        k = np.flatnonzero(rs.rand(n) < 0.5)
        d[k] = np.clip(base[rs.randint(0, world, len(k))] + rs.randint(-3, 4, (len(k), dim)), 0, 255)
        out.append(d.astype(np.float32))
    return out


# ---------------------------------------------------------------------------------------------------------- resident-image arena
def _chain(ctx, oracle, imgs, head=200):
    """Match the first `head` rows of image i (a prefix view) against image i-1: each call places all of image i-1, which the
    arena has not seen, while the oracle's work stays small."""
    for i in range(1, len(imgs)):
        _same(ctx.match_knn2_ratio(imgs[i][:head], imgs[i - 1]), oracle.match_hamming(imgs[i][:head], imgs[i - 1]))


def test_arena_width_switches_32_64_128_16_61_32(oracle):
    """A 32-byte call sizes the arena's buffer for 131 072 rows of 32 bytes; 14 x 9200 new rows of 64 bytes follow, more than
    the 81 924 that buffer holds at 64 bytes.  Then 128, 16, 61 and 32 bytes again, each phase placing more rows than the buffer
    holds at its width when it starts, so each flushes and regrows.  A fresh context: the arena only grows, so on a shared one an
    earlier test would already have enlarged it."""
    c = capi.Context(0)
    try:
        for k, (nbytes, rows, n) in enumerate(((32, 300, 2), (64, 9000, 15), (128, 11000, 9), (16, 40000, 35), (61, 20000, 18),
                                               (32, 9000, 75))):
            _chain(c, oracle, _hamming_images(300 + k, [rows] * n, nbytes))
    finally:
        c.close()


def test_arena_16_then_128_bytes(oracle):
    """A buffer sized by a 16-byte call holds 20 482 rows of 128 bytes; 3 x 11 000 rows of 128 bytes follow."""
    c = capi.Context(0)
    try:
        _chain(c, oracle, _hamming_images(310, [300, 280], 16))
        _chain(c, oracle, _hamming_images(311, [11000] * 4, 128))
    finally:
        c.close()


def test_arena_views_self_refill_and_off(ctx, oracle, monkeypatch):
    a, b = _hamming_images(320, [3000, 2500])
    a0 = a.copy()
    calls = [(a[:1000], a), (a, a[:1500]), (a, a), (b, a), (a[:1000], b), (a, b)]     # prefix views share a's pointer
    on = [ctx.match_knn2_ratio(q, t) for q, t in calls]
    for (q, t), got in zip(calls, on):
        _same(got, oracle.match_hamming(q, t))
    _same(ctx.match_knn2_ratio(a, a), on[2])                                           # resident now
    _chain(ctx, oracle, _hamming_images(321, [9000] * 16))                             # 138 k new rows: flushes the arena
    a[:] = _hamming_images(322, [3000])[0]                                             # the caller refills a's buffer
    _same(ctx.match_knn2_ratio(b, a), oracle.match_hamming(b, a))
    _same(ctx.match_knn2_ratio(a[:1000], a), oracle.match_hamming(a[:1000], a))
    monkeypatch.setenv("SFMB200_MATCH_CACHE", "0")
    for q, t in calls:
        _same(ctx.match_knn2_ratio(q, t), oracle.match_hamming(q, t))
    a[:] = a0
    for (q, t), ref in zip(calls, on):
        _same(ctx.match_knn2_ratio(q, t), ref)                                         # the arena switched off: the same results


# ------------------------------------------------------------------------------------------------------------------------ threads
def test_threads_share_one_context(ctx, oracle):
    """Eight threads match all ordered pairs of eight images through the per-call paths, 32- and 64-byte Hamming and L2 in an
    order that differs per thread, so the arena switches width under contention; a ninth runs a descriptor set meanwhile."""
    h32 = _hamming_images(400, [1500 + 97 * i for i in range(8)], 32)
    h64 = _hamming_images(401, [1200 + 53 * i for i in range(8)], 64)
    l2 = _sift_images(402, [300 + 31 * i for i in range(8)])
    imgs = {"h32": h32, "h64": h64, "l2": l2}
    pairs = [(i, j) for i in range(8) for j in range(8) if i != j]
    ref = {(kind, i, j): (oracle.match_l2 if kind == "l2" else oracle.match_hamming)(imgs[kind][i], imgs[kind][j])
           for kind in imgs for i, j in pairs}
    sd = _hamming_images(403, [2000, 1800, 2200, 1900])
    sd_pairs = [(i, j) for i in range(4) for j in range(4) if i != j]
    sd_ref = [oracle.match_hamming(sd[i], sd[j]) for i, j in sd_pairs]
    ds = ctx.descriptor_set(sd)

    def worker(k):
        out = {}
        for n, (i, j) in enumerate(pairs[k::8]):
            for kind in (("h32", "l2", "h64"), ("h64", "h32", "l2"), ("l2", "h64", "h32"))[(k + n) % 3]:
                f = ctx.match_knn2_ratio_l2 if kind == "l2" else ctx.match_knn2_ratio
                out[(kind, i, j)] = f(imgs[kind][i], imgs[kind][j])
        return out

    def set_worker():
        return [[tuple(np.copy(x) for x in r) for r in ds.match_pairs(sd_pairs)] for _ in range(6)]

    with ThreadPoolExecutor(9) as ex:
        futs = [ex.submit(worker, k) for k in range(8)]
        sfut = ex.submit(set_worker)
        got = {}
        for f in futs:
            got.update(f.result())
        runs = sfut.result()
    ds.close()
    assert got.keys() == ref.keys()
    for key in ref:
        _same(got[key], ref[key])
    for run in runs:
        for r, e in zip(run, sd_ref):
            _same(r, e)


# --------------------------------------------------------------------------------------------------------- degenerate pair batches
SIZES = [0, 1, 2, 127, 128, 129, 255, 256, 257, 383, 5000]
_DEGEN = {}


def _degenerate(oracle, kind, width):
    """Images of SIZES rows; every ordered pair (self pairs included) in a seeded shuffle, then a repeated pair and a pair without
    query rows last.  Returns (images, pairs, oracle result per pair)."""
    key = (kind, width)
    if key not in _DEGEN:
        imgs = _sift_images(500, SIZES, width) if kind == "l2" else _hamming_images(501 + width, SIZES, width)
        pairs = [(i, j) for i in range(len(SIZES)) for j in range(len(SIZES))]
        pairs = [pairs[k] for k in np.random.RandomState(502).permutation(len(pairs))] + [(4, 9), (4, 9), (10, 3), (0, 10)]
        f = oracle.match_l2 if kind == "l2" else oracle.match_hamming
        memo = {}
        for p in pairs:
            if p not in memo:
                memo[p] = f(imgs[p[0]], imgs[p[1]])
        _DEGEN[key] = (imgs, pairs, [memo[p] for p in pairs])
    return _DEGEN[key]


@pytest.mark.parametrize("kind,width,mode", [("hamming", 32, None), ("hamming", 32, "popc"), ("hamming", 64, None), ("hamming", 61, None),
                                             ("l2", 128, None), ("l2", 100, None)])
def test_degenerate_pair_batch(ctx, oracle, monkeypatch, kind, width, mode):
    if mode:
        monkeypatch.setenv("SFMB200_MATCH", mode)
    imgs, pairs, ref = _degenerate(oracle, kind, width)
    assert sum(len(r[0]) for r in ref) > 1000
    ds = ctx.descriptor_set(imgs, norm=kind)
    try:
        got = ds.match_pairs(pairs)
        assert len(got) == len(pairs)
        for p, g, r in zip(pairs, got, ref):
            for x, y in zip(g, r):
                np.testing.assert_array_equal(x, y, err_msg=str(p))
        assert ds.match_pairs([]) == []
    finally:
        ds.close()


@pytest.mark.parametrize("kind", ["hamming", "l2"])
def test_empty_sets_and_batches(ctx, kind):
    dim = 32 if kind == "hamming" else 128
    dt = np.uint8 if kind == "hamming" else np.float32
    for imgs in ([], [np.zeros((0, dim), dt)] * 3):
        ds = ctx.descriptor_set(imgs, norm=kind)
        try:
            assert ds.match_pairs([]) == []
            if imgs:
                assert all(len(r[0]) == 0 for r in ds.match_pairs([(0, 1), (2, 2), (1, 0)]))
        finally:
            ds.close()


# ------------------------------------------------------------------------------------------------------------------------- ties
def _plant(q, t, groups, kind):
    """groups: {query row: [train rows]}.  Train row c-th of a group = the query row with three bits flipped (Hamming) or one
    coordinate stepped by +5 (L2), a different three bits / coordinate per copy: the same nonzero distance, never the same row."""
    for r, rows in groups.items():
        for c, j in enumerate(rows):
            row = q[r].copy()
            if kind == "hamming":
                for b in (3 * c, 3 * c + 1, 3 * c + 2):
                    row[b >> 3] ^= np.uint8(1 << (b & 7))
            else:
                row[c] += 5
            t[j] = row


def _tie_data(kind, nq, nt, groups, seed):
    rs = np.random.RandomState(seed)
    if kind == "hamming":
        q = rs.randint(0, 256, (nq, 32), dtype=np.uint8); t = rs.randint(0, 256, (nt, 32), dtype=np.uint8)
    else:                                                   # queries in [20, 230]: a +5 step stays an integer in [0, 255]
        q = rs.randint(20, 231, (nq, 128)).astype(np.float32); t = rs.randint(0, 256, (nt, 128)).astype(np.float32)
    _plant(q, t, groups, kind)
    return q, t


def _check_ties(ctx, oracle, q, t, groups, kind):
    match = ctx.match_knn2_ratio_l2 if kind == "l2" else ctx.match_knn2_ratio
    ref = oracle.match_l2 if kind == "l2" else oracle.match_hamming
    dist = 5.0 if kind == "l2" else 3.0
    loose = match(q, t, 1.5)
    _same(loose, ref(q, t, 1.5))
    where = dict(zip(loose[0].tolist(), zip(loose[1].tolist(), loose[2].tolist())))
    for r, rows in groups.items():
        assert where[r] == (min(rows), dist), (r, rows, where.get(r))       # the tied pair is the top 2: the lower index wins
    strict = match(q, t)
    _same(strict, ref(q, t))
    assert not set(groups) & set(strict[0].tolist())                         # d0 == d1: dropped at the reference ratio


SMALL_TIES = {0: [0, 2], 7: [257, 258], 31: [8, 40], 63: [5, 6], 64: [127, 128], 127: [255, 256], 128: [130, 380], 20: [129, 260],
              191: [200, 1000], 255: [1151, 1152], 256: [1222, 1223], 299: [3, 700, 1100], 150: [1023, 1024], 100: [10, 266],
              200: [140, 396]}


@pytest.mark.parametrize("kind,mode", [("hamming", None), ("hamming", "popc"), ("l2", None), ("l2", "simt")])
def test_ties_inside_and_across_tiles(ctx, oracle, monkeypatch, kind, mode):
    """Columns 0/2, 257/258 and 5/6 (neighbouring lanes), 8/40 (one thread, two column groups), 127/128 (column halves),
    255/256 and 1023/1024 (tiles), 10/266 and 140/396 (one column half of two tiles), 130/380 and 129/260 (different halves of
    different tiles), 200/1000 (the two splits of the 5-tile image), 1151/1152 and 1222/1223 in the partial last tile of a
    1224-row image, and a three-way tie; the query rows spread over both 64-row halves and both 128-row tiles of the query."""
    if mode:
        monkeypatch.setenv("SFMB200_MATCH" if kind == "hamming" else "SFMB200_MATCH_L2", mode)
    q, t = _tie_data(kind, 300, 1224, SMALL_TIES, 600)
    _check_ties(ctx, oracle, q, t, SMALL_TIES, kind)


@pytest.mark.parametrize("kind,mode", [("hamming", None), ("hamming", "popc"), ("l2", None), ("l2", "simt")])
def test_ties_at_every_tile_boundary_of_70000_rows(ctx, oracle, monkeypatch, kind, mode):
    """Train rows 256m-1 and 256m for every m, query row (m-1) % 100: the split count follows the SM count, so some pair straddles
    whatever split boundary is chosen.  A query's lowest pair must win over its copies at later tiles and splits."""
    if mode:
        monkeypatch.setenv("SFMB200_MATCH" if kind == "hamming" else "SFMB200_MATCH_L2", mode)
    groups = {}
    for m in range(1, 70000 // 256 + 1):
        groups.setdefault((m - 1) % 100, []).extend([256 * m - 1, 256 * m])
    q, t = _tie_data(kind, 100, 70000, groups, 601)
    _check_ties(ctx, oracle, q, t, groups, kind)


# ------------------------------------------------------------------------------------------------------------------- L2 extremes
def _extreme_rows(rs, n, dim):
    """A quarter each: all 255, all 0, random 0/255 mixes, random integers; every squared distance is below 2^24 for dim <= 256."""
    kind = rs.randint(0, 4, n)
    x = rs.randint(0, 256, (n, dim)).astype(np.float32)
    x[kind == 0] = 255; x[kind == 1] = 0
    x[kind == 2] = 255 * rs.randint(0, 2, (int((kind == 2).sum()), dim))
    return x


@pytest.mark.parametrize("dim", [1, 16, 17, 127, 128, 129, 200, 256])
def test_l2_extremes(ctx, oracle, dim):
    """dim <= 128: the u8 GEMM on the tensor cores (|a|^2 up to 128 * 255^2, its packed key 2^31 - 1.7e7 away from overflow);
    dim > 128: the fp32 SIMT kernel, its only path.  64 query rows against 4096 train rows, so the kernel splits."""
    rs = np.random.RandomState(700 + dim)
    t = _extreme_rows(rs, 4096, dim); q = _extreme_rows(rs, 64, dim)
    q[::5] = t[rs.randint(0, 4096, len(q[::5]))]
    for ratio in (RATIO, 2.0):
        _same(ctx.match_knn2_ratio_l2(q, t, ratio), oracle.match_l2(q, t, ratio))


# ------------------------------------------------------------------------------------------------------ match_pairs_device
def _device_run(ctx, ds, pairs, rows):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    n, P = max(rows, 1), len(pairs)
    d_q = torch.full((n,), -5, dtype=torch.int32, device=dev); d_t = torch.full((n,), -5, dtype=torch.int32, device=dev)
    d_d = torch.full((n,), -5.0, dtype=torch.float32, device=dev)
    d_start = torch.full((P + 1,), -7, dtype=torch.int32, device=dev); d_total = torch.full((1,), -9, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()                                        # the fills ran on torch's stream, the matcher runs on the context's
    ds.match_pairs_device(pairs, d_q.data_ptr(), d_t.data_ptr(), d_d.data_ptr(), d_start.data_ptr(), d_total.data_ptr())
    ctx.synchronize()
    total = int(d_total.cpu()[0])
    return total, d_q.cpu().numpy()[:max(total, 0)], d_t.cpu().numpy()[:max(total, 0)], d_d.cpu().numpy()[:max(total, 0)], \
        d_start.cpu().numpy()[:P]


def _check_device(ctx, ds, sizes, pairs):
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2)
    host = ds.match_pairs(pairs)
    total, q, t, d, start = _device_run(ctx, ds, pairs, int(sum(sizes[l] for l, _ in pairs)))
    counts = np.array([len(r[0]) for r in host], np.int64)
    assert total == counts.sum() and total != -1
    cat = lambda k, dt: np.concatenate([r[k] for r in host]) if len(host) else np.zeros(0, dt)
    np.testing.assert_array_equal(q, cat(0, np.int32)); np.testing.assert_array_equal(t, cat(1, np.int32))
    np.testing.assert_array_equal(d, cat(2, np.float32))
    excl = np.concatenate([[0], np.cumsum(counts)[:-1]]) if len(counts) else counts
    want = np.where([sizes[l] > 0 for l, _ in pairs], excl, 0) if len(counts) else counts
    np.testing.assert_array_equal(start, want)
    return total


@pytest.mark.parametrize("kind,width", [("hamming", 32), ("hamming", 61), ("l2", 128)])
def test_match_pairs_device(ctx, oracle, kind, width):
    imgs, pairs, ref = _degenerate(oracle, kind, width)
    ds = ctx.descriptor_set(imgs, norm=kind)
    try:
        assert _check_device(ctx, ds, SIZES, pairs) == sum(len(r[0]) for r in ref) > 1000
        assert _check_device(ctx, ds, SIZES, [(3, 10), (10, 10)]) > 0                    # a short batch after a long one
        assert _check_device(ctx, ds, SIZES, [(3, 0), (4, 1)]) == 0                      # no train image of 2 rows: no launch
        assert _check_device(ctx, ds, SIZES, [(3, 0), (0, 7), (4, 1)]) == 0              # the kernels run, nothing survives
        assert _check_device(ctx, ds, SIZES, [(0, 0), (0, 9)]) == 0                      # no query rows at all
        assert _check_device(ctx, ds, SIZES, []) == 0                                    # n_pairs == 0
    finally:
        ds.close()
    empty = ctx.descriptor_set([], norm=kind)
    try:
        assert _check_device(ctx, empty, [], []) == 0
    finally:
        empty.close()
