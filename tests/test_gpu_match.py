"""GPU parity: sfmb200_match_* (CUDA, through the C ABI) vs the oracle restatement of matchFeatures
(SfM2DFeatureUtilities.cpp:53-71) and the cv2 golden vectors.  Integer path -> bit-exact indices AND distances."""
import numpy as np
import pytest

from sfm_toy_library_b200 import capi, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("case", ["a", "b", "c", "d", "e"])
def test_golden_cv2(ctx, golden, case):
    g = golden("match_cv2.npz")
    _same(ctx.match_knn2_ratio(g[f"{case}_q"], g[f"{case}_t"]), (g[f"{case}_mq"], g[f"{case}_mt"], g[f"{case}_md"]))


def test_ratio_constant(ctx, golden):
    g = golden("match_cv2.npz")
    assert len(ctx.match_knn2_ratio(g["c_q"], g["c_t"])[0]) == 1            # (double)0.8f keeps d0=4, d1=5
    assert len(ctx.match_knn2_ratio(g["c_q"], g["c_t"], ratio=0.8)[0]) == 0


@pytest.mark.parametrize("nq,nt", [(1, 2), (255, 257), (256, 128), (1000, 3), (5000, 5000), (4999, 5003), (37, 9000)])
def test_vs_oracle_ragged_sizes(ctx, oracle, nq, nt):
    t = synth.make_descriptors(nt % 97, nt); q = synth.make_descriptors(nq % 89 + 100, nq, prev=t)
    _same(ctx.match_knn2_ratio(q, t), oracle.match_hamming(q, t))


def test_edge_cases(ctx):
    d = synth.make_descriptors(0, 10)
    assert len(ctx.match_knn2_ratio(d, d[:1])[0]) == 0                      # nt < 2 (UB in the reference) -> empty
    assert len(ctx.match_knn2_ratio(d[:0], d)[0]) == 0                      # empty query
    q, t, dist = ctx.match_knn2_ratio(d, d)                                 # d0 = 0: kept iff 0 < 0.8f*d1, i.e. d1 > 0
    assert np.all(dist == 0) and np.array_equal(q, t)


def test_all_ties_go_to_lowest_train_index(ctx, oracle):
    t = np.repeat(synth.make_descriptors(5, 8), 40, axis=0)                 # every row 40 times
    q = synth.make_descriptors(6, 50)
    q[:8] = t[::40]
    _same(ctx.match_knn2_ratio(q, t, ratio=2.0), oracle.match_hamming(q, t, ratio=2.0))


def test_64_byte_descriptors(ctx, oracle):
    a = synth.make_descriptors(9, 700, nbytes=64); b = synth.make_descriptors(10, 650, nbytes=64, prev=a)
    _same(ctx.match_knn2_ratio(b, a), oracle.match_hamming(b, a))


def test_all_pairs_batched_equals_pairwise(ctx, oracle):
    descs = synth.make_descriptor_set(5, n=1200)
    descs[3] = descs[3][:700]                                                # ragged image sizes
    pairs = [(i, j) for i in range(5) for j in range(i + 1, 5)]              # SfM::createFeatureMatchMatrix (SfM.cpp:166-172)
    ds = ctx.descriptor_set(descs)
    res = ds.match_pairs(pairs)
    for (i, j), r in zip(pairs, res):
        _same(r, oracle.match_hamming(descs[i], descs[j]))
        assert len(r[0]) > (30 if j == i + 1 else 0)
    ds.close()


def test_l2_sift_like(ctx, oracle, golden):
    g = golden("match_cv2.npz")
    _same(ctx.match_knn2_ratio_l2(g["l2_q"], g["l2_t"]), (g["l2_mq"], g["l2_mt"], g["l2_md"]))
    a = synth.make_sift_like(3, 900); b = synth.make_sift_like(4, 800, prev=a)
    _same(ctx.match_knn2_ratio_l2(b, a), oracle.match_l2(b, a))


def test_config4_properties_full_size(ctx):
    """BASELINE.json config 4 sizes (5000 x 5000 per pair): size-independent properties instead of the O(n^2) oracle:
    planted near-duplicates are recovered, output is sorted by queryIdx, distances are integers in [0, 256]."""
    a = synth.make_descriptors(20, 5000); b = synth.make_descriptors(21, 5000, prev=a)
    q, t, d = ctx.match_knn2_ratio(b, a)
    assert np.all(np.diff(q) > 0) and np.all(d == np.round(d)) and d.min() >= 0 and d.max() <= 256
    x = np.unpackbits(b[q] ^ a[t], axis=1).sum(1)
    np.testing.assert_array_equal(x.astype(np.float32), d)                   # reported distance is the true Hamming distance
    assert 0.15 * 5000 < len(q) < 0.3 * 5000


@pytest.mark.parametrize("nq,nt", [(255, 257), (5000, 5000), (130, 9000), (4999, 513)])
def test_popc_and_tensor_core_paths_are_bit_identical(ctx, oracle, monkeypatch, nq, nt):
    """32-byte descriptors default to the wgmma integer-GEMM kernel (match_tc.cu); SFMB200_MATCH=popc forces the
    XOR/POPC kernel.  Both must reproduce the oracle exactly (indices, distances, tie-breaks)."""
    t = synth.make_descriptors(nt % 91, nt); q = synth.make_descriptors(nq % 83 + 200, nq, prev=t)
    t[5:9] = t[4]                                                            # duplicate train rows: tie-break inside one MMA tile
    ref = oracle.match_hamming(q, t)
    monkeypatch.setenv("SFMB200_MATCH", "popc")
    _same(ctx.match_knn2_ratio(q, t), ref)
    monkeypatch.setenv("SFMB200_MATCH", "tc")
    _same(ctx.match_knn2_ratio(q, t), ref)


@pytest.mark.parametrize("nbytes", [61, 20, 100, 128, 16])
def test_any_descriptor_width_up_to_128_bytes(ctx, oracle, nbytes):
    """The reference accepts any cv::Mat width (AKAZE: 61 bytes); widths between the instantiated kernels are zero-padded."""
    rng = np.random.RandomState(nbytes)
    a = rng.randint(0, 256, (300, nbytes)).astype(np.uint8); b = rng.randint(0, 256, (280, nbytes)).astype(np.uint8)
    b[::3] = a[rng.randint(0, 300, len(b[::3]))]
    b[::3, 0] ^= 5
    _same(ctx.match_knn2_ratio(b, a), oracle.match_hamming(b, a))
    ds = ctx.descriptor_set([a, b])
    _same(ds.match_pairs([(1, 0)])[0], oracle.match_hamming(b, a))
    ds.close()


def test_resident_image_cache_detects_reused_buffers(ctx, oracle):
    """Per-call path keeps uploaded images resident, keyed by (pointer, rows, width, content hash): same buffer + same
    content = hit; same buffer + new content must be re-uploaded."""
    a = synth.make_descriptors(20, 900); b = synth.make_descriptors(21, 800, prev=a)
    r1 = ctx.match_knn2_ratio(b, a)
    r2 = ctx.match_knn2_ratio(b, a)                      # both images resident now
    _same(r1, r2); _same(r1, oracle.match_hamming(b, a))
    c = synth.make_descriptors(22, 900)
    a[:] = c                                             # caller reuses the buffer
    _same(ctx.match_knn2_ratio(b, a), oracle.match_hamming(b, a))
    _same(ctx.match_knn2_ratio(a, a), oracle.match_hamming(a, a))


def test_cache_flush_when_arena_is_full(ctx, oracle):
    imgs = [synth.make_descriptors(100 + i, 9000) for i in range(20)]     # 180 k rows > the 128 k row arena
    for i in range(1, 20):
        _same(ctx.match_knn2_ratio(imgs[i][:700], imgs[i - 1]), oracle.match_hamming(imgs[i][:700], imgs[i - 1]))


@pytest.mark.parametrize("nq,nt,dim", [(1, 2, 128), (300, 257, 128), (2000, 2100, 128), (5000, 5000, 128), (700, 650, 64), (129, 1000, 100)])
def test_l2_exact_u8_gemm_vs_oracle(ctx, oracle, nq, nt, dim):
    """SIFT-like (integer-valued) descriptors: the wgmma u8 x u8 -> s32 GEMM path (|a-b|^2 = |a|^2 + |b|^2 - 2<a,b>, exact)
    gives the indices AND float distances of cv::BFMatcher(NORM_L2) (= the oracle's float loop, pinned to cv2 by the golden)."""
    t = synth.make_sift_like(nt % 50, nt, dim=dim); q = synth.make_sift_like(nq % 40 + 60, nq, dim=dim, prev=t)
    q[::7] = t[np.arange(len(q[::7])) % nt]                                   # exact duplicates: distance 0 and ties
    _same(ctx.match_knn2_ratio_l2(q, t), oracle.match_l2(q, t))
    _same(ctx.match_knn2_ratio_l2(q, t, ratio=2.0), oracle.match_l2(q, t, ratio=2.0))    # every row survives: all 2-NN distances checked


def test_l2_batched_all_pairs_and_simt_fallback(ctx, oracle, monkeypatch):
    imgs = [synth.make_sift_like(i, 900 + 37 * i, prev=None if i == 0 else None) for i in range(4)]
    for i in range(1, 4):
        imgs[i][::5] = imgs[i - 1][:len(imgs[i][::5])]
    ds = ctx.descriptor_set(imgs, norm="l2")
    pairs = [(i, j) for i in range(4) for j in range(i + 1, 4)]
    for (i, j), got in zip(pairs, ds.match_pairs(pairs)):
        _same(got, oracle.match_l2(imgs[i], imgs[j]))
    ds.close()
    # non-integer descriptors cannot use the exact GEMM: the set is refused, the per-pair call falls back to the fp32 SIMT kernel
    a = imgs[0][:300] + 0.25; b = imgs[1][:280] * 0.5
    with pytest.raises(capi.SfmB200Error):
        ctx.descriptor_set([a, b], norm="l2")
    q, t, d = ctx.match_knn2_ratio_l2(b, a, ratio=2.0)
    oq, ot, od = oracle.match_l2(b, a, ratio=2.0)
    np.testing.assert_array_equal(q, oq); np.testing.assert_array_equal(t, ot); np.testing.assert_allclose(d, od, rtol=1e-6)
    monkeypatch.setenv("SFMB200_MATCH_L2", "simt")                             # the SIMT kernel on integer data: same answer
    _same(ctx.match_knn2_ratio_l2(imgs[1], imgs[0]), oracle.match_l2(imgs[1], imgs[0]))


def test_l2_real_sift_golden(ctx, golden):
    """Real SIFT descriptors (cv2.SIFT_create on two crazyhorse images, tests/golden/make_cfg1.py) vs cv2.BFMatcher(NORM_L2)."""
    g = golden("sift_crazyhorse.npz")
    _same(ctx.match_knn2_ratio_l2(g["q"], g["t"]), (g["mq"], g["mt"], g["md"]))
    _same(ctx.match_knn2_ratio_l2(g["t"], g["q"]), (g["rq"], g["rt"], g["rd"]))


def test_hamming_many_tiles_per_split(ctx, oracle):
    """One query block against 70 000 train rows: the packed-key epilogue's 16-bit index field (<= 256 tiles per split)."""
    t = synth.make_descriptors(3, 70000); q = synth.make_descriptors(4, 100, prev=t)
    _same(ctx.match_knn2_ratio(q, t), oracle.match_hamming(q, t))
