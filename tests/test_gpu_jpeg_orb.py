"""sfmb200_decode_jpeg_extract_orb on the GPU: JPEG files to ORB key points and descriptors in one call, the images staying on the device.
Per image, every result is compared BIT FOR BIT with `cv2.ORB_create(5000).detectAndCompute` on cv2's decoded (and resized) image and
with this library's two-call chain (decode_jpeg, then orb_detect_and_compute on the downloaded image): the crazyhorse file alone and
seven times over, a batch of mixed sizes (EXIF-rotated copies, grey, odd and tiny images) in any order, three scales, no image download,
a capacity below the count, a batch that spans several groups, and the refused inputs, after each of which the context still works."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_util as J

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _cv(b, scale=1.0):
    im = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    return im if scale == 1.0 else cv2.resize(im, None, fx=scale, fy=scale)


def _cv_orb(img, nf=5000):
    from oracle import orb_oracle as O
    return O.cv2_detect_and_compute(img, nf)


def _same(got, want):
    (k, d), (wk, wd) = got, want
    return k.shape[0] == wk.shape[0] and np.array_equal(k[:, :6], wk) and np.all(k[:, 6] == -1) and np.array_equal(d, wd)


def _equal(a, b):
    return len(a) == len(b) and all(x[0].shape == y[0].shape and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))


@pytest.fixture(scope="module")
def mixed():
    """1023x767 as stored, with EXIF orientation 6 and 8 (767x1023 decoded), grey, odd-sized, and a tiny image with no key point."""
    return [("1023x767", J.encode(1023, 767, seed=11)), ("orient6", J.encode(1023, 767, seed=11, orientation=6)),
            ("orient8", J.encode(1023, 767, seed=11, orientation=8)), ("grey", J.encode(640, 480, grey=True, seed=12)),
            ("1001x333", J.encode(1001, 333, seed=13)), ("48x40", J.encode(48, 40, seed=14))]


def test_crazyhorse_alone_and_seven_times_equals_cv2(ctx):
    b = J.crazyhorse()
    want = _cv_orb(_cv(b))
    assert want[0].shape[0] > 1000
    imgs, feats = ctx.decode_jpeg_orb([b])
    assert np.array_equal(imgs[0], _cv(b)) and _same(feats[0], want)
    imgs, feats = ctx.decode_jpeg_orb([b] * 7)
    assert len(feats) == 7 and all(_same(f, want) for f in feats)
    assert all(np.array_equal(im, imgs[0]) for im in imgs)


def test_mixed_sizes_in_one_call(ctx, mixed):
    from oracle import orb_oracle as O
    from sfm_toy_library_b200 import capi
    blobs = [b for _, b in mixed]
    imgs, feats = ctx.decode_jpeg_orb(blobs)
    assert [im.shape[:2] for im in imgs] == [(767, 1023), (1023, 767), (1023, 767), (480, 640), (333, 1001), (40, 48)]
    for (name, b), im, f in zip(mixed, imgs, feats):
        ref = _cv(b)
        assert np.array_equal(im, ref), name
        assert _same(f, _cv_orb(ref)), name
        assert _equal([f], [ctx.orb_detect_and_compute(ref, 5000)]), name
    assert feats[-1][0].shape[0] == 0 and all(f[0].shape[0] > 500 for f in feats[:-1])
    # the inspection of the last call keeps every image's own layout
    ctx.decode_jpeg_orb(blobs, images=False)
    for i, im in enumerate(imgs):
        pyr = O.pyramid(cv2.cvtColor(im, cv2.COLOR_BGR2GRAY))
        lw, lh, _, _ = capi.orb_layout(im.shape[1], im.shape[0])
        for l in (0, 1, 5):
            assert np.array_equal(ctx.orb_download_level(0, i, l, int(lw[l]), int(lh[l])), pyr[l]), (i, l)
    # any order gives the same per-image results
    for order in ([5, 4, 3, 2, 1, 0], [2, 0, 5, 1, 4, 3]):
        _, got = ctx.decode_jpeg_orb([blobs[k] for k in order], images=False)
        for j, k in enumerate(order):
            assert _equal([got[j]], [feats[k]]), (order, k)


@pytest.mark.parametrize("scale", [0.5, 0.3, 1.0])
def test_scales_equal_cv2_resize_then_orb(ctx, mixed, scale):
    blobs = [b for _, b in mixed[:5]] + [J.crazyhorse()]
    imgs, feats = ctx.decode_jpeg_orb(blobs, scale)
    dec = ctx.decode_jpeg(blobs, scale)
    for (k, b), im, d, f in zip(enumerate(blobs), imgs, dec, feats):
        assert np.array_equal(im, d), k                         # the images decode_jpeg[_scaled] downloads, byte for byte
        ref = _cv(b, scale)
        assert np.array_equal(im, ref), k
        assert _same(f, _cv_orb(ref)), k


def test_without_image_download(ctx, mixed):
    blobs = [b for _, b in mixed]
    imgs, feats = ctx.decode_jpeg_orb(blobs, 0.5)
    with_images = ctx.jpeg_last_stats()["download_bytes"]
    none, feats2 = ctx.decode_jpeg_orb(blobs, 0.5, images=False)
    without = ctx.jpeg_last_stats()["download_bytes"]
    assert none is None and _equal(feats, feats2)
    assert with_images >= sum(im.nbytes for im in imgs)
    assert without < min(im.nbytes for im in imgs)                # the error words and statistics only
    t = ctx.orb_last_timings()
    assert t["candidates_d2h"] >= 0 and t["describe_roundtrip"] > 0


def test_capacity_and_determinism(ctx, mixed):
    from sfm_toy_library_b200 import capi
    blobs = [b for _, b in mixed]
    _, full = ctx.decode_jpeg_orb(blobs, images=False)
    n = len(blobs)
    cap = 10
    kp = np.zeros((n, cap, 7), np.float32); desc = np.zeros((n, cap, 32), np.uint8); cnt = np.zeros(n, np.int32)
    rc = capi.lib().sfmb200_decode_jpeg_extract_orb(ctx._h, (C.c_char_p * n)(*blobs), (C.c_size_t * n)(*[len(b) for b in blobs]), n,
                                                     C.c_double(1.0), 5000, cap, capi._p(kp, C.c_float), capi._p(desc, C.c_uint8),
                                                     capi._p(cnt, C.c_int32), None, None)
    assert rc == 0 and list(cnt) == [f[0].shape[0] for f in full]          # the full counts, past the capacity
    for i in range(n):
        m = min(cap, cnt[i])
        assert np.array_equal(kp[i, :m, :5], full[i][0][:m, :5]) and np.array_equal(desc[i, :m], full[i][1][:m])
    _, again = ctx.decode_jpeg_orb(blobs, capacity=10, images=False)   # the retry
    assert _equal(again, full)
    _, third = ctx.decode_jpeg_orb(blobs, images=False)
    assert _equal(third, full)


def _group_starts(sizes):
    """The groups csrc/orb_groups.h forms for images already on the device (no upload, no staging)."""
    so = os.path.join(ROOT, "tests", "_build", "libhost_orb_groups.so")
    os.makedirs(os.path.dirname(so), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-shared", "-fPIC", "-O2", "-x", "c++", os.path.join(ROOT, "tests", "host_orb_groups.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    L.hog_image_bytes.restype = C.c_longlong
    L.hog_image_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.hog_dev_budget.restype = C.c_longlong
    L.hog_stage_budget.restype = C.c_longlong
    L.hog_groups.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p]
    n = len(sizes)
    dev = (C.c_longlong * n)(*[L.hog_image_bytes(w, h, 5000, 0, None) for w, h in sizes])
    out = (C.c_int * (n + 1))()
    g = L.hog_groups(dev, None, n, L.hog_dev_budget(), L.hog_stage_budget(), L.hog_max_group(), out)
    return list(out[:g + 1])


def test_batch_over_several_groups(ctx):
    distinct = [J.encode(4032, 3024, seed=21), J.encode(4032, 3024, seed=22, orientation=6), J.encode(1023, 767, seed=23)]
    blobs = [distinct[k % 3] for k in range(36)]
    shapes = [(4032, 3024), (3024, 4032), (1023, 767)]
    starts = _group_starts([shapes[k % 3] for k in range(36)])
    assert len(starts) >= 3, starts                           # at least two groups
    _, feats = ctx.decode_jpeg_orb(blobs, images=False)
    for k, b in enumerate(distinct):
        want = _cv_orb(_cv(b))
        for i in range(k, 36, 3):
            assert _same(feats[i], want), (k, i)


def test_refused_inputs_leave_the_context_usable(ctx):
    from sfm_toy_library_b200 import capi
    good = J.encode(200, 150, seed=31)
    want = _cv_orb(_cv(good))
    refused = {name: (b, status) for name, b, status in J.refused()}

    def check_ok():
        _, f = ctx.decode_jpeg_orb([good, good], images=False)
        assert _same(f[0], want) and _same(f[1], want)

    for name in ("truncated", "undefined_code", "progressive"):
        b, status = refused[name]
        with pytest.raises(capi.SfmB200Error) as e:
            ctx.decode_jpeg_orb([good, good, b, good])
        assert f"libsfmb200 error {status}:" in str(e.value) and "image 2" in str(e.value), (name, str(e.value))
        check_ok()
    with pytest.raises(capi.SfmB200Error) as e:                     # 64x48 at 0.1 is 6x5: below ORB's 8 pixels
        ctx.decode_jpeg_orb([good, J.encode(64, 48, seed=32)], 0.1)
    assert "libsfmb200 error 1:" in str(e.value) and "image 1" in str(e.value), str(e.value)
    check_ok()
    assert ctx.decode_jpeg_orb([]) == ([], [])
    assert ctx.decode_jpeg_orb([], images=False) == (None, [])
    rc = capi.lib().sfmb200_decode_jpeg_extract_orb(ctx._h, None, None, 0, C.c_double(1.0), 5000, 0, None, None, None, None, None)
    assert rc == 0
    check_ok()


def test_stage_and_driver_hook_equal_the_two_call_chain(ctx, tmp_path):
    from sfm_toy_library_b200 import runsfm, stages
    src = _cv(J.crazyhorse())
    files = []
    for k, (dx, dy) in enumerate(((0, 0), (24, 6), (48, 14))):
        view = np.ascontiguousarray(src[40 + dy:700 + dy, 40 + dx:940 + dx])
        ok, buf = cv2.imencode(".jpg", view, [cv2.IMWRITE_JPEG_QUALITY, 92])
        b = buf.tobytes()
        if k == 1:
            b = b[:2] + J.exif_app1(6) + b[2:]                      # a portrait shot among landscape ones
        (tmp_path / f"v{k}.jpg").write_bytes(b)
        files.append(str(tmp_path / f"v{k}.jpg"))
    for s in (1.0, 0.5):
        images, feats = stages.readImagesAndFeatures(files, s, ctx=ctx)
        ref = stages.readImages(files, ctx=ctx, downscale=s)
        assert all(np.array_equal(a, b) for a, b in zip(images, ref))
        for f, im in zip(feats, ref):
            g = stages.extractFeatures(im, ctx=ctx)
            assert np.array_equal(f.keyPoints, g.keyPoints) and np.array_equal(f.descriptors, g.descriptors)
            assert np.array_equal(f.points, g.points)
    sfm = runsfm.SfM.from_directory(str(tmp_path), readImagesAndFeatures=lambda fs, downscale: stages.readImagesAndFeatures(fs, downscale, ctx=ctx))
    assert sfm.n == 3 and sfm.mIntrinsics.K[0, 2] == 450 and sfm.mIntrinsics.K[1, 2] == 330
