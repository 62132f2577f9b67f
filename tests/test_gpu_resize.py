"""The image downscale on the GPU: sfmb200_resize_batch byte-identical to cv2.resize and to the oracle (tests/resize_oracle.py) over the
factor x size grid, one batch of mixed sizes and strides against single calls; sfmb200_decode_jpeg_batch_scaled against
cv2.resize(cv2.imdecode(f)) on the JPEG matrix and the crazyhorse file, and at scale 1 against sfmb200_decode_jpeg_batch; refused
scales; the C++ readImages with -s; and SfM.from_directory(downscale=0.5) on both read paths."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import jpeg_util as J
import resize_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

FACTORS = [float(np.float32(s)) for s in (0.2, 0.25, 0.3, 0.45, 0.5, 0.6, 0.7, 0.75, 0.8, 0.9, 1.25, 1.5, 2.0)]
SIZES = [(1, 37), (37, 1), (9, 9), (173, 99), (175, 101), (333, 221), (1024, 768)]


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _image(w, h, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _cv(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def test_resize_images_equals_cv2_and_oracle(ctx):
    imgs = [_image(w, h, k) for k, (w, h) in enumerate(SIZES)]
    diff = 0
    for s in FACTORS:
        keep = [im for im in imgs if R.resize_size(im.shape[1], im.shape[0], s) is not None]
        got = ctx.resize_images(keep, s)
        for im, g in zip(keep, got):
            ref = cv2.resize(im, None, fx=s, fy=s)
            assert g.shape == ref.shape, (im.shape, s)
            diff += int(np.count_nonzero(g != ref))
            assert np.array_equal(g, ref) and np.array_equal(g, R.resize(im, s)), (im.shape, s)
    big = _image(4000, 3000, 77)
    for s in (0.25, 0.5):
        assert np.array_equal(ctx.resize_images([big], s)[0], cv2.resize(big, None, fx=s, fy=s)), s
    print(f"differing bytes against cv2.resize: {diff}")


def test_mixed_batch_and_strides_equal_single_calls(ctx):
    imgs = [_image(w, h, 10 + k) for k, (w, h) in enumerate(SIZES)]
    padded = []
    for im in imgs:                                    # rows with a longer stride than w * 3
        h, w = im.shape[:2]
        buf = np.full((h, w + 5, 3), 7, np.uint8); buf[:, :w] = im
        padded.append(buf[:, :w])
    for s in (0.5, float(np.float32(0.6)), 1.5, 1.0):
        keep = [k for k, im in enumerate(imgs) if R.resize_size(im.shape[1], im.shape[0], s) is not None]
        assert len(keep) >= len(imgs) - 2
        batch = ctx.resize_images([padded[k] for k in keep], s)
        for im, b in zip([imgs[k] for k in keep], batch):
            assert np.array_equal(b, ctx.resize_images([im], s)[0]), (im.shape, s)
            assert np.array_equal(b, im if s == 1.0 else cv2.resize(im, None, fx=s, fy=s)), (im.shape, s)


def test_decode_jpeg_scaled_equals_cv2(ctx):
    files = J.matrix(big=False) + [("crazyhorse_0", J.crazyhorse())]
    for s in (0.5, 0.25, float(np.float32(0.6)), 1.5):
        keep = [(n, b) for n, b in files if R.resize_size(*_cv(b).shape[1::-1], s) is not None]
        got = ctx.decode_jpeg([b for _, b in keep], s)
        st = ctx.jpeg_last_stats()
        # the download is the per-image error flags, the statistics and the resized images only
        assert st["download_bytes"] == _al256(4 * len(got)) + 256 + sum(_al256(g.size) for g in got)
        for (name, b), g in zip(keep, got):
            assert np.array_equal(g, cv2.resize(_cv(b), None, fx=s, fy=s)), (name, s)
        print(f"scale {s:g}: {len(keep)} files, download {st['download_bytes']} bytes")


def _al256(x):
    return (x + 255) // 256 * 256


def test_decode_jpeg_scale_1_is_decode_jpeg(ctx):
    files = [b for _, b in J.matrix(big=False)[:12]] + [J.crazyhorse()]
    a = ctx.decode_jpeg(files)
    st_a = ctx.jpeg_last_stats()
    from sfm_toy_library_b200 import capi
    import ctypes as C
    n = len(files)
    outs = [np.empty_like(x) for x in a]
    data = (C.c_char_p * n)(*files); sizes = (C.c_size_t * n)(*[len(f) for f in files])
    ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    ctx._check(capi.lib().sfmb200_decode_jpeg_batch_scaled(ctx._h, data, sizes, n, C.c_double(1.0), ptrs, None))
    assert ctx.jpeg_last_stats() == st_a
    for x, y in zip(a, outs):
        assert np.array_equal(x, y)


def test_refused_scales_leave_the_context_usable(ctx):
    from sfm_toy_library_b200 import capi
    im = _image(64, 48, 3)
    jpg = J.encode(64, 48, seed=5)
    for s in (0.0, -0.5, float("nan"), float("inf"), 0.001):
        with pytest.raises(capi.SfmB200Error) as e:
            ctx.resize_images([im], s)
        assert "libsfmb200 error 1:" in str(e.value), s
        with pytest.raises(capi.SfmB200Error) as e:
            ctx.decode_jpeg([jpg], s)
        assert "libsfmb200 error 1:" in str(e.value), s
        assert np.array_equal(ctx.resize_images([im], 0.5)[0], cv2.resize(im, None, fx=0.5, fy=0.5)), s
        assert np.array_equal(ctx.decode_jpeg([jpg], 0.25)[0], cv2.resize(_cv(jpg), None, fx=0.25, fy=0.25)), s


def test_cpp_read_images_with_downscale(tmp_path):
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_images")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    blobs = [J.crazyhorse(), J.encode(17, 9, sampling="422", rst=1, seed=3), J.encode(333, 221, q=80, orientation=6, seed=4)]
    names = []
    for k, b in enumerate(blobs):
        p = tmp_path / f"img{k}.jpg"; p.write_bytes(b); names.append(str(p))
    for s in ("0.5", "0.3"):
        out = tmp_path / f"out{s}.bin"
        r = subprocess.run([exe, "-s", s, str(out)] + names, capture_output=True, text=True, timeout=300)
        print(r.stdout[-2000:], r.stderr[-2000:])
        assert r.returncode == 0 and "IMAGES_TEST PASS" in r.stdout
        f = float(np.float32(s))
        d = out.read_bytes(); i = 0
        for b in blobs:
            h, w = np.frombuffer(d[i:i + 8], np.int32); i += 8
            got = np.frombuffer(d[i:i + h * w * 3], np.uint8).reshape(h, w, 3); i += h * w * 3
            assert np.array_equal(got, cv2.resize(_cv(b), None, fx=f, fy=f)), s
        assert i == len(d)


def test_from_directory_downscale(ctx, tmp_path):
    from sfm_toy_library_b200 import runsfm, stages
    for k in range(3):
        shutil.copy(os.path.join(J.GOLDEN, "crazyhorse_0.jpg"), tmp_path / f"ch{k}.jpg")
    ref = cv2.resize(_cv(J.crazyhorse()), None, fx=0.5, fy=0.5)
    h, w = ref.shape[:2]
    K = np.array([[2500, 0, w // 2], [0, 2500, h // 2], [0, 0, 1]], np.float32)
    seen = []

    def extract(images):
        seen.append([im.copy() for im in images])
        return stages.extractAllFeatures(images, ctx=ctx)
    for reader in (None, lambda fs, downscale=1.0: stages.readImages(fs, ctx=ctx, downscale=downscale)):
        sfm = runsfm.SfM.from_directory(str(tmp_path), readImages=reader, extractAllFeatures=extract, downscale=0.5)
        assert sfm.n == 3 and np.array_equal(sfm.mIntrinsics.K, K)
    assert len(seen) == 2
    for a, b in zip(*seen):
        assert np.array_equal(a, ref) and np.array_equal(b, ref)
