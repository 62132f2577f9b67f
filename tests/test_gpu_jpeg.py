"""sfmb200_decode_jpeg_batch on the GPU: byte-identical to cv2.imdecode(IMREAD_COLOR) on the synthetic matrix and the crazyhorse file,
the same bytes alone, batched and on a second call; the crazyhorse chain JPEG -> decode -> grey -> ORB against the committed goldens;
the refused files; and SfM.from_directory with stages.readImages against the cv2.imread replay."""
import os

import numpy as np
import pytest

import jpeg_util as J

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def files():
    return J.matrix() + [("crazyhorse_0", J.crazyhorse())]


def _cv(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def test_batch_equals_cv2_and_single_calls(ctx, files):
    batch = ctx.decode_jpeg([b for _, b in files])
    st = ctx.jpeg_last_stats()
    print("one call over %d files: %s" % (len(files), st))
    for (name, b), got in zip(files, batch):
        assert np.array_equal(got, _cv(b)), name
    again = ctx.decode_jpeg([b for _, b in files])
    for (name, _), x, y in zip(files, batch, again):
        assert np.array_equal(x, y), name
    for (name, b), x in zip(files, batch):
        assert np.array_equal(ctx.decode_jpeg([b])[0], x), name


def test_crazyhorse_chain_to_orb(ctx, golden):
    from sfm_toy_library_b200 import stages
    img = ctx.decode_jpeg([J.crazyhorse()])[0]
    assert np.array_equal(img, _cv(J.crazyhorse()))
    grey = cv2.imread(os.path.join(GOLDEN, "orb_crazyhorse_gray0.png"), cv2.IMREAD_GRAYSCALE)
    assert np.array_equal(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), grey)
    gold = golden("orb_golden.npz")
    f = stages.extractAllFeatures([img], ctx=ctx)[0]
    assert f.keyPoints.shape[0] == gold["kp_5000"].shape[0]
    assert np.array_equal(f.keyPoints[:, :6], gold["kp_5000"]) and np.array_equal(f.descriptors, gold["desc_5000"])


def test_refused_files_leave_the_context_usable(ctx):
    from sfm_toy_library_b200 import capi
    good = J.encode(64, 48, seed=5)
    for name, b, status in J.refused():
        if name not in ("progressive", "truncated", "undefined_code"):
            continue
        with pytest.raises(capi.SfmB200Error) as e:
            ctx.decode_jpeg([good, b])
        assert f"libsfmb200 error {status}:" in str(e.value) and "image 1" in str(e.value), (name, str(e.value))
        assert np.array_equal(ctx.decode_jpeg([good])[0], _cv(good)), name


def test_from_directory_with_device_reads_equals_cv2_imread(ctx, tmp_path):
    from sfm_toy_library_b200 import runsfm, stages
    src = _cv(J.crazyhorse())
    for k, (dx, dy) in enumerate(((0, 0), (24, 6), (48, 14), (70, 20))):
        view = np.ascontiguousarray(src[40 + dy:700 + dy, 40 + dx:940 + dx])
        ok, buf = cv2.imencode(".jpg", view, [cv2.IMWRITE_JPEG_QUALITY, 92])
        (tmp_path / (f"V{k}.JPG" if k % 2 else f"v{k}.jpg")).write_bytes(buf.tobytes())
    (tmp_path / "notes.txt").write_text("not an image")
    runs = []
    for reader in (None, lambda fs: stages.readImages(fs, ctx=ctx)):
        trace = []
        sfm = runsfm.SfM.from_directory(str(tmp_path), readImages=reader, trace=trace)
        try:
            sfm.runSfM()
            outcome = "ok"
        except Exception as e:                     # a degenerate scene may stop the driver; both runs must stop the same way
            outcome = type(e).__name__
        runs.append((sfm, trace, outcome))
    (a, ta, oa), (b, tb, ob) = runs
    assert a.n == b.n == 4 and oa == ob
    for fa, fb in zip(a.mImageFeatures, b.mImageFeatures):
        assert np.array_equal(fa.keyPoints, fb.keyPoints) and np.array_equal(fa.descriptors, fb.descriptors)
    assert len(ta) == len(tb) and [e["stage"] for e in ta] == [e["stage"] for e in tb]
    for x, y in zip(ta, tb):
        assert _same(x, y), x["stage"]


def _same(x, y):
    """Equal structure and values; wall-clock fields (`*_time_s` of a bundle adjustment summary) are not compared."""
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x if not str(k).endswith("time_s"))
    if isinstance(x, (list, tuple)):
        return len(x) == len(y) and all(_same(u, v) for u, v in zip(x, y))
    return np.array_equal(np.asarray(x), np.asarray(y))
