"""PNG decoding on the device (sfmb200_decode_images): the fixture matrix in one call equals cv2.imdecode and each file alone; mixed JPEG
and PNG lists; an all-JPEG list is the JPEG call; the downscale equals cv2.resize; refused files name the caller's index and leave the
context usable; the statistics show which blocks the chain decoded itself and which it took from a probed candidate; a call spanning two memory groups; and SfM.from_directory on a PNG
folder with stages.readImages against the cv2.imread replay."""
import zlib

import numpy as np
import pytest

import jpeg_util as J
import png_util as P

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def files():
    return P.matrix(big=True)


def _cv(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def test_batch_equals_cv2_and_single_calls(ctx, files):
    batch = ctx.decode_images([b for _, b in files])
    st = ctx.png_last_stats()
    print("one call over %d files: %s" % (len(files), st))
    assert st["groups"] == 1 and st["blocks"] >= len(files) and st["speculative_blocks"] > 0
    for (name, b), got in zip(files, batch):
        assert np.array_equal(got, _cv(b)), name
    for (name, b), x in zip(files, batch):
        assert np.array_equal(ctx.decode_images([b])[0], x), name


def test_mixed_and_all_jpeg_lists(ctx, files):
    jpgs = [J.crazyhorse(), J.encode(96, 64, q=90, sampling="422", rst=3, seed=7), J.encode(37, 53, seed=2)]
    pngs = [b for _, b in files[::7]]
    mixed = [pngs[0], jpgs[0], pngs[1], pngs[2], jpgs[1], pngs[3], jpgs[2]]
    out = ctx.decode_images(mixed)
    for k, (b, got) in enumerate(zip(mixed, out)):
        assert np.array_equal(got, _cv(b)), k
    ref = ctx.decode_jpeg(jpgs)
    js = ctx.jpeg_last_stats()
    got = ctx.decode_images(jpgs)
    assert all(np.array_equal(x, y) for x, y in zip(ref, got)) and ctx.jpeg_last_stats() == js
    assert ctx.png_last_stats()["blocks"] == 0
    for s in (0.5, float(np.float32(0.6))):
        assert all(np.array_equal(x, y) for x, y in zip(ctx.decode_jpeg(jpgs, s), ctx.decode_images(jpgs, s))), s


def test_scaled_equals_cv2_resize(ctx, files):
    sel = [b for n, b in files if n.startswith(("crazyhorse", "synthetic", "adam7_7x7", "exif6", "ct3_bd4"))]
    mixed = sel + [J.crazyhorse()]
    for s in (0.5, float(np.float32(0.6)), float(np.float32(0.3))):
        out = ctx.decode_images(mixed, s)
        for k, (b, got) in enumerate(zip(mixed, out)):
            assert np.array_equal(got, cv2.resize(_cv(b), None, fx=s, fy=s)), (s, k)


def test_refused_files_leave_the_context_usable(ctx):
    from sfm_toy_library_b200 import capi
    good = P.make_png(P.picture(20, 30, 1), 2, 8)
    for name, b, status in P.refused():
        for lst, k in (([good, b], 1), ([J.crazyhorse(), good, good, b], 3)):
            with pytest.raises(capi.SfmB200Error) as e:
                ctx.decode_images(lst)
            assert f"libsfmb200 error {status}:" in str(e.value) and f"image {k}:" in str(e.value), (name, str(e.value))
        assert np.array_equal(ctx.decode_images([good])[0], _cv(good)), name
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.decode_images([good, b"GIF89a" + bytes(20)])
    assert "image 1: neither a JPEG nor a PNG file" in str(e.value)
    bad_jpeg = J.crazyhorse()[:3000]
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.decode_images([good, good, bad_jpeg])
    assert "image 2:" in str(e.value)


def test_stats_show_the_chain_and_the_bytes_stay_identical(ctx):
    pic = P.crazyhorse()
    raw = P.raw_data(pic[:, :, ::-1], 2, 8, filters=(4, 1, 0, 2))
    streams = {"dynamic": dict(), "stored": dict(level=0), "fixed": dict(strategy=zlib.Z_FIXED), "sync": dict(flush_every=50000)}
    files = {k: P.make_png(pic[:, :, ::-1], 2, 8, zdata=P.compress(raw, **kw)) for k, kw in streams.items()}
    for k, b in files.items():
        got = ctx.decode_images([b])[0]
        st = ctx.png_last_stats()
        print(k, st)
        assert np.array_equal(got, _cv(b)), k
        assert st["blocks"] == st["chain_blocks"] + st["speculative_blocks"], k
        if k == "dynamic":                                 # every block taken from a probed candidate
            assert st["chain_blocks"] == 0 and st["speculative_blocks"] == st["blocks"] and st["candidates"] >= st["blocks"], k
        elif k in ("stored", "fixed"):                     # no dynamic block: the chain decodes every block itself
            assert st["speculative_blocks"] == 0 and st["chain_blocks"] == st["blocks"], k
        else:                                              # the flushes' stored blocks by the chain, the dynamic ones speculatively
            assert st["chain_blocks"] >= st["stored_blocks"] > 0 and st["speculative_blocks"] > 0, k
        assert (st["stored_blocks"] > 0) == (k in ("stored", "sync")), k
        assert st["fixed_blocks"] == (st["blocks"] if k == "fixed" else 0 if k in ("dynamic", "stored") else st["fixed_blocks"]), k
        assert st["rounds"] >= 1 and st["upload_bytes"] > len(b) // 2 and st["download_bytes"] >= pic.size


def test_a_call_spanning_two_groups(ctx):
    rs = np.random.RandomState(3)
    files = []
    for k in range(5):                                     # 5 x 5 x 48 MB of filtered data: more than one 1 GB group
        g = np.tile(np.arange(8000, dtype=np.uint8)[None, :], (6000, 1)) + rs.randint(0, 3, (6000, 1)).astype(np.uint8) + k
        files.append(P.imencode(g, [cv2.IMWRITE_PNG_COMPRESSION, 1]))
    out = ctx.decode_images(files)
    st = ctx.png_last_stats()
    print(st)
    assert st["groups"] >= 2
    for k, (b, got) in enumerate(zip(files, out)):
        assert np.array_equal(got, _cv(b)), k
    _, feats = ctx.decode_images_orb(files[:1] + files[-1:], 0.25, 500, images=False)
    assert ctx.png_last_stats()["groups"] == 1 and len(feats) == 2


def test_from_directory_with_device_reads_equals_cv2_imread(ctx, tmp_path):
    from sfm_toy_library_b200 import runsfm, stages
    src = _cv(J.crazyhorse())
    for k, (dx, dy) in enumerate(((0, 0), (24, 6), (48, 14), (70, 20))):
        view = np.ascontiguousarray(src[40 + dy:700 + dy, 40 + dx:940 + dx])
        if k == 2:
            ok, buf = cv2.imencode(".jpg", view, [cv2.IMWRITE_JPEG_QUALITY, 92])
            (tmp_path / "v2.jpg").write_bytes(buf.tobytes())
        else:
            (tmp_path / (f"V{k}.PNG" if k % 2 else f"v{k}.png")).write_bytes(P.imencode(view))
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
