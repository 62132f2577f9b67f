"""The C++ readImages and readImagesAndFeatures (host/sfm_images.cpp over sfmb200_decode_images[_extract_orb]) run by their driver
programs on a folder of .png and .jpg files: readImages against cv2.imdecode, readImagesAndFeatures against the Python stage
stages.readImagesAndFeatures (the same images, key points, descriptors and points, bit for bit), at -s 1 and 0.5."""
import os
import subprocess

import numpy as np
import pytest

import jpeg_util as J
import png_util as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _exe(name):
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", name)
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    return exe


def _folder(tmp_path):
    ch = cv2.imread(os.path.join(ROOT, "tests", "golden", "crazyhorse_0.jpg"))
    blobs = [(".png", P.imencode(ch)), (".jpg", J.crazyhorse()),
             (".png", P.make_png(P.picture(221, 333, 4)[:, :, ::-1], 2, 8, 1, filters=(4, 2), pre=P.chunk(b"eXIf", P.exif(6)))),
             (".png", P.imencode(cv2.cvtColor(P.picture(40, 48, 5), cv2.COLOR_BGR2GRAY)))]
    names = []
    for k, (ext, b) in enumerate(blobs):
        p = tmp_path / f"img{k}{ext}"; p.write_bytes(b); names.append(str(p))
    return [b for _, b in blobs], names


def test_cpp_read_images_program_on_png(tmp_path):
    blobs, names = _folder(tmp_path)
    out = tmp_path / "out.bin"
    r = subprocess.run([_exe("test_images"), str(out)] + names, capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "IMAGES_TEST PASS" in r.stdout
    d = out.read_bytes(); i = 0
    for b in blobs:
        h, w = np.frombuffer(d[i:i + 8], np.int32); i += 8
        got = np.frombuffer(d[i:i + h * w * 3], np.uint8).reshape(h, w, 3); i += h * w * 3
        assert np.array_equal(got, cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR))
    assert i == len(d)


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_cpp_read_images_and_features_on_png(tmp_path, scale):
    from sfm_toy_library_b200 import capi, stages
    _, names = _folder(tmp_path)
    out = tmp_path / "out.bin"
    r = subprocess.run([_exe("test_images_features"), "-s", repr(scale), str(out)] + names, capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "IMAGES_FEATURES_TEST PASS" in r.stdout
    ctx = capi.Context(0)
    try:
        images, feats = stages.readImagesAndFeatures(names, scale, ctx=ctx)
    finally:
        ctx.close()
    d = out.read_bytes(); i = 0
    for im, f in zip(images, feats):
        h, w = np.frombuffer(d[i:i + 8], np.int32); i += 8
        assert (h, w) == im.shape[:2]
        assert np.array_equal(np.frombuffer(d[i:i + h * w * 3], np.uint8).reshape(h, w, 3), im); i += h * w * 3
        n = int(np.frombuffer(d[i:i + 4], np.int32)[0]); i += 4
        assert n == f.keyPoints.shape[0]
        rec = np.frombuffer(d[i:i + 28 * n], np.float32).reshape(n, 7); i += 28 * n
        assert np.array_equal(rec[:, :5], f.keyPoints[:, :5])
        assert np.array_equal(rec[:, 5:7].view(np.int32).astype(np.float32), f.keyPoints[:, 5:7])
        assert np.array_equal(np.frombuffer(d[i:i + 32 * n], np.uint8).reshape(n, 32), f.descriptors); i += 32 * n
        assert np.array_equal(np.frombuffer(d[i:i + 8 * n], np.float32).reshape(n, 2), f.points); i += 8 * n
    assert i == len(d)
    assert feats[0].keyPoints.shape[0] > 500
