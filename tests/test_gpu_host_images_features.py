"""The C++ readImagesAndFeatures (host/sfm_images.cpp over sfmb200_decode_jpeg_extract_orb), run by its driver program on the crazyhorse
file and synthetic files of mixed sizes (one EXIF-rotated), at -s 1 and 0.5, against the Python stage stages.readImagesAndFeatures: the
same images, key points, descriptors and points, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import jpeg_util as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_cpp_read_images_and_features_equals_python_stage(tmp_path, scale):
    from sfm_toy_library_b200 import capi, stages
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_images_features")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    blobs = [J.crazyhorse(), J.encode(1023, 767, seed=41, orientation=6), J.encode(333, 221, q=80, seed=42), J.encode(48, 40, seed=43)]
    names = []
    for k, b in enumerate(blobs):
        p = tmp_path / f"img{k}.jpg"; p.write_bytes(b); names.append(str(p))
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, "-s", repr(scale), str(out)] + names, capture_output=True, text=True, timeout=300)
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
    assert feats[0].keyPoints.shape[0] > 500 and feats[-1].keyPoints.shape[0] == 0
