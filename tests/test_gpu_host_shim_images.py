"""The C++ readImages (host/sfm_images.cpp, the imread loop of setImagesDirectory over sfmb200_decode_jpeg_batch), run by its driver
program on the crazyhorse file and two synthetic files, against cv2.imdecode."""
import os
import subprocess

import numpy as np
import pytest

import jpeg_util as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def test_cpp_read_images_program(tmp_path):
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_images")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    blobs = [J.crazyhorse(), J.encode(17, 9, sampling="422", rst=1, seed=3), J.encode(333, 221, q=80, orientation=6, seed=4)]
    names = []
    for k, b in enumerate(blobs):
        p = tmp_path / f"img{k}.jpg"; p.write_bytes(b); names.append(str(p))
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, str(out)] + names, capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "IMAGES_TEST PASS" in r.stdout
    d = out.read_bytes(); i = 0
    for b in blobs:
        h, w = np.frombuffer(d[i:i + 8], np.int32); i += 8
        got = np.frombuffer(d[i:i + h * w * 3], np.uint8).reshape(h, w, 3); i += h * w * 3
        assert np.array_equal(got, cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR))
    assert i == len(d)
