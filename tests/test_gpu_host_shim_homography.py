"""The C++ shim built with SFMB200_SHIM_HOMOGRAPHY: SfMStereoUtilities::findHomographyInliers (reference signature) over
sfmb200_find_homography_pairs, run by its C++ test program on a planar pair with planted inliers and outliers."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_cpp_shim_homography_program():
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_shim_homography")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "SHIM_HOMOGRAPHY_TEST PASS" in r.stdout
