"""The C++ shim built with SFMB200_SHIM_POSE: SfMStereoUtilities::findCameraPoseFrom2D3DMatch (reference signature) over
sfmb200_find_camera_pose.  Its C++ test program checks the reference's find_camera_pose_from_2d3d_match scene; on the five crazyhorse
PnP sets and a set that fails the ratio test, the shim's decision and pose are bitwise those of ransac.findCameraPoseFrom2D3DMatch_gpu
with the same (default) seed."""
import os
import subprocess

import numpy as np
import pytest

from cfg1_util import Cfg1
from sfm_toy_library_b200 import capi, ransac, stages

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _exe():
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_shim_pose")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    return exe


def test_cpp_shim_pose_program():
    r = subprocess.run([_exe()], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "SHIM_POSE_TEST PASS" in r.stdout


def test_shim_equals_the_python_stage(tmp_path):
    cfg = Cfg1(); g = cfg.g
    ctx = capi.Context(0)
    try:
        sets = [(g[f"pnp_{k}_p3"], g[f"pnp_{k}_p2"], np.asarray(g[f"ba_{k}_K_after"], np.float32)) for k in range(cfg.n_pnp)]
        rs = np.random.RandomState(3)
        X, uv, K = sets[0]
        sets.append((X, uv[rs.permutation(len(uv))], K))                   # scrambled: fails the ratio test
        decisions = []
        for i, (X, uv, K) in enumerate(sets):
            path = tmp_path / f"set{i}.bin"
            with open(path, "wb") as f:
                f.write(np.int32(len(X)).tobytes()); f.write(np.ascontiguousarray(K, np.float32).tobytes())
                f.write(np.ascontiguousarray(X, np.float32).tobytes()); f.write(np.ascontiguousarray(uv, np.float32).tobytes())
            r = subprocess.run([_exe(), str(path)], capture_output=True, text=True, timeout=300)
            assert r.returncode == 0, r.stdout + r.stderr
            lines = r.stdout.split("\n")
            acc = int(next(l for l in lines if l.startswith("accepted")).split()[1])
            pose = np.array([float.fromhex(v) for v in next(l for l in lines if l.startswith("pose")).split()[1:]], np.float32).reshape(3, 4)
            ok, ref = ransac.findCameraPoseFrom2D3DMatch_gpu(stages.Intrinsics(K), uv, X, ctx=ctx, seed=0)
            assert acc == int(ok), i
            if ok:
                np.testing.assert_array_equal(pose, ref)
            else:
                assert np.all(pose == -7.0) and "Inliers ratio is too small" in r.stderr
            decisions.append(ok)
        assert decisions[-1] is False and all(decisions[:-1]) == all(bool(g[f"pnp_{k}_ok"]) for k in range(cfg.n_pnp))
    finally:
        ctx.close()
