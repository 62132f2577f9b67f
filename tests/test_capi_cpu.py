"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/sfmb200.h declares, fails loudly
without a GPU (no fallback), and its host-only helpers agree with the oracle."""
import re

import numpy as np
import pytest

from sfm_toy_library_b200 import capi, synth


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as ge
    ge.build()
    return capi.lib()


def test_exports_every_declared_symbol(L):
    header = open(capi.HEADER_PATH).read()
    names = sorted(set(re.findall(r"\b(sfmb200_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 20
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert L.sfmb200_version() == 100


def test_no_silent_cpu_fallback(L):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.SfmB200Error, match="no CUDA device|CUDA"):
        capi.Context(0)


def test_default_options_match_reference_and_ceres_defaults(L, oracle):
    o = capi.ba_default_options(); r = oracle.ba_default_options()
    for k in ("max_num_iterations", "max_solver_time_in_seconds", "function_tolerance", "gradient_tolerance", "parameter_tolerance",
              "initial_trust_region_radius", "max_trust_region_radius", "min_trust_region_radius", "min_relative_decrease",
              "min_lm_diagonal", "max_lm_diagonal", "jacobi_scaling", "max_num_consecutive_invalid_steps"):
        assert getattr(o, k) == getattr(r, k), k
    assert o.max_num_iterations == 500 and o.max_solver_time_in_seconds == 10.0       # SfMBundleAdjustmentUtils.cpp:174,176


def test_pose_conversions_match_oracle(L, oracle):
    rs = np.random.RandomState(2)
    for i in range(60):
        w = rs.normal(0, 1.3, 3) if i % 7 else np.array([0.0, 3.0, 0.3]) * (1 + 0.001 * i)
        R = synth.angle_axis_to_rotmat(w).astype(np.float32)
        np.testing.assert_allclose(capi.rotmat_to_angle_axis_f32(R), oracle.rotmat_to_angle_axis_f32(R), rtol=0, atol=1e-6)
        np.testing.assert_allclose(capi.angle_axis_to_rotmat(w), oracle.angle_axis_to_rotmat(w), rtol=0, atol=1e-15)
    np.testing.assert_array_equal(capi.rotmat_to_angle_axis_f32(np.eye(3, dtype=np.float32)), np.zeros(3, np.float32))
    w = np.array([1e-10, -2e-10, 3e-10])
    np.testing.assert_allclose(capi.angle_axis_to_rotmat(w), oracle.angle_axis_to_rotmat(w), rtol=0, atol=1e-18)


def test_flatten_bundle_follows_reference_assembly_order(L):
    from sfm_toy_library_b200 import stages
    K = np.array([[2500, 0, 512], [0, 2500, 384], [0, 0, 1]], np.float32)
    feats = [stages.Features(points=np.arange(20, dtype=np.float32).reshape(10, 2) + 100 * v) for v in range(4)]
    poses = [np.eye(3, 4, dtype=np.float32) for _ in range(4)]
    poses[1] = np.zeros((3, 4), np.float32)                       # "empty" pose placeholder (:118-122), never observed
    cloud = [stages.Point3DInMap(np.array([0, 0, 5], np.float32), {3: 1, 0: 2}),
             stages.Point3DInMap(np.array([1, 0, 5], np.float32), {2: 4, 0: 5, 3: 6})]
    cams, pts, focal, obs_xy, obs_cam, pt_off, used = stages.flatten_bundle(cloud, poses, stages.Intrinsics(K), feats)
    assert used == [0, 2, 3] and focal == 2500.0
    np.testing.assert_array_equal(pt_off, [0, 2, 5])
    np.testing.assert_array_equal(obs_cam, [0, 2, 0, 1, 2])       # ascending view id within a point (std::map, :146)
    np.testing.assert_array_equal(obs_xy[0], feats[0].points[2] - np.float32([512, 384]))
    np.testing.assert_array_equal(obs_xy[1], feats[3].points[1] - np.float32([512, 384]))
    assert cams.shape == (3, 6) and np.all(cams == 0)


def test_flatten_matches():
    """per-pair match lists -> the match_q / match_t / match_off arrays of the *_pairs calls"""
    mq, mt, off = capi.flatten_matches([], [])
    assert (mq.dtype, mt.dtype, off.dtype) == (np.int32, np.int32, np.int64)
    assert mq.shape == mt.shape == (0,) and off.tolist() == [0]
    from sfm_toy_library_b200 import stages
    m = np.zeros(2, stages.DMATCH); m["queryIdx"] = [4, 0]; m["trainIdx"] = [1, 3]
    mq, mt, off = capi.flatten_matches([m["queryIdx"], np.zeros(0, np.int64), [7], m["queryIdx"][:0]],
                                       [m["trainIdx"], np.zeros(0), np.array([5], np.uint16), m["trainIdx"][:0]])
    assert (mq.dtype, mt.dtype, off.dtype) == (np.int32, np.int32, np.int64)
    assert mq.tolist() == [4, 0, 7] and mt.tolist() == [1, 3, 5] and off.tolist() == [0, 2, 2, 3, 3]
    with pytest.raises(ValueError):
        capi.flatten_matches([[1, 2]], [[1]])


def _naive_validate(nc, obs_cam, pt_off):
    """The obvious nested loop (what the library's slow path and the previous implementation do)."""
    np_, nobs = len(pt_off) - 1, len(obs_cam)
    if np_ == 0:
        return nobs == 0
    if pt_off[0] != 0 or pt_off[np_] != nobs:
        return False
    for p in range(np_):
        if pt_off[p + 1] < pt_off[p] or pt_off[p + 1] > nobs:
            return False
        for o in range(pt_off[p], pt_off[p + 1]):
            if obs_cam[o] < 0 or obs_cam[o] >= nc:
                return False
            if o > pt_off[p] and obs_cam[o] <= obs_cam[o - 1]:
                return False
    return True


def test_ba_validate_accepts_and_rejects_like_the_nested_loop(L):
    """sfmb200_ba_validate (two flat sweeps + descent counting) against the nested loop on valid problems and on every kind of
    corruption: camera out of range / negative, equal or descending cameras inside a point, legal descents at point boundaries,
    empty points, offsets not starting at 0 / not ending at nobs / decreasing / beyond nobs."""
    rs = np.random.RandomState(4)
    p = synth.make_ba_problem(n_cams=9, n_pts=300, obs_per_pt=4, seed=2)
    cam, off = p["obs_cam"].copy(), p["pt_off"].copy()
    assert capi.ba_validate(9, cam, off)[0] == 0
    # ragged with empty points
    ks = rs.randint(0, 5, 200); off2 = np.concatenate([[0], np.cumsum(ks)]).astype(np.int32)
    cam2 = np.concatenate([np.sort(rs.choice(9, k, replace=False)) for k in ks] + [np.empty(0, int)]).astype(np.int32)
    assert _naive_validate(9, cam2, off2) and capi.ba_validate(9, cam2, off2)[0] == 0
    n_bad = 0
    for trial in range(300):
        c, o = cam2.copy(), off2.copy()
        kind = trial % 6
        if kind == 0:
            c[rs.randint(len(c))] = rs.choice([-1, 9, 1000, -2 ** 31])
        elif kind == 1:                                     # duplicate or swap two neighbours somewhere
            i = rs.randint(1, len(c)); c[i] = c[i - 1]
        elif kind == 2:
            i = rs.randint(1, len(c)); c[i - 1], c[i] = c[i], c[i - 1]
        elif kind == 3:
            o[rs.randint(1, len(o) - 1)] += rs.choice([-3, 3])
        elif kind == 4:
            o[-1] += rs.choice([-1, 1])
        else:
            o[0] = 1
        want = _naive_validate(9, c, o)
        rc, msg = capi.ba_validate(9, c, o)
        assert (rc == 0) == want, (kind, msg)
        n_bad += not want
        if not want:
            assert msg
    assert n_bad > 150
    assert capi.ba_validate(5, np.empty(0, np.int32), np.zeros(1, np.int32))[0] == 0           # no points, no observations
    assert capi.ba_validate(5, np.zeros(3, np.int32), np.zeros(1, np.int32))[0] != 0           # observations without points
    rc, msg = capi.ba_validate(300, np.arange(256, dtype=np.int32), np.array([0, 256], np.int32))
    assert rc != 0 and "255" in msg                                                              # more views per point than supported


def test_write_back_rewrites_every_non_empty_pose_like_the_reference(L, oracle):
    """SfMBundleAdjustmentUtils.cpp:192-215: after CONVERGENCE every non-empty pose is rebuilt from its 6-vector -- the
    unobserved ones from their own float angle-axis (a round trip through RotationMatrixToAngleAxis<float> and
    AngleAxisToRotationMatrix<double>); empty poses (:118-122, :196-199) are skipped on the way in and out."""
    from sfm_toy_library_b200 import stages
    rng = np.random.RandomState(3)

    def pose(aa, t):
        P = np.zeros((3, 4), np.float32); P[:, :3] = oracle.angle_axis_to_rotmat(np.asarray(aa, np.float64)); P[:, 3] = t
        return P
    poses = [pose([0.1, -0.2, 0.05], [0, 0, 5]), np.zeros((3, 4), np.float32), pose([0.3, 0.1, -0.4], [1, 2, 3]), pose([-0.2, 0.5, 0.1], [0.5, 0, 4])]
    feats = [stages.Features(points=rng.rand(5, 2).astype(np.float32) * 100) for _ in poses]
    cloud = [stages.Point3DInMap(np.array([0.1 * i, 0.2, 3.0], np.float32), {0: i, 3: i}) for i in range(4)]
    K = np.array([[2500, 0, 512], [0, 2500, 384], [0, 0, 1]], np.float32)
    intr = stages.Intrinsics(K.copy())
    cams, pts, focal, obs_xy, obs_cam, pt_off, used = stages.flatten_bundle(cloud, poses, intr, feats, rot2aa=oracle.rotmat_to_angle_axis_f32)
    assert used == [0, 3] and cams.shape == (2, 6)
    before = [p.copy() for p in poses]
    cams2 = cams.copy(); cams2[:, 3:] += 0.25
    stages.write_back_bundle(cloud, poses, intr, cams2, pts + 1.0, 2400.0, used, rot2aa=oracle.rotmat_to_angle_axis_f32,
                             aa2rot=oracle.angle_axis_to_rotmat)
    assert intr.K[0, 0] == np.float32(2400) and intr.K[1, 1] == np.float32(2400)
    np.testing.assert_array_equal(poses[1], 0)                                   # empty: untouched
    np.testing.assert_allclose(poses[0][:, 3], before[0][:, 3] + 0.25, rtol=1e-6)   # observed: optimised parameters
    aa = oracle.rotmat_to_angle_axis_f32(before[2][:, :3]).astype(np.float64)    # unobserved, non-empty: round trip
    np.testing.assert_array_equal(poses[2][:, :3], oracle.angle_axis_to_rotmat(aa).astype(np.float32))
    np.testing.assert_array_equal(poses[2][:, 3], before[2][:, 3])
    assert np.abs(poses[2] - before[2]).max() < 1e-6
    np.testing.assert_allclose([p.p for p in cloud], pts + 1.0, rtol=1e-6)
    # an observed view with an empty pose enters as CameraVector() = zeros (:120) and is not written back
    poses[3] = np.zeros((3, 4), np.float32)
    cams, *_ = stages.flatten_bundle(cloud, poses, intr, feats, rot2aa=oracle.rotmat_to_angle_axis_f32)
    np.testing.assert_array_equal(cams[1], 0)
