"""ctypes binding of the C ABI (include/sfmb200.h -> lib/libsfmb200.so).

Thin by design: numpy arrays in, numpy arrays out, every call goes straight to the shared library.  There is NO
fallback: if the library is missing or there is no GPU, calls raise SfmB200Error.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsfmb200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "sfmb200.h")
UNIQUE_ID_BYTES = 128
RATIO_REFERENCE = float(np.float64(np.float32(0.8)))     # NN_MATCH_RATIO = (double)0.8f, SfM2DFeatureUtilities.cpp:35
MIN_REPROJECTION_ERROR = 10.0                            # SfMStereoUtilities.cpp:42
CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2
MODEL_HOMOGRAPHY, MODEL_ESSENTIAL, MODEL_POSE = 0, 1, 2

_lib = None


class SfmB200Error(RuntimeError):
    pass


class BAOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int), ("max_solver_time_in_seconds", C.c_double),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
                ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double), ("jacobi_scaling", C.c_int),
                ("max_num_consecutive_invalid_steps", C.c_int), ("verbose", C.c_int), ("profile", C.c_int), ("l2_flush_mb", C.c_int)]


class BASummary(C.Structure):
    _fields_ = [("termination_type", C.c_int), ("num_iterations", C.c_int), ("num_successful_steps", C.c_int),
                ("num_unsuccessful_steps", C.c_int), ("num_jacobian_passes", C.c_int), ("num_linear_solves", C.c_int),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("total_time_s", C.c_double),
                ("schur_ms_total", C.c_double), ("schur_launches", C.c_int), ("pair_ms_total", C.c_double), ("pair_launches", C.c_int), ("camera_ms_total", C.c_double),
                ("solve_ms_total", C.c_double), ("flush_ms_total", C.c_double),
                ("kernel_launches", C.c_int64),
                ("message", C.c_char * 160)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["message"] = self.message.decode()
        return d


class EssentialOptions(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("confidence", C.c_double), ("threshold_px", C.c_double), ("distance_thresh", C.c_double),
                ("seed", C.c_uint64)]


class EssentialSummary(C.Structure):
    _fields_ = [("found", C.c_int), ("n_inliers", C.c_int), ("n_good", C.c_int), ("iterations", C.c_int), ("n_samples", C.c_int),
                ("n_hypotheses", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class PoseOptions(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("confidence", C.c_double), ("threshold_px", C.c_double), ("refine_iters", C.c_int),
                ("seed", C.c_uint64)]


class PoseSummary(C.Structure):
    _fields_ = [("found", C.c_int), ("n_inliers", C.c_int), ("iterations", C.c_int), ("n_samples", C.c_int), ("n_hypotheses", C.c_int),
                ("refined", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class HomographyOptions(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("confidence", C.c_double), ("threshold_px", C.c_double), ("refine_iters", C.c_int),
                ("record_trace", C.c_int)]


class HomographySummary(C.Structure):
    _fields_ = [("found", C.c_int), ("n_inliers", C.c_int), ("ransac_inliers", C.c_int), ("iterations", C.c_int)]


def lib():
    """Load libsfmb200.so (built by build.py / __graft_entry__.build()).  No fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SfmB200Error(f"{LIB_PATH} not found: run `python sfm-toy-library_b200/build.py` (nvcc, sm_90a). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.sfmb200_last_error.restype = C.c_char_p
        L.sfmb200_last_error.argtypes = [C.c_void_p]
        L.sfmb200_stream.restype = C.c_void_p
        L.sfmb200_stream.argtypes = [C.c_void_p]
        L.sfmb200_kernel_launches.restype = C.c_int64
        L.sfmb200_kernel_launches.argtypes = [C.c_void_p]
        for name in ("sfmb200_destroy", "sfmb200_descset_destroy", "sfmb200_ba_problem_destroy"):
            getattr(L, name).restype = None
            getattr(L, name).argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def _vp(x):
    return C.c_void_p(x)


def flatten_matches(q_list, t_list):
    """Per-pair match lists (queryIdx / trainIdx arrays, one of each per pair) -> (match_q int32, match_t int32, match_off int64
    [len(q_list) + 1]), the concatenated form the *_pairs calls take."""
    if len(q_list) != len(t_list) or any(len(q) != len(t) for q, t in zip(q_list, t_list)):
        raise ValueError("flatten_matches: every pair needs as many query as train indices")
    off = np.zeros(len(q_list) + 1, np.int64); off[1:] = np.cumsum([len(q) for q in q_list])
    cat = lambda xs: np.concatenate([np.asarray(x, np.int32) for x in xs]) if len(xs) else np.zeros(0, np.int32)
    return cat(q_list), cat(t_list), off


def _pair_batch_args(points, pairs, match_q, match_t, match_off):
    """The image-pair batch arrays of include/sfmb200.h as ctypes arguments, in the C order pts, img_off, n_img, pairs, n_pairs,
    match_q, match_t, match_off; and the numbers of pairs and matches.  The arrays are kept alive by the returned pointers."""
    pts = [np.ascontiguousarray(p, np.float32).reshape(-1, 2) for p in points]
    img_off = np.zeros(len(pts) + 1, np.int32); img_off[1:] = np.cumsum([len(p) for p in pts])
    allp = np.ascontiguousarray(np.concatenate(pts, 0)) if pts else np.zeros((0, 2), np.float32)
    pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    mq = np.ascontiguousarray(match_q, np.int32); mt = np.ascontiguousarray(match_t, np.int32)
    moff = np.ascontiguousarray(match_off, np.int64)
    P = pairs.shape[0]
    if moff.shape[0] != P + 1 or mq.shape != mt.shape or (P and moff[-1] != mq.shape[0]):
        raise ValueError("match_off must have len(pairs) + 1 entries ending at the number of matches")
    args = (_p(allp, C.c_float), _p(img_off, C.c_int32), len(pts), _p(pairs, C.c_int32), P, _p(mq, C.c_int32), _p(mt, C.c_int32),
            _p(moff, C.c_int64))
    return args, P, mq.shape[0]


class Context:
    """sfmb200_ctx: one per GPU."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().sfmb200_create(int(device), C.byref(self._h))
        if rc != 0:
            raise SfmB200Error(f"sfmb200_create failed ({rc}): {lib().sfmb200_last_error(None).decode()}")
        self.device = device
        self._children = []          # weak references to live DescriptorSets / BAProblems: they must die before the context

    def _adopt(self, child):
        import weakref
        self._children.append(weakref.ref(child))

    def close(self):
        if self._h:
            for ref in self._children:          # a problem / descriptor set destroyed after its context would touch freed memory
                child = ref()
                if child is not None:
                    child.close()
            self._children = []
            lib().sfmb200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise SfmB200Error(f"libsfmb200 error {rc}: {lib().sfmb200_last_error(self._h).decode()}")

    @property
    def stream(self):
        return lib().sfmb200_stream(self._h)

    @property
    def kernel_launches(self):
        return int(lib().sfmb200_kernel_launches(self._h))

    def synchronize(self):
        self._check(lib().sfmb200_synchronize(self._h))

    # ------------------------------------------------------------------ a-1 matching
    def match_knn2_ratio(self, q, t, ratio=RATIO_REFERENCE):
        q = np.ascontiguousarray(q, np.uint8); t = np.ascontiguousarray(t, np.uint8)
        nq, nt = q.shape[0], t.shape[0]
        nb = q.shape[1] if q.ndim == 2 and nq else (t.shape[1] if t.ndim == 2 else 32)
        oq = np.empty(max(nq, 1), np.int32); ot = np.empty(max(nq, 1), np.int32); od = np.empty(max(nq, 1), np.float32)
        n = C.c_int(0)
        self._check(lib().sfmb200_match_knn2_ratio(self._h, _p(q, C.c_uint8), nq, _p(t, C.c_uint8), nt, nb, C.c_double(ratio),
                                                   _p(oq, C.c_int32), _p(ot, C.c_int32), _p(od, C.c_float), C.byref(n)))
        return oq[:n.value].copy(), ot[:n.value].copy(), od[:n.value].copy()

    def match_knn2_ratio_l2(self, q, t, ratio=RATIO_REFERENCE):
        q = np.ascontiguousarray(q, np.float32); t = np.ascontiguousarray(t, np.float32)
        nq, nt, dim = q.shape[0], t.shape[0], q.shape[1]
        oq = np.empty(max(nq, 1), np.int32); ot = np.empty(max(nq, 1), np.int32); od = np.empty(max(nq, 1), np.float32)
        n = C.c_int(0)
        self._check(lib().sfmb200_match_knn2_ratio_l2(self._h, _p(q, C.c_float), nq, _p(t, C.c_float), nt, dim, C.c_double(ratio),
                                                      _p(oq, C.c_int32), _p(ot, C.c_int32), _p(od, C.c_float), C.byref(n)))
        return oq[:n.value].copy(), ot[:n.value].copy(), od[:n.value].copy()

    def descriptor_set(self, desc_list, norm="hamming"):
        return DescriptorSet(self, desc_list, norm)

    # ------------------------------------------------------------------ a-2 triangulation
    def triangulate(self, K, Pl, Pr, pts_left, pts_right, match_q=None, match_t=None, max_reproj=MIN_REPROJECTION_ERROR):
        K = np.ascontiguousarray(K, np.float32).reshape(9); Pl = np.ascontiguousarray(Pl, np.float32).reshape(12)
        Pr = np.ascontiguousarray(Pr, np.float32).reshape(12)
        L = np.ascontiguousarray(pts_left, np.float32).reshape(-1, 2); R = np.ascontiguousarray(pts_right, np.float32).reshape(-1, 2)
        if match_q is not None:
            match_q = np.ascontiguousarray(match_q, np.int32); match_t = np.ascontiguousarray(match_t, np.int32); m = match_q.shape[0]
        else:
            m = min(L.shape[0], R.shape[0])
        X = np.empty((max(m, 1), 3), np.float32); keep = np.empty(max(m, 1), np.uint8); nk = C.c_int(0)
        self._check(lib().sfmb200_triangulate(self._h, _p(K, C.c_float), _p(Pl, C.c_float), _p(Pr, C.c_float), _p(L, C.c_float), L.shape[0],
                                              _p(R, C.c_float), R.shape[0], _p(match_q, C.c_int32), _p(match_t, C.c_int32), m,
                                              C.c_float(max_reproj), _p(X, C.c_float), _p(keep, C.c_uint8), C.byref(nk)))
        return X[:m], keep[:m], nk.value

    def triangulate_pairs(self, K, poses, points, pairs, match_q, match_t, match_off, max_reproj=MIN_REPROJECTION_ERROR):
        """sfmb200_triangulate_pairs: triangulate for every pair in one call, with the arguments of find_camera_matrices_pairs
        (points: list of [n_i, 2] key points per image; pairs [P, 2]; match_q / match_t: all pairs' matches concatenated, pair p
        owning match_off[p]:match_off[p+1]).  poses [P, 2, 3, 4]: pair p's (Pleft, Pright).
        Returns (X [sum of matches, 3], keep [sum of matches], n_keep [P])."""
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        batch, P, M = _pair_batch_args(points, pairs, match_q, match_t, match_off)
        poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 24)
        if poses.shape[0] != P:
            raise ValueError("poses must hold one (Pleft, Pright) per pair")
        X = np.empty((max(M, 1), 3), np.float32); keep = np.empty(max(M, 1), np.uint8); nk = np.zeros(max(P, 1), np.int32)
        self._check(lib().sfmb200_triangulate_pairs(self._h, _p(K, C.c_float), _p(poses, C.c_float), *batch, C.c_float(max_reproj),
                                                    _p(X, C.c_float), _p(keep, C.c_uint8), _p(nk, C.c_int32)))
        return X[:M], keep[:M], nk[:P]

    def triangulate_device(self, K, Pl, Pr, d_left, d_right, d_mq, d_mt, m, d_X, d_keep, d_nkeep, max_reproj=MIN_REPROJECTION_ERROR):
        """All d_* are raw device pointers (ints); nothing is synchronised."""
        K = np.ascontiguousarray(K, np.float32).reshape(9); Pl = np.ascontiguousarray(Pl, np.float32).reshape(12)
        Pr = np.ascontiguousarray(Pr, np.float32).reshape(12)
        self._check(lib().sfmb200_triangulate_device(self._h, _p(K, C.c_float), _p(Pl, C.c_float), _p(Pr, C.c_float), _vp(d_left), _vp(d_right),
                                                     _vp(d_mq), _vp(d_mt), int(m), C.c_float(max_reproj), _vp(d_X), _vp(d_keep), _vp(d_nkeep)))

    # ------------------------------------------------------------------ a-3/a-4 bundle adjustment
    def ba_problem(self, cams, pts, focal, obs_xy, obs_cam, pt_off):
        return BAProblem(self, cams, pts, focal, obs_xy, obs_cam, pt_off)

    def ba_solve(self, cams, pts, focal, obs_xy, obs_cam, pt_off, options=None, inplace=False):
        """One-shot sfmb200_ba_solve with host buffers.  Returns (cams, pts, focal, summary dict).
        inplace=True hands the caller's float64 C-contiguous cams / pts arrays (e.g. pinned memory) to the library, which
        overwrites them with the result -- exactly what the C ABI does; the default works on copies."""
        if inplace:
            for x in (cams, pts):
                if not (isinstance(x, np.ndarray) and x.dtype == np.float64 and x.flags.c_contiguous and x.flags.writeable):
                    raise ValueError("inplace=True needs writeable float64 C-contiguous arrays")
            cams = cams.reshape(-1, 6); pts = pts.reshape(-1, 3)
        else:
            cams = np.array(cams, np.float64, order="C").reshape(-1, 6); pts = np.array(pts, np.float64, order="C").reshape(-1, 3)
        obs_xy = np.ascontiguousarray(obs_xy, np.float32).reshape(-1, 2); obs_cam = np.ascontiguousarray(obs_cam, np.int32)
        pt_off = np.ascontiguousarray(pt_off, np.int32)
        f = C.c_double(float(focal)); s = BASummary(); o = options or ba_default_options()
        self._check(lib().sfmb200_ba_solve(self._h, C.byref(o), cams.shape[0], pts.shape[0], obs_cam.shape[0], _p(cams, C.c_double),
                                           _p(pts, C.c_double), C.byref(f), _p(obs_xy, C.c_float), _p(obs_cam, C.c_int32),
                                           _p(pt_off, C.c_int32), C.byref(s)))
        return cams, pts, f.value, s.as_dict()

    # ------------------------------------------------------------------ f-2 RANSAC hypothesis scoring
    def ransac_score(self, model, a, b, hyps, aux=None, threshold=10.0, want_mask=True):
        """sfmb200_ransac_score: model 0 homography / 1 essential / 2 pose.  Returns (inlier counts [nh], best index, best mask [n])."""
        a = np.ascontiguousarray(a, np.float32).reshape(-1, 3 if model == 2 else 2); b = np.ascontiguousarray(b, np.float32).reshape(-1, 2)
        hd = 12 if model == 2 else 9
        hyps = np.ascontiguousarray(hyps, np.float64).reshape(-1, hd)
        n, nh = b.shape[0], hyps.shape[0]
        aux9 = np.zeros(9)
        if aux is not None:
            av = np.asarray(aux, np.float64).reshape(-1); aux9[:len(av)] = av
        counts = np.zeros(max(nh, 1), np.int32); best = C.c_int32(-1); mask = np.zeros(max(n, 1), np.uint8)
        self._check(lib().sfmb200_ransac_score(self._h, int(model), _p(a, C.c_float), _p(b, C.c_float), n, _p(hyps, C.c_double), nh, _p(aux9, C.c_double),
                                               C.c_double(float(threshold)), _p(counts, C.c_int32), C.byref(best), _p(mask, C.c_uint8) if want_mask else None))
        return counts[:nh], int(best.value), mask[:n]

    # ------------------------------------------------------------------ f-2 essential-matrix RANSAC + pose recovery
    def find_camera_matrices(self, K, pts_left, pts_right, match_q=None, match_t=None, options=None, **kw):
        """sfmb200_find_camera_matrices: findEssentialMat(RANSAC) + recoverPose on the device.  options: EssentialOptions or
        keyword overrides of the defaults (max_iters, confidence, threshold_px, distance_thresh, seed).
        Returns (E [3,3], R [3,3], t [3], inlier_mask [m], pose_mask [m], summary dict)."""
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        L = np.ascontiguousarray(pts_left, np.float32).reshape(-1, 2); R = np.ascontiguousarray(pts_right, np.float32).reshape(-1, 2)
        if match_q is not None:
            match_q = np.ascontiguousarray(match_q, np.int32); match_t = np.ascontiguousarray(match_t, np.int32); m = match_q.shape[0]
        else:
            m = min(L.shape[0], R.shape[0])
        o = options or essential_default_options(**kw)
        E = np.zeros(9); Rm = np.zeros(9); t = np.zeros(3)
        inl = np.zeros(max(m, 1), np.uint8); pm = np.zeros(max(m, 1), np.uint8); s = EssentialSummary()
        self._check(lib().sfmb200_find_camera_matrices(self._h, _p(K, C.c_float), _p(L, C.c_float), L.shape[0], _p(R, C.c_float), R.shape[0],
                                                       _p(match_q, C.c_int32), _p(match_t, C.c_int32), m, C.byref(o), _p(E, C.c_double),
                                                       _p(Rm, C.c_double), _p(t, C.c_double), _p(inl, C.c_uint8), _p(pm, C.c_uint8), C.byref(s)))
        return E.reshape(3, 3), Rm.reshape(3, 3), t, inl[:m], pm[:m], s.as_dict()

    def find_camera_matrices_pairs(self, K, points, pairs, match_q, match_t, match_off, options=None, **kw):
        """sfmb200_find_camera_matrices_pairs: find_camera_matrices for every pair in one call, with the arguments of
        find_homography_pairs (points: list of [n_i, 2] key points per image; pairs [P, 2]; match_q / match_t: all pairs' matches
        concatenated, pair p owning match_off[p]:match_off[p+1]).  options: EssentialOptions or keyword overrides of the defaults.
        Returns (E [P, 3, 3], R [P, 3, 3], t [P, 3], inlier_mask [sum of matches], pose_mask [sum of matches], summary dict of
        arrays found / n_inliers / n_good / iterations / n_samples / n_hypotheses [P])."""
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        batch, P, M = _pair_batch_args(points, pairs, match_q, match_t, match_off)
        o = options or essential_default_options(**kw)
        E = np.zeros((max(P, 1), 9)); Rm = np.zeros((max(P, 1), 9)); t = np.zeros((max(P, 1), 3))
        inl = np.zeros(max(M, 1), np.uint8); pm = np.zeros(max(M, 1), np.uint8); s = (EssentialSummary * max(P, 1))()
        self._check(lib().sfmb200_find_camera_matrices_pairs(self._h, _p(K, C.c_float), *batch, C.byref(o), _p(E, C.c_double), _p(Rm, C.c_double),
                                                             _p(t, C.c_double), _p(inl, C.c_uint8), _p(pm, C.c_uint8), s))
        summ = {k: np.array([getattr(s[p], k) for p in range(P)], np.int32) for k, _ in EssentialSummary._fields_}
        return E[:P].reshape(P, 3, 3), Rm[:P].reshape(P, 3, 3), t[:P], inl[:M], pm[:M], summ

    def five_point(self, x1, x2):
        """sfmb200_five_point: x1, x2 [ns, 5, 2] normalised coordinates -> (E [ns, 10, 3, 3], nsol [ns])."""
        x1 = np.ascontiguousarray(x1, np.float64).reshape(-1, 5, 2); x2 = np.ascontiguousarray(x2, np.float64).reshape(-1, 5, 2)
        ns = x1.shape[0]
        E = np.zeros((max(ns, 1), 10, 9)); n = np.zeros(max(ns, 1), np.int32)
        self._check(lib().sfmb200_five_point(self._h, _p(x1, C.c_double), _p(x2, C.c_double), ns, _p(E, C.c_double), _p(n, C.c_int32)))
        return E[:ns].reshape(ns, 10, 3, 3), n[:ns]

    def essential_last_trace(self):
        """sfmb200_essential_last_trace: (samples [S, 5], nsol [S], counts [sum nsol]) of the last find_camera_matrices call."""
        f = lib().sfmb200_essential_last_trace
        S = f(self._h, 0, None, None, None)
        if S < 0:
            raise SfmB200Error("sfmb200_essential_last_trace failed")
        smp = np.zeros((max(S, 1), 5), np.int32); n = np.zeros(max(S, 1), np.int32); c = np.zeros(max(10 * S, 1), np.int32)
        if f(self._h, S, _p(smp, C.c_int32), _p(n, C.c_int32), _p(c, C.c_int32)) != S:
            raise SfmB200Error("sfmb200_essential_last_trace failed")
        return smp[:S], n[:S], c[:int(n[:S].sum())]

    # ------------------------------------------------------------------ f-2 PnP RANSAC + refit
    def find_camera_pose(self, K, pts3, pts2, options=None, **kw):
        """sfmb200_find_camera_pose: cv::solvePnPRansac's job on the device (seeded EPnP samples, OpenCV's selection, least-squares
        refit).  pts3 [m, 3], pts2 [m, 2] float; options: PoseOptions or keyword overrides of the defaults (max_iters, confidence,
        threshold_px, refine_iters, seed).  Returns (rvec [3], R [3, 3], t [3], inlier_mask [m], summary dict)."""
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        X = np.ascontiguousarray(pts3, np.float32).reshape(-1, 3); uv = np.ascontiguousarray(pts2, np.float32).reshape(-1, 2)
        if X.shape[0] != uv.shape[0]:
            raise ValueError("find_camera_pose: as many 3D as 2D points")
        m = X.shape[0]
        o = options or pose_default_options(**kw)
        rv = np.zeros(3); Rm = np.zeros(9); t = np.zeros(3); mask = np.zeros(max(m, 1), np.uint8); s = PoseSummary()
        self._check(lib().sfmb200_find_camera_pose(self._h, _p(K, C.c_float), _p(X, C.c_float), _p(uv, C.c_float), m, C.byref(o), _p(rv, C.c_double),
                                                   _p(Rm, C.c_double), _p(t, C.c_double), _p(mask, C.c_uint8), C.byref(s)))
        return rv, Rm.reshape(3, 3), t, mask[:m], s.as_dict()

    def epnp(self, X, uv, K):
        """sfmb200_epnp: the device EPnP solver on given samples, X [ns, 5, 3], uv [ns, 5, 2] pixels, K [3, 3] ->
        (Rt [ns, 3, 4], ok [ns])."""
        X = np.ascontiguousarray(X, np.float64).reshape(-1, 5, 3); uv = np.ascontiguousarray(uv, np.float64).reshape(-1, 5, 2)
        K = np.ascontiguousarray(K, np.float64).reshape(9)
        ns = X.shape[0]
        Rt = np.zeros((max(ns, 1), 12)); ok = np.zeros(max(ns, 1), np.uint8)
        self._check(lib().sfmb200_epnp(self._h, _p(X, C.c_double), _p(uv, C.c_double), _p(K, C.c_double), ns, _p(Rt, C.c_double), _p(ok, C.c_uint8)))
        return Rt[:ns].reshape(ns, 3, 4), ok[:ns]

    def pose_last_trace(self):
        """sfmb200_pose_last_trace: (samples [S, 5], inlier counts [S], -1 where a sample gave no pose) of the last find_camera_pose."""
        f = lib().sfmb200_pose_last_trace
        S = f(self._h, 0, None, None)
        if S < 0:
            raise SfmB200Error("sfmb200_pose_last_trace failed")
        smp = np.zeros((max(S, 1), 5), np.int32); c = np.zeros(max(S, 1), np.int32)
        if f(self._h, S, _p(smp, C.c_int32), _p(c, C.c_int32)) != S:
            raise SfmB200Error("sfmb200_pose_last_trace failed")
        return smp[:S], c[:S]

    # ------------------------------------------------------------------ f-2 homography RANSAC for many pairs
    def find_homography_pairs(self, points, pairs, match_q, match_t, match_off, options=None, **kw):
        """sfmb200_find_homography_pairs: cv::findHomography(RANSAC) for every pair in one call.  points: list of [n_i, 2] key
        points per image; pairs [P, 2]; match_q / match_t: all pairs' matches concatenated, pair p owning match_off[p]:match_off[p+1].
        options: HomographyOptions or keyword overrides of the defaults (max_iters, confidence, threshold_px, refine_iters,
        record_trace).  Returns (H [P, 3, 3], mask [sum of matches] uint8, summary dict of arrays found / n_inliers /
        ransac_inliers / iterations [P])."""
        batch, P, M = _pair_batch_args(points, pairs, match_q, match_t, match_off)
        o = options or homography_default_options(**kw)
        H = np.zeros((max(P, 1), 9)); mask = np.zeros(max(M, 1), np.uint8); s = (HomographySummary * max(P, 1))()
        self._check(lib().sfmb200_find_homography_pairs(self._h, *batch, C.byref(o), _p(H, C.c_double), _p(mask, C.c_uint8), s))
        summ = {k: np.array([getattr(s[p], k) for p in range(P)], np.int32) for k, _ in HomographySummary._fields_}
        return H[:P].reshape(P, 3, 3), mask[:M], summ

    def homography_last_trace(self, pair):
        """sfmb200_homography_last_trace: (quads [V, 4], RANSAC counts [V]) visited for `pair` by the last find_homography_pairs call
        made with record_trace=1."""
        f = lib().sfmb200_homography_last_trace
        V = f(self._h, int(pair), 0, None, None)
        if V < 0:
            raise SfmB200Error("sfmb200_homography_last_trace failed (no trace recorded?)")
        q = np.zeros((max(V, 1), 4), np.int32); c = np.zeros(max(V, 1), np.int32)
        if f(self._h, int(pair), V, _p(q, C.c_int32), _p(c, C.c_int32)) != V:
            raise SfmB200Error("sfmb200_homography_last_trace failed")
        return q[:V], c[:V]

    # ------------------------------------------------------------------ f-3 ORB extraction
    def orb_detect_and_compute(self, images, nfeatures=5000, capacity=None):
        """sfmb200_orb_detect_and_compute[_batch]: `ORB::create(nfeatures)->detectAndCompute` (SfM2DFeatureUtilities.cpp:39, 48).
        `images`: one uint8 array [h, w] / [h, w, 3] (B,G,R) or a list of equally sized ones.
        Returns per image (key points [n, 7] float32: x, y, size, angle, response, octave, class_id -- cv::KeyPoint's fields -- and
        descriptors [n, 32] uint8)."""
        single = isinstance(images, np.ndarray)
        imgs = [images] if single else list(images)
        imgs = [np.ascontiguousarray(im, np.uint8) for im in imgs]
        if not imgs:
            return []
        h, w = imgs[0].shape[:2]; ch = 1 if imgs[0].ndim == 2 else imgs[0].shape[2]
        if any(im.shape != imgs[0].shape for im in imgs):
            raise SfmB200Error("batched ORB extraction needs equally sized images")
        n = len(imgs)
        cap = int(capacity) if capacity is not None else int(nfeatures) + 64
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        while True:
            kp = np.zeros((n, max(cap, 1), 7), np.float32); desc = np.zeros((n, max(cap, 1), 32), np.uint8); cnt = np.zeros(n, np.int32)
            self._check(lib().sfmb200_orb_detect_and_compute_batch(self._h, ptrs, n, int(w), int(h), int(ch), C.c_size_t(0), int(nfeatures), cap,
                                                                   _p(kp, C.c_float), _p(desc, C.c_uint8), _p(cnt, C.c_int32)))
            if cnt.max(initial=0) <= cap:
                break
            cap = int(cnt.max())                      # ties at a selection threshold: more key points than asked for
        out = []
        for i in range(n):
            k = kp[i, :cnt[i]].copy()
            k[:, 5:7] = k[:, 5:7].view(np.int32).astype(np.float32)      # octave, class_id are int32 in the record
            out.append((k, desc[i, :cnt[i]].copy()))
        return out[0] if single else out

    def orb_prepare(self, images, nfeatures=5000, capacity=None):
        """Pre-marshalled form of orb_detect_and_compute for timing the C call itself: returns (call, kp, desc, cnt); call() runs
        sfmb200_orb_detect_and_compute_batch into the preallocated kp [n, cap, 7] (raw records) / desc [n, cap, 32] / cnt [n]."""
        imgs = [np.ascontiguousarray(im, np.uint8) for im in images]
        h, w = imgs[0].shape[:2]; ch = 1 if imgs[0].ndim == 2 else imgs[0].shape[2]
        n = len(imgs); cap = int(capacity) if capacity is not None else int(nfeatures) + 64
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        kp = np.zeros((n, cap, 7), np.float32); desc = np.zeros((n, cap, 32), np.uint8); cnt = np.zeros(n, np.int32)
        args = (self._h, ptrs, n, int(w), int(h), int(ch), C.c_size_t(0), int(nfeatures), cap, _p(kp, C.c_float), _p(desc, C.c_uint8), _p(cnt, C.c_int32))
        fn = lib().sfmb200_orb_detect_and_compute_batch

        def call(_keep=imgs):
            self._check(fn(*args))
            return cnt
        return call, kp, desc, cnt

    def orb_last_timings(self):
        """Host wall-clock (ms) of the phases of the last ORB call (sfmb200_orb_last_timings)."""
        ms = np.zeros(8)
        self._check(lib().sfmb200_orb_last_timings(self._h, _p(ms, C.c_double)))
        names = ("stage_upload_enqueue", "wait_detect", "candidates_d2h", "select_fast", "harris_roundtrip", "select_harris", "describe_roundtrip", "copy_out")
        return dict(zip(names, ms.tolist()))

    def orb_download_level(self, stage, image, level, w, h):
        out = np.zeros((h, w), np.uint8)
        self._check(lib().sfmb200_orb_download_level(self._h, int(stage), int(image), int(level), _p(out, C.c_uint8)))
        return out

    # ------------------------------------------------------------------ f-3 JPEG decoding
    @staticmethod
    def jpeg_info(data):
        """sfmb200_jpeg_info (host only): (status, width, height, components) of a JPEG file given as bytes."""
        return jpeg_info(data)

    def decode_jpeg(self, files, scale=1.0):
        """sfmb200_decode_jpeg_batch: `files` is a list of JPEG files as bytes; returns a list of uint8 [h, w, 3] B,G,R images,
        byte-identical to cv2.imdecode(buf, IMREAD_COLOR), in one call.  Raises SfmB200Error (naming the file) if any file is
        unsupported (status 5) or corrupt (status 1).  With scale != 1 (sfmb200_decode_jpeg_batch_scaled) every image is also
        downscaled on the device, byte-identical to cv2.resize(img, None, fx=scale, fy=scale), and only the resized images are
        downloaded."""
        files = [bytes(f) for f in files]
        n = len(files)
        scale = float(scale)
        if n == 0:
            return []
        outs = []
        for f in files:
            rc, w, h, _ = jpeg_info(f)
            if rc == 0 and scale != 1.0:
                w, h = resize_size(w, h, scale) or (1, 1)     # a refused scale fails the call below
            outs.append(np.empty((h, w, 3) if rc == 0 else (1, 1, 3), np.uint8))    # a failing file fails the call below
        data = (C.c_char_p * n)(*files)
        sizes = (C.c_size_t * n)(*[len(f) for f in files])
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        if scale == 1.0:
            self._check(lib().sfmb200_decode_jpeg_batch(self._h, data, sizes, n, ptrs, None))
        else:
            self._check(lib().sfmb200_decode_jpeg_batch_scaled(self._h, data, sizes, n, C.c_double(scale), ptrs, None))
        return outs

    def decode_jpeg_orb(self, files, scale=1.0, nfeatures=5000, capacity=None, images=True):
        """sfmb200_decode_jpeg_extract_orb: decode_jpeg(files, scale) and orb_detect_and_compute on every image in one call, with the
        images staying on the device in between; they may differ in size.  Returns (images or None, [(key points, descriptors), ...]):
        the images as decode_jpeg returns them when `images` is true (else they are not downloaded), and per image what
        orb_detect_and_compute returns for it.  A capacity below a key point count repeats the call with the count."""
        files = [bytes(f) for f in files]
        n = len(files)
        scale = float(scale)
        if n == 0:
            return ([] if images else None), []
        outs = None
        if images:
            outs = []
            for f in files:
                rc, w, h, _ = jpeg_info(f)
                if rc == 0 and scale != 1.0:
                    w, h = resize_size(w, h, scale) or (1, 1)     # a refused scale fails the call below
                outs.append(np.empty((h, w, 3) if rc == 0 else (1, 1, 3), np.uint8))
        data = (C.c_char_p * n)(*files)
        sizes = (C.c_size_t * n)(*[len(f) for f in files])
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs]) if images else None
        cap = int(capacity) if capacity is not None else int(nfeatures) + 64
        while True:
            kp = np.zeros((n, max(cap, 1), 7), np.float32); desc = np.zeros((n, max(cap, 1), 32), np.uint8); cnt = np.zeros(n, np.int32)
            self._check(lib().sfmb200_decode_jpeg_extract_orb(self._h, data, sizes, n, C.c_double(scale), int(nfeatures), cap,
                                                              _p(kp, C.c_float), _p(desc, C.c_uint8), _p(cnt, C.c_int32), ptrs, None))
            if cnt.max(initial=0) <= cap:
                break
            cap = int(cnt.max())                      # ties at a selection threshold: more key points than asked for
        feats = []
        for i in range(n):
            k = kp[i, :cnt[i]].copy()
            k[:, 5:7] = k[:, 5:7].view(np.int32).astype(np.float32)      # octave, class_id are int32 in the record
            feats.append((k, desc[i, :cnt[i]].copy()))
        return outs, feats

    def _image_outputs(self, files, scale):
        outs = []
        for f in files:
            rc, _, w, h = image_info(f)
            if rc == 0 and scale != 1.0:
                w, h = resize_size(w, h, scale) or (1, 1)     # a refused scale fails the call below
            outs.append(np.empty((h, w, 3) if rc == 0 else (1, 1, 3), np.uint8))    # a failing file fails the call below
        return outs

    def decode_images(self, files, scale=1.0):
        """sfmb200_decode_images: decode_jpeg for any mix of JPEG and PNG files (bytes), each byte-identical to
        cv2.imdecode(buf, IMREAD_COLOR), then resized as cv2.resize(img, None, fx=scale, fy=scale) when scale != 1."""
        files = [bytes(f) for f in files]
        n = len(files)
        scale = float(scale)
        if n == 0:
            return []
        outs = self._image_outputs(files, scale)
        data = (C.c_char_p * n)(*files)
        sizes = (C.c_size_t * n)(*[len(f) for f in files])
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        self._check(lib().sfmb200_decode_images(self._h, data, sizes, n, C.c_double(scale), ptrs, None))
        return outs

    def decode_images_orb(self, files, scale=1.0, nfeatures=5000, capacity=None, images=True):
        """sfmb200_decode_images_extract_orb: decode_jpeg_orb for any mix of JPEG and PNG files; same returns and capacity retry."""
        files = [bytes(f) for f in files]
        n = len(files)
        scale = float(scale)
        if n == 0:
            return ([] if images else None), []
        outs = self._image_outputs(files, scale) if images else None
        data = (C.c_char_p * n)(*files)
        sizes = (C.c_size_t * n)(*[len(f) for f in files])
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs]) if images else None
        cap = int(capacity) if capacity is not None else int(nfeatures) + 64
        while True:
            kp = np.zeros((n, max(cap, 1), 7), np.float32); desc = np.zeros((n, max(cap, 1), 32), np.uint8); cnt = np.zeros(n, np.int32)
            self._check(lib().sfmb200_decode_images_extract_orb(self._h, data, sizes, n, C.c_double(scale), int(nfeatures), cap,
                                                                _p(kp, C.c_float), _p(desc, C.c_uint8), _p(cnt, C.c_int32), ptrs, None))
            if cnt.max(initial=0) <= cap:
                break
            cap = int(cnt.max())                      # ties at a selection threshold: more key points than asked for
        feats = []
        for i in range(n):
            k = kp[i, :cnt[i]].copy()
            k[:, 5:7] = k[:, 5:7].view(np.int32).astype(np.float32)      # octave, class_id are int32 in the record
            feats.append((k, desc[i, :cnt[i]].copy()))
        return outs, feats

    def png_last_stats(self):
        """PNG counters of the last decode_images[_orb] call (sfmb200_png_last_stats)."""
        s = np.zeros(PNG_STATS, np.int64)
        self._check(lib().sfmb200_png_last_stats(self._h, _p(s, C.c_int64)))
        return dict(zip(("blocks", "speculative_blocks", "chain_blocks", "candidates", "rounds", "upload_bytes", "download_bytes", "groups",
                         "stored_blocks", "fixed_blocks"), s.tolist()))

    def resize_images(self, images, scale):
        """sfmb200_resize_batch: `images` is a list of uint8 [h, w, 3] B,G,R arrays (any sizes, strided rows allowed); returns them
        resized by `scale`, byte-identical to cv2.resize(img, None, fx=scale, fy=scale) (INTER_LINEAR), in one call.  A refused scale
        raises SfmB200Error (status 1)."""
        n = len(images)
        if n == 0:
            return []
        srcs, outs = [], []
        for im in images:
            im = np.asarray(im)
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError("resize_images: expects uint8 [h, w, 3] B,G,R images")
            if im.strides[1:] != (3, 1) or im.strides[0] < 3 * im.shape[1]:
                im = np.ascontiguousarray(im)                    # pixels packed B,G,R; rows may keep a longer stride
            srcs.append(im)
            h, w = im.shape[:2]
            dw, dh = resize_size(w, h, scale) or (1, 1)          # a refused scale fails the call below
            outs.append(np.empty((dh, dw, 3), np.uint8))
        ptr = (C.c_void_p * n)(*[s.ctypes.data for s in srcs])
        ws = (C.c_int * n)(*[s.shape[1] for s in srcs]); hs = (C.c_int * n)(*[s.shape[0] for s in srcs])
        strides = (C.c_size_t * n)(*[s.strides[0] for s in srcs])
        dptr = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        self._check(lib().sfmb200_resize_batch(self._h, ptr, ws, hs, strides, n, C.c_double(float(scale)), dptr, None))
        return outs

    def jpeg_last_stats(self):
        """Huffman-phase counters of the last decode_jpeg call (sfmb200_jpeg_last_stats)."""
        s = np.zeros(7, np.int64)
        self._check(lib().sfmb200_jpeg_last_stats(self._h, _p(s, C.c_int64)))
        return dict(zip(("subsequences", "codewords_first_pass", "codewords_sync", "rounds", "swept", "upload_bytes", "download_bytes"), s.tolist()))

    # ------------------------------------------------------------------ multi-GPU
    def comm_init(self, unique_id, rank, nranks):
        buf = (C.c_uint8 * UNIQUE_ID_BYTES).from_buffer_copy(bytes(unique_id)) if unique_id is not None else None
        self._check(lib().sfmb200_comm_init(self._h, buf, int(rank), int(nranks)))

    @property
    def comm_size(self):
        return lib().sfmb200_comm_size(self._h)


def orb_layout(width, height, nfeatures=5000):
    """Pyramid layout of the ORB stage (host-side, no GPU): level widths, heights, scales, key point quotas."""
    w = np.zeros(8, np.int32); h = np.zeros(8, np.int32); s = np.zeros(8, np.float32); q = np.zeros(8, np.int32)
    rc = lib().sfmb200_orb_layout(int(width), int(height), int(nfeatures), _p(w, C.c_int32), _p(h, C.c_int32), _p(s, C.c_float), _p(q, C.c_int32))
    if rc != 0:
        raise SfmB200Error(f"sfmb200_orb_layout failed ({rc})")
    return w, h, s, q


def orb_linear_exact_taps(src, dst):
    i0 = np.zeros(dst, np.int32); i1 = np.zeros(dst, np.int32); a = np.zeros(dst, np.int32)
    rc = lib().sfmb200_orb_linear_exact_taps(int(src), int(dst), _p(i0, C.c_int32), _p(i1, C.c_int32), _p(a, C.c_int32))
    if rc != 0:
        raise SfmB200Error(f"sfmb200_orb_linear_exact_taps failed ({rc})")
    return i0, i1, a


def orb_retain_best(response, n_points):
    r = np.ascontiguousarray(response, np.float32); order = np.zeros(max(len(r), 1), np.int32)
    n = lib().sfmb200_orb_retain_best(_p(r, C.c_float), len(r), int(n_points), _p(order, C.c_int32))
    if n < 0:
        raise SfmB200Error("sfmb200_orb_retain_best: bad arguments")
    return order[:n].copy()


def jpeg_info(data):
    """sfmb200_jpeg_info: (status, width, height, components) of a JPEG file given as bytes, without a context or a GPU.  width and
    height are the decoded image's (after EXIF orientation); status 0 = decodable, 1 = invalid, 5 = unsupported."""
    data = bytes(data)
    w = C.c_int(0); h = C.c_int(0); c = C.c_int(0)
    rc = lib().sfmb200_jpeg_info(C.c_char_p(data), C.c_size_t(len(data)), C.byref(w), C.byref(h), C.byref(c))
    return int(rc), w.value, h.value, c.value


FORMAT_JPEG, FORMAT_PNG = 1, 2
PNG_STATS = 10
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def image_info(data):
    """sfmb200_image_info: (status, format, width, height) of a JPEG or PNG file given as bytes, without a context or a GPU.  format is
    FORMAT_JPEG or FORMAT_PNG; width and height are the decoded image's (after EXIF orientation); status 0 = decodable, 1 = invalid
    (also for a file that is neither JPEG nor PNG), 5 = unsupported."""
    data = bytes(data)
    f = C.c_int(0); w = C.c_int(0); h = C.c_int(0)
    rc = lib().sfmb200_image_info(C.c_char_p(data), C.c_size_t(len(data)), C.byref(f), C.byref(w), C.byref(h))
    return int(rc), f.value, w.value, h.value


def resize_size(width, height, scale):
    """sfmb200_resize_size: (width, height) of cv2.resize(img, None, fx=scale, fy=scale) for a width x height image, without a
    context or a GPU; None where cv::resize refuses (scale not finite or <= 0, or no pixels left)."""
    w = C.c_int(0); h = C.c_int(0)
    rc = lib().sfmb200_resize_size(int(width), int(height), C.c_double(float(scale)), C.byref(w), C.byref(h))
    return (w.value, h.value) if rc == 0 else None


def comm_unique_id():
    buf = (C.c_uint8 * UNIQUE_ID_BYTES)()
    rc = lib().sfmb200_comm_unique_id(buf)
    if rc != 0:
        raise SfmB200Error(f"sfmb200_comm_unique_id failed ({rc}): {lib().sfmb200_last_error(None).decode()}")
    return bytes(buf)


def ba_default_options(**kw):
    o = BAOptions()
    lib().sfmb200_ba_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def essential_default_options(**kw):
    o = EssentialOptions()
    lib().sfmb200_essential_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def pose_default_options(**kw):
    o = PoseOptions()
    lib().sfmb200_pose_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def homography_default_options(**kw):
    o = HomographyOptions()
    lib().sfmb200_homography_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def ba_validate(nc, obs_cam, pt_off):
    """sfmb200_ba_validate: host-only check of a flattened problem.  Returns (status, message); status 0 = valid."""
    obs_cam = np.ascontiguousarray(obs_cam, np.int32); pt_off = np.ascontiguousarray(pt_off, np.int32)
    msg = C.create_string_buffer(200)
    f = lib().sfmb200_ba_validate
    f.restype = C.c_int
    rc = f(C.c_int(int(nc)), C.c_int(max(0, pt_off.shape[0] - 1)), C.c_int(obs_cam.shape[0]), _p(obs_cam, C.c_int32), _p(pt_off, C.c_int32), msg, C.c_int(200))
    return int(rc), msg.value.decode()


def rotmat_to_angle_axis_f32(R):
    R = np.ascontiguousarray(R, np.float32).reshape(9); aa = np.empty(3, np.float32)
    lib().sfmb200_rotmat_to_angle_axis_f32(_p(R, C.c_float), _p(aa, C.c_float))
    return aa


def angle_axis_to_rotmat(aa):
    aa = np.ascontiguousarray(aa, np.float64).reshape(3); R = np.empty(9, np.float64)
    lib().sfmb200_angle_axis_to_rotmat(_p(aa, C.c_double), _p(R, C.c_double))
    return R.reshape(3, 3)


class DescriptorSet:
    """sfmb200_descset: the descriptors of all images resident in HBM; all-pairs matching in one call."""

    @classmethod
    def from_packed(cls, ctx, allrows, sizes, norm="hamming"):
        """Rows of all images already concatenated (what a C++ host hands to sfmb200_descset_create): no per-call numpy copy."""
        self = cls.__new__(cls)
        self.ctx = ctx; self.norm = norm; self.sizes = [int(x) for x in sizes]
        off = np.zeros(len(self.sizes) + 1, np.int32); off[1:] = np.cumsum(self.sizes)
        self._h = C.c_void_p()
        if norm == "hamming":
            ctx._check(lib().sfmb200_descset_create(ctx._h, _p(allrows, C.c_uint8), _p(off, C.c_int32), len(self.sizes), allrows.shape[1], C.byref(self._h)))
        else:
            ctx._check(lib().sfmb200_descset_create_l2(ctx._h, _p(allrows, C.c_float), _p(off, C.c_int32), len(self.sizes), allrows.shape[1], C.byref(self._h)))
        ctx._adopt(self)
        return self

    def __init__(self, ctx, desc_list, norm="hamming"):
        """norm="hamming": uint8 rows (ORB; the reference's case).  norm="l2": float32 rows with integer values in [0, 255] and
        dim <= 128 (SIFT): exact u8 GEMM on the tensor cores, distances like cv2.BFMatcher(NORM_L2)."""
        self.ctx = ctx
        self.norm = norm
        dt = np.uint8 if norm == "hamming" else np.float32
        desc_list = [np.ascontiguousarray(d, dt) for d in desc_list]
        self.sizes = [d.shape[0] for d in desc_list]
        nb = desc_list[0].shape[1] if desc_list else 32
        off = np.zeros(len(desc_list) + 1, np.int32); off[1:] = np.cumsum(self.sizes)
        allrows = np.ascontiguousarray(np.concatenate(desc_list, 0)) if desc_list else np.zeros((0, nb), dt)
        self._h = C.c_void_p()
        if norm == "hamming":
            ctx._check(lib().sfmb200_descset_create(ctx._h, _p(allrows, C.c_uint8), _p(off, C.c_int32), len(desc_list), nb, C.byref(self._h)))
        else:
            ctx._check(lib().sfmb200_descset_create_l2(ctx._h, _p(allrows, C.c_float), _p(off, C.c_int32), len(desc_list), nb, C.byref(self._h)))
        ctx._adopt(self)

    def close(self):
        if self._h:
            lib().sfmb200_descset_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def match_pairs(self, pairs, ratio=RATIO_REFERENCE):
        """pairs: [(left, right), ...] -> list of (queryIdx, trainIdx, distance) per pair."""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        npairs = pairs.shape[0]
        total = int(sum(self.sizes[l] for l, _ in pairs))
        oq = np.empty(max(total, 1), np.int32); ot = np.empty(max(total, 1), np.int32); od = np.empty(max(total, 1), np.float32)
        off = np.zeros(npairs + 1, np.int64); cnt = np.zeros(max(npairs, 1), np.int32)
        self.ctx._check(lib().sfmb200_match_pairs(self.ctx._h, self._h, _p(pairs, C.c_int32), npairs, C.c_double(ratio),
                                                  _p(oq, C.c_int32), _p(ot, C.c_int32), _p(od, C.c_float), _p(off, C.c_int64), _p(cnt, C.c_int32)))
        return [(oq[off[p]:off[p] + cnt[p]], ot[off[p]:off[p] + cnt[p]], od[off[p]:off[p] + cnt[p]]) for p in range(npairs)]   # views

    def match_pairs_prepare(self, pairs, ratio=RATIO_REFERENCE, buffers=None):
        """Pre-marshalled sfmb200_match_pairs for timing the C call itself: caller-owned result buffers (touched once), no per-call numpy work.
        Returns (call, buffers); call() -> (off, cnt); buffers = (oq, ot, od, off, cnt) can be handed to another set of the same sizes."""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        npairs = pairs.shape[0]
        if buffers is None:
            total = int(sum(self.sizes[l] for l, _ in pairs))
            buffers = (np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.float32),
                       np.zeros(npairs + 1, np.int64), np.zeros(max(npairs, 1), np.int32))
        oq, ot, od, off, cnt = buffers
        args = (self.ctx._h, self._h, _p(pairs, C.c_int32), npairs, C.c_double(ratio), _p(oq, C.c_int32), _p(ot, C.c_int32), _p(od, C.c_float),
                _p(off, C.c_int64), _p(cnt, C.c_int32))
        fn = lib().sfmb200_match_pairs

        def call(_keep=(pairs,)):
            self.ctx._check(fn(*args))
            return off, cnt
        return call, buffers

    def match_pairs_device(self, pairs, d_q, d_t, d_d, d_pair_start, d_total, ratio=RATIO_REFERENCE):
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        self.ctx._check(lib().sfmb200_match_pairs_device(self.ctx._h, self._h, _p(pairs, C.c_int32), pairs.shape[0], C.c_double(ratio),
                                                         _vp(d_q), _vp(d_t), _vp(d_d), _vp(d_pair_start), _vp(d_total)))


class BAProblem:
    """sfmb200_ba_problem: a flattened adjustBundle problem resident in HBM."""

    def __init__(self, ctx, cams, pts, focal, obs_xy, obs_cam, pt_off):
        self.ctx = ctx
        cams = np.ascontiguousarray(cams, np.float64).reshape(-1, 6); pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        obs_xy = np.ascontiguousarray(obs_xy, np.float32).reshape(-1, 2); obs_cam = np.ascontiguousarray(obs_cam, np.int32)
        pt_off = np.ascontiguousarray(pt_off, np.int32)
        self.nc, self.np, self.nobs = cams.shape[0], pts.shape[0], obs_cam.shape[0]
        self._h = C.c_void_p()
        ctx._check(lib().sfmb200_ba_problem_create(ctx._h, self.nc, self.np, self.nobs, _p(cams, C.c_double), _p(pts, C.c_double),
                                                   C.c_double(float(focal)), _p(obs_xy, C.c_float), _p(obs_cam, C.c_int32),
                                                   _p(pt_off, C.c_int32), C.byref(self._h)))
        ctx._adopt(self)

    def close(self):
        if self._h:
            lib().sfmb200_ba_problem_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def ipc_handle(self):
        buf = (C.c_uint8 * 64)()
        self.ctx._check(lib().sfmb200_ba_problem_ipc_handle(self._h, buf))
        return bytes(buf)

    def ipc_attach(self, handles):
        blob = b"".join(handles)
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        self.ctx._check(lib().sfmb200_ba_problem_ipc_attach(self._h, buf))

    def reset(self):
        self.ctx._check(lib().sfmb200_ba_problem_reset(self._h))

    def run(self, options=None):
        s = BASummary(); o = options or ba_default_options()
        self.ctx._check(lib().sfmb200_ba_problem_run(self._h, C.byref(o), C.byref(s)))
        return s.as_dict()

    def download(self):
        cams = np.empty((self.nc, 6)); pts = np.empty((self.np, 3)); f = C.c_double()
        self.ctx._check(lib().sfmb200_ba_problem_download(self._h, _p(cams, C.c_double), _p(pts, C.c_double), C.byref(f)))
        return cams, pts, f.value

    def reduced_system(self, radius=1e4, options=None):
        n = 6 * self.nc + 1
        S = np.empty((n, n)); rhs = np.empty(n); g = np.empty(n); cost = C.c_double()
        o = options or ba_default_options()
        self.ctx._check(lib().sfmb200_ba_problem_reduced_system(self._h, C.byref(o), C.c_double(radius), _p(S, C.c_double),
                                                                _p(rhs, C.c_double), _p(g, C.c_double), C.byref(cost)))
        return dict(S=S, rhs=rhs, grad_cf=g, cost=cost.value)
