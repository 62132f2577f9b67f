"""The image-pair batch layout shared by sfmb200_triangulate_pairs, sfmb200_find_camera_matrices_pairs and
sfmb200_find_homography_pairs (include/sfmb200.h, "image-pair batches"): every refusal of the shared host-side check for each of
the three calls, after which the context returns the same outputs as before; the empty batch; and triangulation's NULL
arguments around the shared check."""
import ctypes as C

import numpy as np
import pytest

from essential_util import CX, CY, F, synthetic_scene
from sfm_toy_library_b200 import capi

pytestmark = pytest.mark.gpu
CALLS = ("triangulate", "essential", "homography")
K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float32)
A, B, R, T, _ = synthetic_scene(5, 60)                      # two images of 60 key points, the second seen from [R|t]
POSE = np.r_[np.eye(3, 4).ravel(), np.c_[R, T].ravel()].astype(np.float32)      # (Pleft, Pright) of every pair
IDX = np.arange(60)
GOOD = dict(img_off=[0, 60, 120], pairs=[(0, 1)], mq=IDX, mt=IDX, moff=[0, 60])
BAD = [(dict(pairs=[(0, 2)]), "outside \\[0, 2\\)"),
       (dict(pairs=[(-1, 1)]), "outside \\[0, 2\\)"),
       (dict(img_off=[0, 70, 60]), "img_off is not monotone"),
       (dict(img_off=[1, 60, 120]), "img_off\\[0\\] must be 0"),
       (dict(pairs=[(0, 1), (0, 1)], moff=[0, 60, 30]), "match_off is not monotone"),
       (dict(moff=[5, 60]), "match_off\\[0\\] must be 0"),
       (dict(mq=np.r_[IDX[:59], 60]), "indexes outside its images"),
       (dict(mt=np.r_[-1, IDX[1:]]), "indexes outside its images")]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _raw(ctx, call, img_off, pairs, mq, mt, moff, null=()):
    """One of the three C calls on A and B with the caller's own img_off (the binding derives img_off from the images), default
    options and POSE for every pair.  Triangulation passes NULL for the arguments named in `null` (K, poses, X, keep, n_keep).
    Returns the outputs; the summaries as int32 rows, n_keep as None when it was NULL."""
    allp = np.ascontiguousarray(np.r_[A, B], np.float32); img_off = np.asarray(img_off, np.int32)
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2); mq = np.asarray(mq, np.int32); mt = np.asarray(mt, np.int32)
    moff = np.asarray(moff, np.int64)
    P, M = len(pairs), len(mq)
    ptr = lambda x, tp: x.ctypes.data_as(C.POINTER(tp))
    batch = (ptr(allp, C.c_float), ptr(img_off, C.c_int32), len(img_off) - 1, ptr(pairs, C.c_int32), P, ptr(mq, C.c_int32),
             ptr(mt, C.c_int32), ptr(moff, C.c_int64))
    rows = lambda s: np.frombuffer(bytes(s), np.int32).reshape(len(s), -1)[:P]
    L = capi.lib()
    if call == "triangulate":
        poses = np.ascontiguousarray(np.tile(POSE, (P, 1)))
        X = np.full((max(M, 1), 3), np.nan, np.float32); keep = np.full(max(M, 1), 7, np.uint8); nk = np.full(max(P, 1), -1, np.int32)
        a = dict(K=ptr(K, C.c_float), poses=ptr(poses, C.c_float), X=ptr(X, C.c_float), keep=ptr(keep, C.c_uint8), n_keep=ptr(nk, C.c_int32))
        a.update(dict.fromkeys(null))
        ctx._check(L.sfmb200_triangulate_pairs(ctx._h, a["K"], a["poses"], *batch, C.c_float(10.0), a["X"], a["keep"], a["n_keep"]))
        return X[:M], keep[:M], (None if "n_keep" in null else nk[:P])
    if call == "essential":
        E = np.zeros((max(P, 1), 9)); Rm = np.zeros((max(P, 1), 9)); t = np.zeros((max(P, 1), 3))
        inl = np.zeros(max(M, 1), np.uint8); pm = np.zeros(max(M, 1), np.uint8); s = (capi.EssentialSummary * max(P, 1))()
        o = capi.essential_default_options()
        ctx._check(L.sfmb200_find_camera_matrices_pairs(ctx._h, ptr(K, C.c_float), *batch, C.byref(o), ptr(E, C.c_double), ptr(Rm, C.c_double),
                                                        ptr(t, C.c_double), ptr(inl, C.c_uint8), ptr(pm, C.c_uint8), s))
        return E[:P], Rm[:P], t[:P], inl[:M], pm[:M], rows(s)
    H = np.zeros((max(P, 1), 9)); mask = np.zeros(max(M, 1), np.uint8); s = (capi.HomographySummary * max(P, 1))()
    o = capi.homography_default_options()
    ctx._check(L.sfmb200_find_homography_pairs(ctx._h, *batch, C.byref(o), ptr(H, C.c_double), ptr(mask, C.c_uint8), s))
    return H[:P], mask[:M], rows(s)


@pytest.mark.parametrize("call", CALLS)
def test_invalid_inputs_are_refused_and_the_context_stays_usable(ctx, call):
    ref = _raw(ctx, call, **GOOD)
    if call == "triangulate":                       # a batch of one pair is the single call
        X1, keep1, nk1 = ctx.triangulate(K, POSE[:12], POSE[12:], A, B, IDX, IDX)
        np.testing.assert_array_equal(ref[0], X1); np.testing.assert_array_equal(ref[1], keep1); assert ref[2][0] == nk1
    if call == "essential":
        assert ref[5][0][0] == 1                    # summary[0].found
    for change, msg in BAD:
        with pytest.raises(capi.SfmB200Error, match=msg):
            _raw(ctx, call, **{**GOOD, **change})
        for x, y in zip(_raw(ctx, call, **GOOD), ref):
            np.testing.assert_array_equal(x, y, err_msg=msg)


@pytest.mark.parametrize("call", CALLS)
def test_empty_batch(ctx, call):
    """n_pairs == 0 returns no outputs; only the homography call still checks img_off then"""
    empty = dict(img_off=[0, 60, 120], pairs=np.zeros((0, 2)), mq=np.zeros(0), mt=np.zeros(0), moff=[0])
    assert all(len(x) == 0 for x in _raw(ctx, call, **empty))
    bad_off = {**empty, "img_off": [1, 60, 120]}
    if call == "homography":
        with pytest.raises(capi.SfmB200Error, match="img_off\\[0\\] must be 0"):
            _raw(ctx, call, **bad_off)
    else:
        assert all(len(x) == 0 for x in _raw(ctx, call, **bad_off))


def test_triangulate_without_n_keep(ctx):
    """n_keep = NULL: the same X and keep"""
    args = dict(img_off=[0, 60, 120], pairs=[(0, 1), (1, 0), (0, 1)], mq=np.r_[IDX, IDX[::-2]], mt=np.r_[IDX, IDX[::-2]], moff=[0, 60, 60, 90])
    X, keep, nk = _raw(ctx, "triangulate", **args)
    assert nk[1] == 0 and nk[0] > 0
    X0, keep0, nk0 = _raw(ctx, "triangulate", **args, null=("n_keep",))
    assert nk0 is None
    np.testing.assert_array_equal(X0, X); np.testing.assert_array_equal(keep0, keep)


def test_triangulate_refuses_null_arguments(ctx):
    """K, poses, and X and keep when there are matches: the checks triangulation makes around the shared one"""
    ref = _raw(ctx, "triangulate", **GOOD)
    for arg in ("K", "poses", "X", "keep"):
        with pytest.raises(capi.SfmB200Error, match="null buffer"):
            _raw(ctx, "triangulate", **GOOD, null=(arg,))
        for x, y in zip(_raw(ctx, "triangulate", **GOOD), ref):
            np.testing.assert_array_equal(x, y, err_msg=arg)
    empty = dict(GOOD, mq=IDX[:0], mt=IDX[:0], moff=[0, 0])
    assert _raw(ctx, "triangulate", **empty, null=("X", "keep"))[2].tolist() == [0]      # no matches: X and keep may be NULL
