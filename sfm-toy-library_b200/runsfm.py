"""Host-side mirror (Python) of the reference's driver `sfmtoylib::SfM` (SfMToyLib/SfM.h:46-145, SfM.cpp:63-629).

The C++ product driver is host/ (shim.cpp + sfm_glue.cpp behind the reference's own SfM.cpp); it needs C++ OpenCV for the
RANSAC stages, which this image does not have.  This file is the same control flow in Python so that BASELINE configs[0]
(crazyhorse, 7 images) can be run stage by stage in this image and on the GPU box:

  * the three hot-path stages are injected as callables with the reference's names and argument order
    (`matchFeatures`, `triangulateViews`, `adjustBundle`; default = stages.py over the C ABI);
  * the RANSAC stages that SURVEY.md 8 marks "next" (f-2) are the reference's own OpenCV calls through cv2
    (SfMStereoUtilities.cpp:51-118, 208-243), or the batched-scoring versions of `ransac.py` when injected;
  * find2D3DMatches / mergeNewPointCloud keep the reference's first-hit-in-list-order semantics (SfM.cpp:471-600) through
    per-pair first-occurrence maps -- the Python twin of host/sfm_glue.cpp.

`trace` (optional list) receives one dict per stage call with the inputs and outputs of the call, which is what
tests/golden/make_cfg1.py stores and tests/test_gpu_cfg1.py replays call by call.
"""
import time
from typing import Callable, Dict, List, Optional

import numpy as np

from . import stages
from .stages import DMATCH, Features, ImagePair, Intrinsics, Point3DInMap

MERGE_CLOUD_POINT_MIN_MATCH_DISTANCE = float(np.float32(0.01))      # SfM.cpp:50 (const float)
MERGE_CLOUD_FEATURE_MIN_MATCH_DISTANCE = np.float32(20.0)           # SfM.cpp:51
MIN_POINT_COUNT_FOR_HOMOGRAPHY = 100                                # SfM.cpp:52
POSE_INLIERS_MINIMAL_RATIO = 0.5                                    # SfMCommon.h:53
RANSAC_THRESHOLD = 10.0                                             # SfMStereoUtilities.cpp:41


# ------------------------------------------------------------------------------------------------ RANSAC stages (cv2)
def findHomographyInliers_cv2(left: Features, right: Features, matches: np.ndarray) -> int:
    """SfMStereoUtilities::findHomographyInliers (SfMStereoUtilities.cpp:51-72)."""
    import cv2
    if len(matches) < 4:
        return 0
    pl = left.points[matches["queryIdx"]]; pr = right.points[matches["trainIdx"]]
    H, mask = cv2.findHomography(pl, pr, cv2.RANSAC, RANSAC_THRESHOLD)
    if H is None:
        return 0
    return int(np.count_nonzero(mask))


def findCameraMatricesFromMatch_cv2(intrinsics: Intrinsics, matches: np.ndarray, left: Features, right: Features):
    """SfMStereoUtilities::findCameraMatricesFromMatch (SfMStereoUtilities.cpp:74-118).
    Returns (success, prunedMatches, Pleft, Pright)."""
    import cv2
    K = intrinsics.K
    focal = float(K[0, 0]); pp = (float(K[0, 2]), float(K[1, 2]))
    pl = left.points[matches["queryIdx"]]; pr = right.points[matches["trainIdx"]]
    E, mask = cv2.findEssentialMat(pl, pr, focal, pp, cv2.RANSAC, 0.999, 1.0)
    _, R, t, mask = cv2.recoverPose(E, pl, pr, focal=focal, pp=pp, mask=mask)
    Pleft = np.eye(3, 4, dtype=np.float32)
    Pright = np.concatenate([R, t.reshape(3, 1)], 1).astype(np.float32)
    pruned = matches[mask.reshape(-1) != 0].copy()
    return True, pruned, Pleft, Pright


def findCameraPoseFrom2D3DMatch_cv2(intrinsics: Intrinsics, points2D: np.ndarray, points3D: np.ndarray):
    """SfMStereoUtilities::findCameraPoseFrom2D3DMatch (SfMStereoUtilities.cpp:208-243).  Returns (success, pose 3x4 float32)."""
    import cv2
    ok, rvec, tvec, inliers = cv2.solvePnPRansac(points3D.reshape(-1, 1, 3), points2D.reshape(-1, 1, 2), intrinsics.K,
                                                 np.zeros((1, 4), np.float32), None, None, False, 100, RANSAC_THRESHOLD, 0.99)
    n_in = 0 if inliers is None else len(inliers)
    if np.float32(n_in) / np.float32(len(points2D)) < POSE_INLIERS_MINIMAL_RATIO:
        return False, None
    Rm, _ = cv2.Rodrigues(rvec)
    pose = np.zeros((3, 4), np.float32)
    pose[:, :3] = Rm.astype(np.float32); pose[:, 3] = tvec.reshape(3).astype(np.float32)
    return True, pose


# ------------------------------------------------------------------------------------------------ first-hit match index
class _PairIndex:
    """First occurrence per queryIdx / trainIdx of one match list: what the linear scans with `break` return
    (SfM.cpp:498-516, :566-575)."""

    def __init__(self, m: np.ndarray):
        self.m = m
        self.q_first: Dict[int, int] = {}
        self.t_first: Dict[int, int] = {}
        self.qt: Dict[tuple, List[int]] = {}
        for pos in range(len(m)):
            q = int(m["queryIdx"][pos]); t = int(m["trainIdx"][pos])
            self.q_first.setdefault(q, pos); self.t_first.setdefault(t, pos)
            self.qt.setdefault((q, t), []).append(pos)


class SfM:
    """sfmtoylib::SfM (SfM.h:46-145) with the image container replaced by pre-extracted Features (extraction is row f-3)."""

    def __init__(self, features: List[Features], image_size, *, matchFeatures: Callable = None, triangulateViews: Callable = None,
                 adjustBundle: Callable = None, matchAllPairs: Callable = None, findHomographyInliers: Callable = None,
                 findCameraMatricesFromMatch: Callable = None, findCameraPoseFrom2D3DMatch: Callable = None,
                 homographyInliersAllPairs: Callable = None, trace: Optional[list] = None, verbose: bool = False):
        self.mImageFeatures = features
        self.n = len(features)
        w, h = image_size
        # SfM.cpp:70-72 (integer division of cols/rows)
        self.mIntrinsics = Intrinsics(K=np.array([[2500, 0, w // 2], [0, 2500, h // 2], [0, 0, 1]], np.float32))
        self.mCameraPoses = [np.zeros((3, 4), np.float32) for _ in range(self.n)]
        self.mFeatureMatchMatrix = [[np.zeros(0, DMATCH) for _ in range(self.n)] for _ in range(self.n)]
        self.mReconstructionCloud: List[Point3DInMap] = []
        self.mDoneViews = set(); self.mGoodViews = set()
        self.matchFeatures = matchFeatures or stages.matchFeatures
        self.matchAllPairs = matchAllPairs
        self.triangulateViews = triangulateViews or stages.triangulateViews
        self.adjustBundle = adjustBundle or stages.adjustBundle
        self.findHomographyInliers = findHomographyInliers or findHomographyInliers_cv2
        self.homographyInliersAllPairs = homographyInliersAllPairs
        self.findCameraMatricesFromMatch = findCameraMatricesFromMatch or findCameraMatricesFromMatch_cv2
        self.findCameraPoseFrom2D3DMatch = findCameraPoseFrom2D3DMatch or findCameraPoseFrom2D3DMatch_cv2
        self.trace = trace
        self.verbose = verbose
        self.seconds = {"match": 0.0, "homography": 0.0, "essential": 0.0, "triangulate": 0.0, "bundle": 0.0, "pnp": 0.0, "glue": 0.0}
        self.calls = {k: 0 for k in self.seconds}

    @classmethod
    def from_images(cls, images, extractAllFeatures: Callable = None, **kw):
        """setImagesDirectory + extractFeatures of the reference driver (SfM.cpp:97-139, 141-154) for already decoded images
        (uint8 B,G,R or grey, equal sizes): ORB(5000) per image through the injected stage (default: stages.extractAllFeatures, GPU)."""
        t0 = time.perf_counter()
        feats = (extractAllFeatures or stages.extractAllFeatures)(list(images))
        dt = time.perf_counter() - t0
        h, w = images[0].shape[:2]
        sfm = cls(feats, (w, h), **kw)
        sfm.seconds["extract"] = dt; sfm.calls["extract"] = len(images)
        return sfm

    @classmethod
    def from_directory(cls, path, readImages: Callable = None, extractAllFeatures: Callable = None, **kw):
        """SfM::setImagesDirectory (SfM.cpp:97-139): the .jpg / .png files of `path` (extension compared case-insensitively), sorted
        by name, read by the injected stage (default cv2.imread per file; stages.readImages decodes them all on the device), then
        from_images.  The reference's optional downscale (:127-129) is not applied."""
        import os
        names = sorted(f for f in os.listdir(path) if os.path.splitext(f)[1].lower() in (".jpg", ".png"))
        if not names:
            raise ValueError(f"Unable to find valid files in images directory (\"{path}\").")
        files = [os.path.join(path, f) for f in names]
        t0 = time.perf_counter()
        if readImages is None:
            import cv2
            images = [cv2.imread(f) for f in files]
        else:
            images = list(readImages(files))
        dt = time.perf_counter() - t0
        for f, im in zip(files, images):
            if im is None or im.size == 0:
                raise ValueError(f"Unable to read image from file: {f}")
        sfm = cls.from_images(images, extractAllFeatures, **kw)
        sfm.seconds["read"] = dt; sfm.calls["read"] = len(files)
        return sfm

    # ---- timing helper
    def _timed(self, key, fn, *a, **kw):
        t0 = time.perf_counter()
        r = fn(*a, **kw)
        self.seconds[key] += time.perf_counter() - t0; self.calls[key] += 1
        return r

    def runSfM(self):
        """SfM::runSfM (SfM.cpp:63-95) after extractFeatures."""
        self.createFeatureMatchMatrix()
        self.findBaselineTriangulation()
        self.addMoreViewsToReconstruction()
        return 0

    def createFeatureMatchMatrix(self):
        """SfM.cpp:157-212: all i<j pairs.  The reference fans the pairs out over threads; `matchAllPairs`, when given, is the
        batched all-pairs call (one launch sequence), else the per-pair function is called in pair order."""
        pairs = [(i, j) for i in range(self.n) for j in range(i + 1, self.n)]
        if self.matchAllPairs is not None:
            res = self._timed("match", self.matchAllPairs, self.mImageFeatures, pairs)
            for (i, j), m in zip(pairs, res):
                self.mFeatureMatchMatrix[i][j] = m
        else:
            for (i, j) in pairs:
                self.mFeatureMatchMatrix[i][j] = self._timed("match", self.matchFeatures, self.mImageFeatures[i], self.mImageFeatures[j])
        if self.trace is not None:
            self.trace.append({"stage": "match", "pairs": pairs, "matches": [self.mFeatureMatchMatrix[i][j].copy() for i, j in pairs]})

    def sortViewsForBaseline(self):
        """SfM.cpp:333-364: std::map<float, ImagePair> keyed by the homography inlier ratio (later pairs overwrite equal keys).
        `homographyInliersAllPairs`, when given, counts the inliers of every pair with enough matches in one batched call
        (features, pairs, matches) -> counts; else the per-pair function is called in pair order."""
        sizes: Dict[float, tuple] = {}
        batched = {}
        if self.homographyInliersAllPairs is not None:
            todo = [(i, j) for i in range(self.n - 1) for j in range(i + 1, self.n)
                    if len(self.mFeatureMatchMatrix[i][j]) >= MIN_POINT_COUNT_FOR_HOMOGRAPHY]
            counts = self._timed("homography", self.homographyInliersAllPairs, self.mImageFeatures, todo,
                                 [self.mFeatureMatchMatrix[i][j] for i, j in todo])
            batched = {pr: int(c) for pr, c in zip(todo, counts)}
        for i in range(self.n - 1):
            for j in range(i + 1, self.n):
                m = self.mFeatureMatchMatrix[i][j]
                if len(m) < MIN_POINT_COUNT_FOR_HOMOGRAPHY:
                    sizes[np.float32(1.0)] = (i, j)
                    continue
                if self.homographyInliersAllPairs is not None:
                    n_in = batched[(i, j)]
                else:
                    n_in = self._timed("homography", self.findHomographyInliers, self.mImageFeatures[i], self.mImageFeatures[j], m)
                ratio = np.float32(n_in) / np.float32(len(m))
                sizes[ratio] = (i, j)
                if self.trace is not None:
                    self.trace.append({"stage": "homography", "pair": (i, j), "inliers": n_in, "matches": len(m)})
        return sorted(sizes.items(), key=lambda kv: kv[0])

    def findBaselineTriangulation(self):
        """SfM.cpp:215-321."""
        for ratio, (i, j) in self.sortViewsForBaseline():
            ok, pruned, Pl, Pr = self._timed("essential", self.findCameraMatricesFromMatch, self.mIntrinsics,
                                             self.mFeatureMatchMatrix[i][j], self.mImageFeatures[i], self.mImageFeatures[j])
            if not ok:
                continue
            if np.float32(len(pruned)) / np.float32(len(self.mFeatureMatchMatrix[i][j])) < POSE_INLIERS_MINIMAL_RATIO:
                continue
            self.mFeatureMatchMatrix[i][j] = pruned
            cloud: List[Point3DInMap] = []
            ok = self._triangulate(i, j, Pl, Pr, cloud)
            if not ok:
                continue
            self.mReconstructionCloud = cloud
            self.mCameraPoses[i] = Pl.copy(); self.mCameraPoses[j] = Pr.copy()
            self.mDoneViews |= {i, j}; self.mGoodViews |= {i, j}
            self.adjustCurrentBundle()
            break

    def _triangulate(self, i, j, Pl, Pr, cloud):
        n0 = len(cloud)
        ok = self._timed("triangulate", self.triangulateViews, self.mIntrinsics, ImagePair(i, j), self.mFeatureMatchMatrix[i][j],
                         self.mImageFeatures[i], self.mImageFeatures[j], Pl, Pr, cloud)
        if self.trace is not None:
            self.trace.append({"stage": "triangulate", "pair": (i, j), "K": self.mIntrinsics.K.copy(), "Pl": np.array(Pl, np.float32),
                               "Pr": np.array(Pr, np.float32), "matches": self.mFeatureMatchMatrix[i][j].copy(),
                               "X": np.array([p.p for p in cloud[n0:]], np.float32).reshape(-1, 3),
                               "back": np.array([[p.originatingViews[i], p.originatingViews[j]] for p in cloud[n0:]], np.int32).reshape(-1, 2)})
        return ok

    def adjustCurrentBundle(self):
        """SfM.cpp:324-330."""
        if self.trace is not None:
            before = stages.flatten_bundle(self.mReconstructionCloud, self.mCameraPoses, self.mIntrinsics, self.mImageFeatures)
        summary = self._timed("bundle", self.adjustBundle, self.mReconstructionCloud, self.mCameraPoses, self.mIntrinsics, self.mImageFeatures)
        if self.trace is not None:
            cams, pts, focal, obs_xy, obs_cam, pt_off, used = before
            self.trace.append({"stage": "bundle", "cams": cams, "pts": pts, "focal": focal, "obs_xy": obs_xy, "obs_cam": obs_cam,
                               "pt_off": pt_off, "used": np.array(used, np.int32), "summary": summary,
                               "K_after": self.mIntrinsics.K.copy(),
                               "poses_after": np.array([self.mCameraPoses[v] for v in used], np.float32),
                               "pts_after": np.array([p.p for p in self.mReconstructionCloud], np.float32).reshape(-1, 3)})
        return summary

    def find2D3DMatches(self):
        """SfM.cpp:471-528."""
        t0 = time.perf_counter()
        index = {}
        out = {}
        for view in range(self.n):
            if view in self.mDoneViews:
                continue
            p2, p3 = [], []
            for cp in self.mReconstructionCloud:
                for oview in sorted(cp.originatingViews):
                    ofeat = cp.originatingViews[oview]
                    l, r = (oview, view) if oview < view else (view, oview)
                    idx = index.get((l, r))
                    if idx is None:
                        idx = index[(l, r)] = _PairIndex(self.mFeatureMatchMatrix[l][r])
                    if oview < view:
                        pos = idx.q_first.get(ofeat, -1)
                        hit = int(idx.m["trainIdx"][pos]) if pos >= 0 else -1
                    else:
                        pos = idx.t_first.get(ofeat, -1)
                        hit = int(idx.m["queryIdx"][pos]) if pos >= 0 else -1
                    if hit >= 0:
                        p2.append(self.mImageFeatures[view].points[hit]); p3.append(cp.p)
                        break
            out[view] = (np.array(p2, np.float32).reshape(-1, 2), np.array(p3, np.float32).reshape(-1, 3))
        self.seconds["glue"] += time.perf_counter() - t0; self.calls["glue"] += 1
        return out

    def mergeNewPointCloud(self, cloud):
        """SfM.cpp:530-600 (debug visualisation dropped)."""
        t0 = time.perf_counter()
        index = {}
        recon = self.mReconstructionCloud
        P = np.array([p.p for p in recon], np.float32).reshape(-1, 3)
        n_new = n_merged = 0
        grown = []
        for np_ in cloud:
            q = np.asarray(np_.p, np.float32)
            any_view = False; near3d = False
            cand = []
            if len(P):
                d = P - q                                                              # Point3f difference in float
                nrm = np.sqrt((d.astype(np.float64) ** 2).sum(1))                      # cv::norm accumulates in double
                cand = list(np.nonzero(nrm < MERGE_CLOUD_POINT_MIN_MATCH_DISTANCE)[0])
            for g in grown:                                                            # points appended during this merge
                d = (np.asarray(recon[g].p, np.float32) - q)
                if np.sqrt((d.astype(np.float64) ** 2).sum()) < MERGE_CLOUD_POINT_MIN_MATCH_DISTANCE:
                    cand.append(g)
            for e in cand:
                ep = recon[e]
                near3d = True
                for nview in sorted(np_.originatingViews):
                    nfeat = np_.originatingViews[nview]
                    ekeys = sorted(ep.originatingViews)
                    k = 0
                    while k < len(ekeys):                                              # std::map iteration with insertion (:553, :579)
                        eview = ekeys[k]; efeat = ep.originatingViews[eview]
                        new_left = nview < eview
                        lv, lf, rv, rf = (nview, nfeat, eview, efeat) if new_left else (eview, efeat, nview, nfeat)
                        idx = index.get((lv, rv))
                        if idx is None:
                            idx = index[(lv, rv)] = _PairIndex(self.mFeatureMatchMatrix[lv][rv])
                        hit = False
                        for pos in idx.qt.get((lf, rf), ()):
                            if idx.m["distance"][pos] < MERGE_CLOUD_FEATURE_MIN_MATCH_DISTANCE:
                                hit = True
                                break
                        if hit:
                            ep.originatingViews[nview] = nfeat
                            any_view = True
                            ekeys = sorted(ep.originatingViews)
                            k = ekeys.index(eview)
                        k += 1
                if any_view:
                    n_merged += 1
                    break
            if not any_view and not near3d:
                recon.append(np_); grown.append(len(recon) - 1); n_new += 1
        self.seconds["glue"] += time.perf_counter() - t0; self.calls["glue"] += 1
        return n_new, n_merged

    def addMoreViewsToReconstruction(self):
        """SfM.cpp:366-469."""
        while len(self.mDoneViews) != self.n:
            m23 = self.find2D3DMatches()
            best, best_n = None, 0
            for view in sorted(m23):
                if len(m23[view][0]) > best_n:
                    best, best_n = view, len(m23[view][0])
            if best is None:
                # the reference reads an uninitialised bestView here (SfM.cpp:374-381); stop instead
                break
            self.mDoneViews.add(best)
            ok, pose = self._timed("pnp", self.findCameraPoseFrom2D3DMatch, self.mIntrinsics, m23[best][0], m23[best][1])
            if self.trace is not None:
                self.trace.append({"stage": "pnp", "view": best, "points2D": m23[best][0], "points3D": m23[best][1], "ok": ok,
                                   "pose": None if pose is None else pose.copy()})
            if not ok:
                continue
            self.mCameraPoses[best] = pose
            any_ok = False
            for good in sorted(self.mGoodViews):
                l, r = (good, best) if good < best else (best, good)
                _, pruned, _, _ = self._timed("essential", self.findCameraMatricesFromMatch, self.mIntrinsics, self.mFeatureMatchMatrix[l][r],
                                              self.mImageFeatures[l], self.mImageFeatures[r])
                self.mFeatureMatchMatrix[l][r] = pruned
                cloud: List[Point3DInMap] = []
                ok = self._triangulate(l, r, self.mCameraPoses[l], self.mCameraPoses[r], cloud)
                if ok:
                    nn, nm = self.mergeNewPointCloud(cloud)
                    if self.verbose:
                        print(f"merge {l},{r}: {len(cloud)} triangulated, new {nn}, merged {nm}")
                    any_ok = True
            if any_ok:
                self.adjustCurrentBundle()
            self.mGoodViews.add(best)
