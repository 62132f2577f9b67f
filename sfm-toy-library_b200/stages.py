"""Host-side mirror (Python) of the reference's stage interface, over the C ABI.

Same names, argument order and semantics as the stage functions the reference's SfM class calls
(SfM.cpp:148, 197, 293, 435, 325):
    SfM2DFeatureUtilities::extractFeatures      SfMToyLib/SfM2DFeatureUtilities.h:41-42   (SURVEY.md 8 row f-3)
    SfM2DFeatureUtilities::matchFeatures        SfMToyLib/SfM2DFeatureUtilities.h:44-46
    SfMStereoUtilities::triangulateViews        SfMToyLib/SfMStereoUtilities.h:82-91
    SfMBundleAdjustmentUtils::adjustBundle      SfMToyLib/SfMBundleAdjustmentUtils.h:44-49
and the SfMCommon.h data carriers (:55-99).  The C++ twin of this file (what main.cpp links) is host/.
All arithmetic happens in libsfmb200.so; this file only flattens / unflattens the containers.
"""
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from . import capi

# cv::DMatch as a structured array: queryIdx, trainIdx, imgIdx, distance (16 bytes, like the C++ struct)
DMATCH = np.dtype([("queryIdx", np.int32), ("trainIdx", np.int32), ("imgIdx", np.int32), ("distance", np.float32)])


@dataclass
class Intrinsics:                      # SfMCommon.h:55-59
    K: np.ndarray                      # 3x3 float32
    Kinv: Optional[np.ndarray] = None
    distortion: Optional[np.ndarray] = None


@dataclass
class ImagePair:                       # SfMCommon.h:61-63
    left: int
    right: int


@dataclass
class Features:                        # SfMCommon.h:76-80
    keyPoints: Optional[list] = None   # unused by the hot path (points carries kp.pt)
    points: np.ndarray = field(default_factory=lambda: np.zeros((0, 2), np.float32))
    descriptors: np.ndarray = field(default_factory=lambda: np.zeros((0, 32), np.uint8))


@dataclass
class Point3DInMap:                    # SfMCommon.h:82-88
    p: np.ndarray                      # 3 float32
    originatingViews: Dict[int, int] = field(default_factory=dict)


PointCloud = List[Point3DInMap]

_default_ctx = None


def default_context():
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = capi.Context(0)
    return _default_ctx


def GetAlignedMatching(size):          # SfMCommon.cpp:120-126
    m = np.zeros(size, DMATCH)
    m["queryIdx"] = np.arange(size); m["trainIdx"] = np.arange(size)
    return m


def _reference_factor(downscale) -> float:
    """The reference keeps the factor as `float mDownscaleFactor` (SfM.h) and passes it to cv::resize widened to double."""
    return float(np.float32(downscale))


def _read_files(files: List[str]) -> List[bytes]:
    blobs = []
    for f in files:
        with open(f, "rb") as fh:
            blobs.append(fh.read())
    return blobs


def _any_png(blobs: List[bytes]) -> bool:
    return any(b[:8] == capi.PNG_SIGNATURE for b in blobs)


def readImages(files: List[str], ctx=None, downscale: float = 1.0) -> List[np.ndarray]:
    """The imread loop of SfM::setImagesDirectory (SfM.cpp:123-135) on the device: every file decoded in one call, byte-identical to
    cv2.imread(file) (B,G,R, EXIF orientation applied).  The reference reads .jpg and .png files; a list with any PNG file goes to
    sfmb200_decode_images (any mix of the two formats), an all-JPEG list to sfmb200_decode_jpeg_batch.  With downscale != 1 the
    loop's resize (:127-129) runs on the device in the same call, byte-identical to cv2.resize(cv2.imread(file), None, fx=s, fy=s)
    with s the factor as the reference's float.  There is no host fallback: a file that is neither JPEG nor PNG, or a corrupt or
    unsupported one, raises capi.SfmB200Error naming it."""
    ctx = ctx or default_context()
    blobs = _read_files(files)
    if _any_png(blobs):
        return ctx.decode_images(blobs, _reference_factor(downscale))
    return ctx.decode_jpeg(blobs, _reference_factor(downscale))


def resizeImages(images: List[np.ndarray], downscale: float, ctx=None) -> List[np.ndarray]:
    """The resize of SfM::setImagesDirectory (SfM.cpp:127-129) for images already in host memory (PNG files, cv2.imread):
    all of them in one sfmb200_resize_batch call, byte-identical to cv2.resize(img, None, fx=s, fy=s) with s the factor as the
    reference's float.  A factor of 1 returns the images unchanged, as the reference skips the call."""
    s = _reference_factor(downscale)
    if s == 1.0:
        return list(images)
    return (ctx or default_context()).resize_images(list(images), s)


ORB_FEATURES = 5000                    # mDetector = ORB::create(5000), SfM2DFeatureUtilities.cpp:39


def _features_from(kp, desc) -> Features:
    # keyPoints: the cv::KeyPoint fields as rows (x, y, size, angle, response, octave, class_id); points = KeyPointsToPoints (SfMCommon.cpp:89-94)
    return Features(keyPoints=kp, points=np.ascontiguousarray(kp[:, :2]), descriptors=desc)


def extractFeatures(image: np.ndarray, ctx=None) -> Features:
    """SfM2DFeatureUtilities::extractFeatures (SfM2DFeatureUtilities.cpp:46-51): ORB(5000) detectAndCompute + KeyPointsToPoints.
    `image`: uint8 [h, w, 3] in B,G,R order (what cv::imread returns, SfM.cpp:124) or [h, w] grey."""
    ctx = ctx or default_context()
    return _features_from(*ctx.orb_detect_and_compute(image, ORB_FEATURES))


def extractAllFeatures(images: List[np.ndarray], ctx=None) -> List[Features]:
    """The batched form of SfM::extractFeatures (SfM.cpp:141-154): all (equally sized) images of a run in one launch sequence."""
    ctx = ctx or default_context()
    if len({im.shape for im in images}) > 1:
        return [extractFeatures(im, ctx) for im in images]
    return [_features_from(k, d) for k, d in ctx.orb_detect_and_compute(list(images), ORB_FEATURES)]


def readImagesAndFeatures(files: List[str], downscale: float = 1.0, ctx=None):
    """readImages followed by extractFeatures on every image, with the images staying on the device in between
    (sfmb200_decode_jpeg_extract_orb, or sfmb200_decode_images_extract_orb when any file is a PNG): returns (images, features), the
    images as readImages returns them and per image the Features extractFeatures gives for it.  The images may differ in size
    (portrait and landscape shots of one folder) and format."""
    ctx = ctx or default_context()
    blobs = _read_files(files)
    if _any_png(blobs):
        images, feats = ctx.decode_images_orb(blobs, _reference_factor(downscale), ORB_FEATURES)
    else:
        images, feats = ctx.decode_jpeg_orb(blobs, _reference_factor(downscale), ORB_FEATURES)
    return images, [_features_from(k, d) for k, d in feats]


def matchFeatures(featuresLeft: Features, featuresRight: Features, ctx=None) -> np.ndarray:
    """SfM2DFeatureUtilities::matchFeatures (SfM2DFeatureUtilities.cpp:53-71)."""
    ctx = ctx or default_context()
    q, t, d = ctx.match_knn2_ratio(featuresLeft.descriptors, featuresRight.descriptors, capi.RATIO_REFERENCE)
    m = np.zeros(len(q), DMATCH)
    m["queryIdx"] = q; m["trainIdx"] = t; m["distance"] = d
    return m


def triangulateViews(intrinsics: Intrinsics, imagePair: ImagePair, matches: np.ndarray, featuresLeft: Features,
                     featuresRight: Features, Pleft: np.ndarray, Pright: np.ndarray, pointCloud: PointCloud, ctx=None) -> bool:
    """SfMStereoUtilities::triangulateViews (SfMStereoUtilities.cpp:120-206): APPENDS to pointCloud, returns True."""
    ctx = ctx or default_context()
    mq = np.ascontiguousarray(matches["queryIdx"]); mt = np.ascontiguousarray(matches["trainIdx"])
    X, keep, _ = ctx.triangulate(intrinsics.K, Pleft, Pright, featuresLeft.points, featuresRight.points, mq, mt,
                                 capi.MIN_REPROJECTION_ERROR)
    for i in np.nonzero(keep)[0]:
        pointCloud.append(Point3DInMap(X[i].copy(), {int(imagePair.left): int(mq[i]), int(imagePair.right): int(mt[i])}))
    return True


def triangulateManyPairs(intrinsics: Intrinsics, features: List[Features], pairs, matches, poses, ctx=None) -> List[PointCloud]:
    """triangulateViews for every pair in one device call (sfmb200_triangulate_pairs).  features: per image Features; pairs
    [(i, j), ...]; matches: per pair a structured array with queryIdx / trainIdx; poses: per pair (Pleft, Pright).  Returns one
    PointCloud per pair, each exactly what triangulateViews appends for that pair."""
    ctx = ctx or default_context()
    if len(pairs) == 0:
        return []
    mq, mt, off = capi.flatten_matches([m["queryIdx"] for m in matches], [m["trainIdx"] for m in matches])
    X, keep, _ =ctx.triangulate_pairs(intrinsics.K, [np.stack([Pl, Pr]) for Pl, Pr in poses], [f.points for f in features], pairs, mq, mt, off,
                                       capi.MIN_REPROJECTION_ERROR)
    clouds = []
    for p, (left, right) in enumerate(pairs):
        clouds.append([Point3DInMap(X[i].copy(), {int(left): int(mq[i]), int(right): int(mt[i])})
                       for i in off[p] + np.nonzero(keep[off[p]:off[p + 1]])[0]])
    return clouds


def pose_is_empty(pose) -> bool:
    """The reference's "empty pose" rule (SfMBundleAdjustmentUtils.cpp:118-122, :196-199): R diagonal exactly zero."""
    pose = np.asarray(pose, np.float32).reshape(3, 4)
    return bool(pose[0, 0] == 0 and pose[1, 1] == 0 and pose[2, 2] == 0)


def flatten_bundle(pointCloud: PointCloud, cameraPoses: List[np.ndarray], intrinsics: Intrinsics, image2dFeatures: List[Features],
                   rot2aa=None):
    """The problem assembly of adjustBundle (SfMBundleAdjustmentUtils.cpp:111-166) into the flat arrays of the C ABI.
    Only views that appear in some originatingViews become camera blocks (Ceres only knows parameter blocks that appear
    in a residual block); `cam_ids` maps dense index -> view id.  An observed view whose pose is "empty" (:118-122) enters
    with the all-zero CameraVector() the reference pushes for it (:120) -- and is never written back (:196-199)."""
    rot2aa = rot2aa or capi.rotmat_to_angle_axis_f32
    K = np.asarray(intrinsics.K, np.float32)
    used = sorted({v for p in pointCloud for v in p.originatingViews})
    dense = {v: i for i, v in enumerate(used)}
    cams = np.zeros((len(used), 6))
    for v in used:
        pose = np.asarray(cameraPoses[v], np.float32).reshape(3, 4)
        if pose_is_empty(pose):
            continue                                                             # CameraVector() = zeros (:120)
        cams[dense[v], :3] = rot2aa(pose[:, :3])                                 # float conversion (:126), widened
        cams[dense[v], 3:] = pose[:, 3]
    focal = float(K[0, 0])                                                       # :138
    pts = np.array([p.p for p in pointCloud], np.float32).astype(np.float64).reshape(-1, 3)
    obs_xy, obs_cam, pt_off = [], [], [0]
    cx, cy = K[0, 2], K[1, 2]
    for p in pointCloud:
        for v in sorted(p.originatingViews):                                     # std::map iteration order (:146)
            p2d = np.asarray(image2dFeatures[v].points[p.originatingViews[v]], np.float32)
            obs_xy.append((np.float32(p2d[0] - cx), np.float32(p2d[1] - cy)))    # float subtraction (:152-153)
            obs_cam.append(dense[v])
        pt_off.append(len(obs_cam))
    return (cams, pts, focal, np.asarray(obs_xy, np.float32).reshape(-1, 2), np.asarray(obs_cam, np.int32),
            np.asarray(pt_off, np.int32), used)


def write_back_bundle(pointCloud, cameraPoses, intrinsics, cams, pts, focal, used, rot2aa=None, aa2rot=None):
    """The write-back of adjustBundle (SfMBundleAdjustmentUtils.cpp:188-221), run only after CONVERGENCE.  EVERY non-empty pose
    is rewritten from its 6-vector (:192-215): the observed ones from the optimised parameters, the unobserved ones from the
    float angle-axis of their own rotation widened to double (their CameraVector never entered the problem) -- i.e. they
    are round-tripped through RotationMatrixToAngleAxis<float> / AngleAxisToRotationMatrix<double>.  Empty poses are skipped."""
    rot2aa = rot2aa or capi.rotmat_to_angle_axis_f32
    aa2rot = aa2rot or capi.angle_axis_to_rotmat
    intrinsics.K[0, 0] = np.float32(focal); intrinsics.K[1, 1] = np.float32(focal)     # :188-189
    dense = {v: i for i, v in enumerate(used)}
    for v in range(len(cameraPoses)):
        pose = cameraPoses[v]
        if pose_is_empty(pose):
            continue
        if v in dense:
            aa = cams[dense[v], :3]; t = cams[dense[v], 3:]
        else:
            aa = rot2aa(np.asarray(pose, np.float32)[:, :3]).astype(np.float64); t = np.asarray(pose, np.float32)[:, 3].astype(np.float64)
        pose[:, :3] = aa2rot(aa).astype(np.float32)
        pose[:, 3] = np.asarray(t).astype(np.float32)
    for i, p in enumerate(pointCloud):                                           # :217-221
        p.p = pts[i].astype(np.float32)


def adjustBundle(pointCloud: PointCloud, cameraPoses: List[np.ndarray], intrinsics: Intrinsics, image2dFeatures: List[Features],
                 ctx=None, options=None):
    """SfMBundleAdjustmentUtils::adjustBundle (SfMBundleAdjustmentUtils.cpp:99-222).  Mutates pointCloud, cameraPoses
    and intrinsics in place iff the solver reports CONVERGENCE (:182-185).  Returns the solver summary."""
    ctx = ctx or default_context()
    cams, pts, focal, obs_xy, obs_cam, pt_off, used = flatten_bundle(pointCloud, cameraPoses, intrinsics, image2dFeatures)
    cams, pts, focal, summary = ctx.ba_solve(cams, pts, focal, obs_xy, obs_cam, pt_off, options)
    if summary["termination_type"] != capi.CONVERGENCE:
        print("Bundle adjustment failed.")                                       # :183
        return summary
    write_back_bundle(pointCloud, cameraPoses, intrinsics, cams, pts, focal, used)
    return summary


def matchAllPairs(features: List[Features], pairs, ctx=None) -> List[np.ndarray]:
    """The batched form of SfM::createFeatureMatchMatrix (SfM.cpp:157-212): descriptors uploaded once
    (sfmb200_descset), every (left, right) pair matched in one launch sequence (sfmb200_match_pairs)."""
    ctx = ctx or default_context()
    ds = ctx.descriptor_set([f.descriptors for f in features])
    try:
        res = ds.match_pairs(pairs, capi.RATIO_REFERENCE)
    finally:
        ds.close()
    out = []
    for q, t, d in res:
        m = np.zeros(len(q), DMATCH)
        m["queryIdx"] = q; m["trainIdx"] = t; m["distance"] = d
        out.append(m)
    return out
