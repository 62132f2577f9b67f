"""Host mirror of the one-call front end (stages.readImagesAndFeatures, the readImagesAndFeatures hook of runsfm.SfM.from_directory) with a
stand-in context: the files reach the context as bytes in name order with the reference's float factor, the features are built like
extractFeatures builds them, and the driver takes them as they are with K from image 0's size.  The arithmetic is tested on the GPU
(test_gpu_jpeg_orb.py)."""
import numpy as np

from sfm_toy_library_b200 import runsfm, stages


class FakeCtx:
    def __init__(self, shapes):
        self.shapes = shapes
        self.calls = []

    def decode_jpeg_orb(self, blobs, scale=1.0, nfeatures=5000, capacity=None, images=True):
        self.calls.append((list(blobs), scale, nfeatures))
        imgs, feats = [], []
        for b, (h, w) in zip(blobs, self.shapes):
            n = len(b)
            imgs.append(np.full((h, w, 3), n, np.uint8))
            kp = np.zeros((n, 7), np.float32); kp[:, 0] = np.arange(n); kp[:, 1] = 3 * np.arange(n); kp[:, 6] = -1
            feats.append((kp, np.full((n, 32), n, np.uint8)))
        return (imgs if images else None), feats


def _files(tmp_path, sizes):
    paths = []
    for k, n in enumerate(sizes):
        p = tmp_path / f"img{k}.jpg"
        p.write_bytes(bytes(range(n)))
        paths.append(str(p))
    return paths


def test_read_images_and_features_builds_the_reference_containers(tmp_path):
    files = _files(tmp_path, [5, 9, 2])
    ctx = FakeCtx([(20, 30), (30, 20), (8, 8)])
    images, feats = stages.readImagesAndFeatures(files, 0.3, ctx=ctx)
    blobs, scale, nf = ctx.calls[0]
    assert len(ctx.calls) == 1 and nf == 5000                                   # ORB::create(5000), SfM2DFeatureUtilities.cpp:39
    assert blobs == [bytes(range(n)) for n in (5, 9, 2)]
    assert scale == float(np.float32(0.3)) and scale != 0.3                      # the reference's float factor, widened
    assert [im.shape for im in images] == [(20, 30, 3), (30, 20, 3), (8, 8, 3)]
    for f, n in zip(feats, (5, 9, 2)):
        assert f.points.shape == (n, 2) and f.points.dtype == np.float32 and f.descriptors.shape == (n, 32)
        assert np.array_equal(f.points, f.keyPoints[:, :2])                    # KeyPointsToPoints, SfMCommon.cpp:89-94
    _, _ = stages.readImagesAndFeatures(files, ctx=ctx)
    assert ctx.calls[1][1] == 1.0


def test_from_directory_hook_replaces_read_and_extract(tmp_path):
    _files(tmp_path, [4, 6, 3])
    (tmp_path / "notes.txt").write_text("not an image")
    ctx = FakeCtx([(600, 800), (800, 600), (600, 800)])
    seen = []

    def hook(files, downscale):
        seen.append((files, downscale))
        return stages.readImagesAndFeatures(files, downscale, ctx=ctx)

    def never(*a, **k):
        raise AssertionError("readImages / extractAllFeatures must not run when readImagesAndFeatures is given")

    sfm = runsfm.SfM.from_directory(str(tmp_path), readImages=never, extractAllFeatures=never, readImagesAndFeatures=hook, downscale=0.5)
    assert [f.rsplit("/", 1)[1] for f in seen[0][0]] == ["img0.jpg", "img1.jpg", "img2.jpg"] and seen[0][1] == 0.5
    assert sfm.n == 3 and [len(f.points) for f in sfm.mImageFeatures] == [4, 6, 3]
    assert sfm.mIntrinsics.K[0, 2] == 400 and sfm.mIntrinsics.K[1, 2] == 300      # SfM.cpp:70-72 from image 0's size
    assert sfm.calls["read"] == 3 and sfm.seconds["read"] >= 0
