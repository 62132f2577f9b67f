"""The stages send lists with a PNG file to the mixed-format calls (decode_images / decode_images_orb) and all-JPEG lists to the JPEG
calls, with the bytes in name order and the reference's float factor; SfM.from_directory hands .png files to readImagesAndFeatures.
A stand-in context records the calls; the arithmetic is tested on the GPU (test_gpu_png.py, test_gpu_png_orb.py)."""
import numpy as np

from sfm_toy_library_b200 import capi, runsfm, stages


class FakeCtx:
    def __init__(self):
        self.calls = []

    def _imgs(self, blobs):
        return [np.full((9, 10, 3), len(b), np.uint8) for b in blobs]

    def _feats(self, blobs):
        out = []
        for b in blobs:
            n = len(b)
            kp = np.zeros((n, 7), np.float32); kp[:, 0] = np.arange(n); kp[:, 6] = -1
            out.append((kp, np.full((n, 32), n, np.uint8)))
        return out

    def decode_jpeg(self, blobs, scale=1.0):
        self.calls.append(("decode_jpeg", list(blobs), scale)); return self._imgs(blobs)

    def decode_images(self, blobs, scale=1.0):
        self.calls.append(("decode_images", list(blobs), scale)); return self._imgs(blobs)

    def decode_jpeg_orb(self, blobs, scale=1.0, nfeatures=5000, capacity=None, images=True):
        self.calls.append(("decode_jpeg_orb", list(blobs), scale)); return self._imgs(blobs), self._feats(blobs)

    def decode_images_orb(self, blobs, scale=1.0, nfeatures=5000, capacity=None, images=True):
        self.calls.append(("decode_images_orb", list(blobs), scale)); return self._imgs(blobs), self._feats(blobs)


def _write(tmp_path, names):
    paths = []
    for k, n in enumerate(names):
        p = tmp_path / n
        p.write_bytes((capi.PNG_SIGNATURE if n.lower().endswith(".png") else b"\xff\xd8") + bytes(range(k + 3)))
        paths.append(str(p))
    return paths


def test_stages_route_by_signature(tmp_path):
    ctx = FakeCtx()
    mixed = _write(tmp_path, ["a.jpg", "b.png", "c.jpg"])
    jpgs = [mixed[0], mixed[2]]
    stages.readImages(mixed, ctx=ctx, downscale=0.3)
    stages.readImages(jpgs, ctx=ctx)
    stages.readImagesAndFeatures(mixed, 0.3, ctx=ctx)
    images, feats = stages.readImagesAndFeatures(jpgs, ctx=ctx)
    names = [c[0] for c in ctx.calls]
    assert names == ["decode_images", "decode_jpeg", "decode_images_orb", "decode_jpeg_orb"]
    blobs = [open(f, "rb").read() for f in mixed]
    assert ctx.calls[0][1] == blobs and ctx.calls[2][1] == blobs
    assert ctx.calls[0][2] == float(np.float32(0.3)) != 0.3 and ctx.calls[1][2] == 1.0
    assert len(feats) == 2 and feats[1].points.shape == (len(blobs[2]), 2)


def test_from_directory_hands_png_files_to_the_hook(tmp_path):
    _write(tmp_path, ["x1.PNG", "x0.png", "x2.jpg"])
    (tmp_path / "notes.txt").write_text("not an image")
    ctx = FakeCtx()
    seen = []

    def hook(files, downscale):
        seen.append(files)
        return stages.readImagesAndFeatures(files, downscale, ctx=ctx)

    sfm = runsfm.SfM.from_directory(str(tmp_path), readImagesAndFeatures=hook)
    assert [f.rsplit("/", 1)[1] for f in seen[0]] == ["x0.png", "x1.PNG", "x2.jpg"]
    assert ctx.calls[0][0] == "decode_images_orb" and sfm.n == 3
