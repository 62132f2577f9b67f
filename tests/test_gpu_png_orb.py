"""sfmb200_decode_images_extract_orb on the GPU: PNG (and mixed JPEG + PNG) files to ORB key points and descriptors in one call, the
images staying on the device.  Per image, every result equals, bit for bit, cv2.ORB_create(5000).detectAndCompute on cv2's decoded (and
resized) image: mixed sizes and formats, scale 0.5, no image download, and a decoded image below 8 pixels refused."""
import numpy as np
import pytest

import jpeg_util as J
import png_util as P

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _cv(b, scale=1.0):
    im = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    return im if scale == 1.0 else cv2.resize(im, None, fx=scale, fy=scale)


def _same(got, want):
    from oracle import orb_oracle as O
    (k, d), (wk, wd) = got, O.cv2_detect_and_compute(want, 5000)
    return k.shape[0] == wk.shape[0] and np.array_equal(k[:, :6], wk) and np.all(k[:, 6] == -1) and np.array_equal(d, wd)


def _files():
    ch = cv2.imread(P.os.path.join(P.ROOT, "tests", "golden", "crazyhorse_0.jpg"))
    return [P.imencode(ch),
            J.crazyhorse(),
            P.make_png(P.picture(300, 217, 5)[:, :, ::-1], 2, 8, 1, filters=(4, 1), post=P.chunk(b"eXIf", P.exif(6))),
            P.imencode(cv2.cvtColor(P.picture(190, 260, 6), cv2.COLOR_BGR2GRAY), [cv2.IMWRITE_PNG_COMPRESSION, 9]),
            J.encode(333, 221, q=80, seed=42),
            P.make_png(np.random.RandomState(2).randint(0, 16, (120, 90, 1)), 3, 4, palette=list(range(48))),
            P.imencode(P.picture(48, 40, 7))]


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_decode_images_orb_equals_cv2(ctx, scale):
    files = _files()
    images, feats = ctx.decode_images_orb(files, scale)
    for k, b in enumerate(files):
        want = _cv(b, scale)
        assert np.array_equal(images[k], want), k
        assert _same(feats[k], want), k
    assert sum(f[0].shape[0] for f in feats) > 2000


def test_without_images_and_order(ctx):
    files = _files()[::-1]
    none, feats = ctx.decode_images_orb(files, 1.0, images=False)
    assert none is None
    for k, b in enumerate(files):
        assert _same(feats[k], _cv(b)), k


def test_tiny_image_refused(ctx):
    from sfm_toy_library_b200 import capi
    good = P.imencode(P.picture(40, 40, 1))
    tiny = P.make_png(P.picture(7, 30, 2), 2, 8)
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.decode_images_orb([good, J.crazyhorse(), tiny])
    assert "image 2:" in str(e.value) and "minimum of 8" in str(e.value)
    with pytest.raises(capi.SfmB200Error) as e:
        ctx.decode_images_orb([good, good], 0.1)
    assert "image 0:" in str(e.value)
    _, feats = ctx.decode_images_orb([good])
    assert _same(feats[0], _cv(good))
