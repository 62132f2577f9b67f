"""The five decode entry points check every file before their first launch.  For each call and each refusal -- a file that is neither
JPEG nor PNG, a corrupt file, a missing output buffer, a scale that leaves an image with no pixels, an output stride below a row, an
image under ORB's 8 pixels -- the status, the index of the refused image, no kernel launched and a context that still decodes.  The
mixed-format calls meet the bad file as a PNG after a JPEG: its checks too come before the JPEG decode launches.  Lists with several
faults report the one the order of the checks puts first: format, then parse and output buffer, then downscale size, then per file
the output stride and ORB's limits, each step in the caller's order."""
import ctypes as C

import numpy as np
import pytest

import jpeg_util as J
import png_util as P

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

JPEG_ENTRIES = ("decode_jpeg_batch", "decode_jpeg_batch_scaled", "decode_jpeg_extract_orb")
MIXED_ENTRIES = ("decode_images", "decode_images_extract_orb")
SCALE = 0.04                                       # 64x48 -> 3x2, 20x30 -> 1x1; 16x10 -> no pixels


@pytest.fixture(scope="module")
def ctx():
    from sfm_toy_library_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _jpg():
    return J.encode(64, 48, seed=1)


def _png(h=30, w=20, seed=1):
    return P.make_png(P.picture(h, w, seed), 2, 8)


def _call(ctx, entry, files, scale=1.0, missing=(), strides=None):
    """sfmb200_<entry> through ctypes, with an output buffer for every image but those in `missing`, and the row strides `strides`
    (None: packed).  Returns (status, message)."""
    from sfm_toy_library_b200 import capi
    n = len(files)
    outs = []
    for f in files:
        rc, _, w, h = capi.image_info(f)
        if rc == 0 and scale != 1.0:
            w, h = capi.resize_size(w, h, scale) or (1, 1)
        outs.append(np.zeros(max(h, 1) * (3 * max(w, 1) + 16), np.uint8))
    ptrs = (C.c_void_p * n)(*[None if i in missing else o.ctypes.data for i, o in enumerate(outs)])
    st = (C.c_size_t * n)(*strides) if strides is not None else None
    data = (C.c_char_p * n)(*files)
    sizes = (C.c_size_t * n)(*[len(f) for f in files])
    fn = getattr(capi.lib(), "sfmb200_" + entry)
    if entry == "decode_jpeg_batch":
        rc = fn(ctx._h, data, sizes, n, ptrs, st)
    elif entry.endswith("_orb"):
        cap = 600
        kp = np.zeros((n, cap, 7), np.float32); desc = np.zeros((n, cap, 32), np.uint8); cnt = np.zeros(n, np.int32)
        rc = fn(ctx._h, data, sizes, n, C.c_double(scale), 500, cap, capi._p(kp, C.c_float), capi._p(desc, C.c_uint8), capi._p(cnt, C.c_int32),
                ptrs, st)
    else:
        rc = fn(ctx._h, data, sizes, n, C.c_double(scale), ptrs, st)
    return rc, capi.lib().sfmb200_last_error(ctx._h).decode()


def _refused(ctx, entry, files, k, text, **kw):
    """The call refuses image k with status 1 and `text` before it launches anything, and the context decodes afterwards."""
    l0 = ctx.kernel_launches
    rc, msg = _call(ctx, entry, files, **kw)
    assert (rc, ctx.kernel_launches) == (1, l0), (entry, msg)
    assert msg.startswith(f"image {k}:") and text in msg, (entry, msg)
    scale = 1.0 if entry == "decode_jpeg_batch" else 0.5
    assert _call(ctx, entry, [_jpg(), _png()] if entry in MIXED_ENTRIES else [_jpg(), _jpg()], scale)[0] == 0, entry


def _kind(kind):
    """(bad JPEG, bad PNG, call arguments, message) of a refusal."""
    return {
        "neither": (b"GIF89a" + bytes(20), b"GIF89a" + bytes(20), {}, ""),
        "corrupt": (_jpg()[:600], _png()[:60], {}, ""),
        "no_buffer": (_jpg(), _png(), dict(missing=(2,)), "no output buffer"),
        "empty_scale": (J.encode(16, 10, seed=5), _png(10, 16, 5), dict(scale=SCALE), "gives no image"),
        "short_stride": (_jpg(), _png(), {}, "output stride"),
        "below_orb": (J.encode(40, 6, seed=3), _png(7, 20, 3), {}, "below ORB's minimum"),
    }[kind]


# every refusal of every call (sfmb200_decode_jpeg_batch takes no scale; only the ORB calls have a minimum size)
CASES = [(entry, kind) for kind in ("neither", "corrupt", "no_buffer", "empty_scale", "short_stride", "below_orb") for entry in JPEG_ENTRIES + MIXED_ENTRIES
         if not (kind == "empty_scale" and entry == "decode_jpeg_batch") and not (kind == "below_orb" and not entry.endswith("_orb"))]


@pytest.mark.parametrize("entry,kind", CASES)
def test_each_refusal_before_any_launch(ctx, entry, kind):
    bad_jpg, bad_png, kw, text = _kind(kind)
    mixed = entry in MIXED_ENTRIES
    files = [_png(), _jpg(), bad_png] if mixed else [_jpg(), J.encode(40, 32, seed=2), bad_jpg]
    if kind == "short_stride":
        kw = dict(strides=[0, 0, 3 * (20 if mixed else 64) - 3])
    if kind == "neither" and mixed:
        text = "neither a JPEG nor a PNG file"
    _refused(ctx, entry, files, 2, text, **kw)


def test_mixed_lists_refuse_a_late_png_before_the_jpeg_decode(ctx):
    _refused(ctx, "decode_images_extract_orb", [_png(), _jpg(), _png(7, 20, 3)], 2, "below ORB's minimum")
    _refused(ctx, "decode_images", [_png(), _jpg(), _png()], 2, "output stride", strides=[0, 0, 3 * 20 - 1])


def test_several_faults_follow_the_order_of_the_checks(ctx):
    tiny = J.encode(40, 6, seed=3)                 # below ORB's minimum (step 5)
    entry = "decode_images_extract_orb"
    stride = [0, 3 * 20 - 3, 0, 0]                 # image 1's rows too short (step 5)
    # a format fault (step 2) goes before every later one
    _refused(ctx, entry, [tiny, _png(), _jpg(), b"GIF89a" + bytes(20)], 3, "neither a JPEG nor a PNG file", missing=(2,), strides=stride)
    # parse and output buffers (step 3), in the caller's order, before the per-file checks of images 0 and 1
    _refused(ctx, entry, [tiny, _png(), _jpg(), _png()[:60]], 2, "no output buffer", missing=(2,), strides=stride)
    _refused(ctx, entry, [tiny, _png(), _jpg(), _png()[:60]], 3, "", strides=stride)
    # the downscale's sizes (step 4): a 20x1 image has no pixels at 0.5
    _refused(ctx, entry, [tiny, _png(), _jpg(), _png(1, 20, 4)], 3, "gives no image", scale=0.5, strides=[0, 3 * 10 - 3, 0, 0])
    # per file (step 5): image 0's ORB minimum before image 1's stride
    _refused(ctx, entry, [tiny, _png(), _jpg(), _png()], 0, "below ORB's minimum", strides=stride)
    _refused(ctx, entry, [_jpg(), _png(), _jpg(), _png()], 1, "output stride", strides=stride)
