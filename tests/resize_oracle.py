"""numpy restatement of cv::resize(src, dst, Size(), s, s) with the default INTER_LINEAR on 8-bit B,G,R images (OpenCV 4.13), the
rules csrc/resize_math.cuh implements:

  output size   dw = cvRound(w * s), dh = cvRound(h * s) (half to even); the map scale is 1 / s
  same size     an output of the input's size is a copy (cv::resize's dsize == ssize shortcut)
  1 / s == 2    the fast INTER_AREA path: (a + b + c + d + 2) >> 2 over each 2x2 block; a block cut by the right or bottom edge
                averages its in-bounds pixels, cvRound((float)sum / count)
  otherwise     fixed-point bilinear with Q11 weights: per output column f = (float)((dx + 0.5) / s - 0.5), sx = floor(f), f -= sx,
                clamped to [0, w - 1] with f = 0 at either end; weights rint((1 - f) * 2048), rint(f * 2048) in float; rows the same
                but only their indices are clamped, not their weights; horizontal pass in int32, vertical pass with the rounding of
                OpenCV's SIMD kernel: sat_u8(((((A0 >> 4) * b0) >> 16) + (((A1 >> 4) * b1) >> 16) + 2) >> 2)

Vectorised: a 4000x3000 image resizes in well under a second."""
import math

import numpy as np


def resize_size(w, h, s):
    """(dw, dh) of cv::resize for factor s, or None where cv::resize asserts (s not finite or <= 0, or an empty output)."""
    s = float(s)
    if not math.isfinite(s) or s <= 0:
        return None
    dw, dh = np.rint(w * s), np.rint(h * s)
    if not (1 <= dw < 2**31 and 1 <= dh < 2**31):
        return None
    return int(dw), int(dh)


def taps(n_src, n_dst, s, clamp_weights):
    """Source indices (i0, i1) and Q11 weights (a0, a1) of every output column (clamp_weights=True) or row (False)."""
    d = np.arange(n_dst, dtype=np.float64)
    f = ((d + 0.5) * (1.0 / float(s)) - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    f = (f - i.astype(np.float32)).astype(np.float32)
    if clamp_weights:
        lo = i < 0
        i[lo] = 0; f[lo] = 0
        hi = i >= n_src - 1
        i[hi] = n_src - 1; f[hi] = 0
        i0, i1 = i, np.minimum(i + 1, n_src - 1)
    else:
        i0, i1 = np.clip(i, 0, n_src - 1), np.clip(i + 1, 0, n_src - 1)
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return i0, i1, a0, a1


def _linear(src, dw, dh, s):
    h, w = src.shape[:2]
    x0, x1, a0, a1 = taps(w, dw, s, True)
    y0, y1, b0, b1 = taps(h, dh, s, False)
    S = src.astype(np.int64)

    def hpass(rows):
        R = S[rows]
        return R[:, x0] * a0[None, :, None] + R[:, x1] * a1[None, :, None]
    A0, A1 = hpass(y0), hpass(y1)
    v = (((A0 >> 4) * b0[:, None, None]) >> 16) + (((A1 >> 4) * b1[:, None, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def _area2(src, dw, dh):
    h, w = src.shape[:2]
    out = np.empty((dh, dw, 3), np.uint8)
    S = src.astype(np.int64)
    iw, ih = min(dw, w // 2), min(dh, h // 2)
    blk = S[:2 * ih, :2 * iw].reshape(ih, 2, iw, 2, 3)
    out[:ih, :iw] = (blk.sum(axis=(1, 3)) + 2) >> 2
    # blocks cut by the right or bottom edge: the in-bounds pixels' mean, rounded half to even in float
    P = np.zeros((2 * dh, 2 * dw, 3), np.int64); M = np.zeros((2 * dh, 2 * dw), np.int64)
    P[:h, :w] = S[:2 * dh, :2 * dw]; M[:h, :w] = 1
    sums = P.reshape(dh, 2, dw, 2, 3).sum(axis=(1, 3)); cnt = M.reshape(dh, 2, dw, 2).sum(axis=(1, 3))
    edge = np.ones((dh, dw), bool); edge[:ih, :iw] = False
    mean = np.rint(sums[edge].astype(np.float32) / cnt[edge][:, None].astype(np.float32))
    out[edge] = np.clip(mean, 0, 255).astype(np.uint8)
    return out


def resize(src, s):
    """cv2.resize(src, None, fx=s, fy=s) of a uint8 [h, w, 3] image (interpolation INTER_LINEAR)."""
    src = np.asarray(src)
    assert src.dtype == np.uint8 and src.ndim == 3 and src.shape[2] == 3
    h, w = src.shape[:2]
    size = resize_size(w, h, s)
    if size is None:
        raise ValueError(f"cv::resize refuses factor {s!r} for a {w}x{h} image")
    dw, dh = size
    if (dw, dh) == (w, h):
        return src.copy()
    if 1.0 / float(s) == 2.0:
        return _area2(src, dw, dh)
    return _linear(src, dw, dh, s)
