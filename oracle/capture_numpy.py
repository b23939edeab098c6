"""Numpy restatement of the live-capture kernels (splatam_b200/csrc/ingest.cu: sb_ingest_capture,
sb_capture_depth_u16), i.e. of what the reference's online demo and capture script do to one NeRFCapture packet
(R/scripts/iphone_demo.py:177-182, 218-243; nerfcapture2dataset.py:133-138):

  colour: cv2.resize(uint8 rgb, (W, H), INTER_LINEAR).float() / 255
  depth : cv2.resize(float32 metres, (W, H), INTER_NEAREST)
  saved : cv2.resize((depth * 65535 / float(depth_scale)).astype(uint16), (w, h), INTER_NEAREST)

cv2 4.13 and NumPy 2 on x86-64, restated (test infrastructure only; the product path is the CUDA kernels).  cv2 runs
uint8 INTER_LINEAR in fixed point, so these rules differ from the float64 ones of oracle/ingest_numpy.py; the
nearest-neighbour index rule is the same and is taken from there.
"""
import numpy as np

from .ingest_numpy import nearest_index


def linear_taps_u8(n_dst, n_src, horizontal=True):
    """(i0, i1, a0, a1) per destination index of cv2's uint8 INTER_LINEAR: fx = float32((d + 0.5) * scale - 0.5) with
    scale = 1 / (n_dst / n_src) in double, sx = floor(fx), f = fx - sx in float32; weights a0 = rint((1 - f) * 2048),
    a1 = rint(f * 2048).  Horizontally a tap below 0 becomes 0 and one at or past n_src - 1 becomes n_src - 1, both with
    f = 0.  Vertically (`horizontal` False) the taps sx and sx + 1 are clamped to [0, n_src - 1] and f is kept: the two
    rows are then the same row with both weights, which the vertical rounding can leave 1 below the copy.  That case
    only arises when upscaling."""
    fx = ((np.arange(n_dst, dtype=np.float64) + 0.5) * (1.0 / (n_dst / n_src)) - 0.5).astype(np.float32)
    sx = np.floor(fx)
    f = (fx - sx).astype(np.float32)
    i = sx.astype(np.int64)
    if horizontal:
        edge = (i < 0) | (i >= n_src - 1)
        f = np.where(edge, np.float32(0), f).astype(np.float32)
        i0 = np.clip(i, 0, n_src - 1)
        i1 = np.where(edge, i0, i0 + 1)
    else:
        i0, i1 = np.clip(i, 0, n_src - 1), np.clip(i + 1, 0, n_src - 1)
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return i0, i1, a0, a1


def resize_linear_u8(img, H, W):
    """cv2.resize(uint8 img, (W, H), interpolation=INTER_LINEAR) of an [h, w, C] array, as cv2 4.13 computes it on
    x86-64 (a different rule from ingest_numpy's float64 one):
    * equal size: a copy;
    * an exact 2x downscale in both axes: INTER_AREA, (a + b + c + d + 2) >> 2;
    * otherwise the fixed-point taps of `linear_taps_u8`; the horizontal pass row = S[x0] * a0 + S[x1] * a1 in int32,
      then the vertical pass with the vectorised rounding
      (((row0 >> 4) * b0 >> 16) + ((row1 >> 4) * b1 >> 16) + 2) >> 2, clamped to [0, 255].  The scalar rounding
      (row0 * b0 + row1 * b1 + 2^21) >> 22 differs from cv2 at some sizes (700x500, 333x257)."""
    src = np.asarray(img, dtype=np.uint8)
    h, w = src.shape[:2]
    if (h, w) == (H, W):
        return src.copy()
    s = src.astype(np.int64)
    if h == 2 * H and w == 2 * W:
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    x0, x1, a0, a1 = linear_taps_u8(W, w)
    y0, y1, b0, b1 = linear_taps_u8(H, h, horizontal=False)
    rows = s[:, x0] * a0[None, :, None] + s[:, x1] * a1[None, :, None]
    v = ((((rows[y0] >> 4) * b0[:, None, None]) >> 16) + (((rows[y1] >> 4) * b1[:, None, None]) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def resize_nearest(a, H, W):
    """cv2.resize(a, (W, H), interpolation=INTER_NEAREST) of a 2-D array, any dtype (values are copied)."""
    return a[nearest_index(H, a.shape[0])][:, nearest_index(W, a.shape[1])]


def quantise_u16(depth, depth_scale):
    """(depth * 65535 / float(depth_scale)).astype(uint16) of a float32 array as NumPy 2 computes it on x86-64: both
    operations in float32, then the cast truncates to int32 and keeps the low 16 bits (10.5 m at scale 10 -> 3275,
    -0.5 m -> 62260); NaN, +-inf and values outside int32 -> 0."""
    v = (np.asarray(depth, np.float32) * np.float32(65535)) / np.float32(depth_scale)
    ok = (v > np.float32(-2.0 ** 31)) & (v < np.float32(2.0 ** 31))
    i = np.where(ok, np.trunc(np.where(ok, v, 0)).astype(np.int64), -2 ** 31)
    return (i & 0xFFFF).astype(np.uint16)


def ingest_capture(rgb, depth, H, W):
    """One live packet (rgb uint8 [h, w, 3], depth float32 [hd, wd] in metres) as the online demo turns it into a
    frame (R/scripts/iphone_demo.py:218-243): (colour float32 [3, H, W] = resize_linear_u8 / 255, depth float32
    [1, H, W] = resize_nearest), as sb_ingest_capture writes them."""
    color = (resize_linear_u8(rgb, H, W).astype(np.float32) / np.float32(255.0)).transpose(2, 0, 1)
    depth = resize_nearest(np.asarray(depth, np.float32), H, W)[None]
    return np.ascontiguousarray(color), np.ascontiguousarray(depth)


def capture_depth_u16(depth, depth_scale, H, W):
    """The depth image the capture writers save (nerfcapture2dataset.py:133-138): the nearest resize of the quantised
    depth to the colour's size, as sb_capture_depth_u16 writes it."""
    return np.ascontiguousarray(resize_nearest(quantise_u16(depth, depth_scale), H, W))
