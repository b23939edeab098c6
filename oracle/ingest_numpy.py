"""Float64 numpy restatement of the frame-ingest kernel (splatam_b200/csrc/ingest.cu), i.e. of what the reference's
dataset loader does to one frame (R/datasets/gradslam_datasets/basedataset.py:224-257, 296-341):

  colour: float32(cv2.resize(float64 rgb, (W, H), INTER_LINEAR)) / 255
  depth : float32(cv2.resize(float64 raw, (W, H), INTER_NEAREST) / png_depth_scale)

cv2's rules, restated (test infrastructure only; the product path is the CUDA kernel):
* equal size: a copy;
* an exact 2x downscale in both axes: INTER_LINEAR becomes INTER_AREA, the mean of each 2x2 box;
* otherwise bilinear with half-pixel centres, in double: per axis f = (d + 0.5) * (1 / (n_dst / n_src)) - 0.5, the
  taps are floor(f) and floor(f) + 1 with weights (1 - frac, frac); a tap below 0 becomes 0 and a tap at or past
  n_src - 1 becomes n_src - 1, both with weight 0 on the second tap.  The horizontal pass runs first.  This differs
  from cv2's float64 result by about 1e-11 (cv2 evaluates the same weights in another order), far below the float32
  rounding applied next.
* nearest: s = min(floor(d * (1 / (n_dst / n_src))), n_src - 1).
"""
import numpy as np


def linear_taps(n_dst, n_src):
    """(i0, i1, w0, w1) per destination index: the two source taps and their float64 weights."""
    f = (np.arange(n_dst, dtype=np.float64) + 0.5) * (1.0 / (n_dst / n_src)) - 0.5
    i = np.floor(f).astype(np.int64)
    f = f - i
    edge = (i < 0) | (i >= n_src - 1)
    f = np.where(edge, 0.0, f)
    i0 = np.clip(i, 0, n_src - 1)
    i1 = np.where(edge, i0, i0 + 1)
    return i0, i1, 1.0 - f, f


def resize_linear(img, H, W):
    """cv2.resize(img.astype(float64), (W, H), interpolation=INTER_LINEAR) of an [h, w, C] or [h, w] array."""
    src = np.asarray(img, dtype=np.float64)
    flat = src.ndim == 2
    if flat:
        src = src[:, :, None]
    h, w = src.shape[:2]
    if (h, w) == (H, W):
        out = src.copy()
    elif h == 2 * H and w == 2 * W:
        out = (src[0::2, 0::2] + src[0::2, 1::2] + src[1::2, 0::2] + src[1::2, 1::2]) * 0.25
    else:
        x0, x1, a0, a1 = linear_taps(W, w)
        y0, y1, b0, b1 = linear_taps(H, h)
        rows = src[:, x0] * a0[None, :, None] + src[:, x1] * a1[None, :, None]
        out = rows[y0] * b0[:, None, None] + rows[y1] * b1[:, None, None]
    return out[:, :, 0] if flat else out


def nearest_index(n_dst, n_src):
    return np.minimum(np.floor(np.arange(n_dst, dtype=np.float64) * (1.0 / (n_dst / n_src))).astype(np.int64),
                      n_src - 1)


def ingest(rgb, depth_raw, H, W, png_depth_scale):
    """rgb: uint8 [h, w, 3]; depth_raw: uint16 [hd, wd].  Returns (colour float32 [3, H, W], depth float32 [1, H, W])
    as the kernel writes them."""
    color = (resize_linear(rgb, H, W).astype(np.float32) / np.float32(255.0)).transpose(2, 0, 1)
    d = np.asarray(depth_raw, dtype=np.float64)
    d = d[nearest_index(H, d.shape[0])][:, nearest_index(W, d.shape[1])]
    depth = (d / float(png_depth_scale)).astype(np.float32)[None]
    return np.ascontiguousarray(color), np.ascontiguousarray(depth)
