"""CPU suite for the per-instance coverage masks the blend kernels cull with (csrc/binning.cu, cover_mask), through
their numpy restatement in tools/lane_packing_model.py: on the C oracle's geometry and binning, no (warp, Gaussian) pair
with a pixel that passes the kernels' float32 alpha test may have its bit cleared, and every mask is a subset of the
projection kernel's box test.  The forward's bit-equality on the GPU depends on the first property."""
import numpy as np
import pytest

import scenes
from util import load

M = load("tools/lane_packing_model.py")


def blended_pairs(xy, co, tile, grid_x, W, H):
    """uint8 [n]: bit w set iff the Gaussian passes the blend kernels' per-pixel test (power <= 0, alpha >= 1/255,
    float32 in the kernels' operation order) at some in-image pixel of warp w's 8x4 rectangle of its tile."""
    f32 = np.float32
    gx, gy = xy[:, 0].astype(f32)[:, None, None], xy[:, 1].astype(f32)[:, None, None]
    a, b, c, op = (co[:, k].astype(f32)[:, None, None] for k in range(4))
    tile = np.asarray(tile, np.int64)
    tx, ty = (tile % grid_x)[:, None, None], (tile // grid_x)[:, None, None]
    r = np.arange(16)
    px, py = tx * 16 + r[None, None, :], ty * 16 + r[None, :, None]
    dx, dy = gx - px.astype(f32), gy - py.astype(f32)
    # __fmaf_rn(dx, dx*a, dy*(dy*c)): the product of two floats is exact in float64, one rounding to float32 after
    sxy = (dx.astype(np.float64) * (dx * a).astype(np.float64) + (dy * (dy * c)).astype(np.float64)).astype(f32)
    power = sxy * f32(-0.5) + (-(dy * (dx * b)))
    with np.errstate(over="ignore", invalid="ignore"):
        alpha = np.minimum(op * np.exp(power), f32(0.99))
    hit = ~(power > 0) & ~(alpha < f32(1.0) / f32(255.0)) & (px < W) & (py < H)     # [n,16,16]
    out = np.zeros(tile.shape, np.uint8)
    for w in range(8):
        ys, xs = (w >> 1) * 4, (w & 1) * 8
        out |= hit[:, ys:ys + 4, xs:xs + 8].any(axis=(1, 2)).astype(np.uint8) << w
    return out


def check_scene(sc, n_tiles, seed=0):
    """Mask rule against the per-pixel test on `n_tiles` sampled non-empty tiles (all of them if fewer).  Returns
    (pairs the mask keeps, pairs the box keeps, pairs that blend) over the sample."""
    o = sc.oracle()
    geo, b = o.geometry(), o.binning()
    xy, co, radii = geo["means2D"], geo["conic_opacity"], geo["radii"]
    hx, hy = M.cull_half_extents_f32(co[:, :3], co[:, 3], radii)
    ranges, plist = b["ranges"], b["point_list"]
    grid_x = (sc.w + 15) // 16
    nonempty = np.nonzero(ranges[:, 1] > ranges[:, 0])[0]
    rng = np.random.default_rng(seed)
    sample = nonempty if nonempty.size <= n_tiles else rng.choice(nonempty, size=n_tiles, replace=False)
    kept = boxed = blended = 0
    for t in sample:
        ids = plist[int(ranges[t, 0]):int(ranges[t, 1])]
        tile = np.full(ids.shape, t)
        mask, box, _ = M.cover_masks(xy[ids], co[ids, :3], hx[ids], hy[ids], tile, grid_x)
        blend = blended_pairs(xy[ids], co[ids], tile, grid_x, sc.w, sc.h)
        assert not (mask & ~box).any(), "a coverage bit outside the box test (tile %d)" % t
        dropped = blend & ~mask
        assert not dropped.any(), "tile %d: %d (warp, Gaussian) pairs blend but their bit is clear" % (
            t, int(np.unpackbits(dropped).sum()))
        kept += int(np.unpackbits(mask).sum())
        boxed += int(np.unpackbits(box).sum())
        blended += int(np.unpackbits(blend).sum())
    return kept, boxed, blended


def test_config3_masks_cover_every_blended_pair_and_cull_more_than_the_box():
    kept, boxed, blended = check_scene(scenes.config3(), 120)
    assert blended <= kept < 0.95 * boxed, (blended, kept, boxed)


@pytest.mark.parametrize("name", sorted(scenes.adversarial()))
def test_adversarial_masks_cover_every_blended_pair(name):
    check_scene(scenes.adversarial()[name](), 80)


@pytest.mark.parametrize("anisotropic", [False, True])
def test_view_filling_masks_cover_every_blended_pair(anisotropic):
    check_scene(scenes.view_filling(anisotropic=anisotropic), 60, seed=1)


def test_cover_masks_edge_values():
    """hx = -1 clears the mask even where the box test passes (centre inside the rectangle); hx = 1e30 keeps the box;
    NaN geometry culls."""
    xy = np.array([[3.5, 1.5], [3.5, 1.5], [np.nan, 1.5]], np.float32)
    conic = np.array([[1.0, 0.0, 1.0]] * 3, np.float32)
    hx = np.array([-1.0, 1e30, 2.0], np.float32)
    hy = np.array([-1.0, 1e30, 2.0], np.float32)
    mask, box, _ = M.cover_masks(xy, conic, hx, hy, np.zeros(3, np.int64), 4)
    assert box[0] == 1 and mask[0] == 0
    assert mask[1] == box[1] == 0xFF
    assert box[2] == 0 and mask[2] == 0
