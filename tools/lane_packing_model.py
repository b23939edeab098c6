"""CPU model of the blend kernels' warp traversal on the real bench workload (config3, 1M Gaussians, 1200x680), built on
the C oracle's geometry + binning (tools/ may use oracle/ as a checker/analysis aid; nothing here ships).

For a random sample of tiles it replays, per warp (8x4 pixel rectangle, as csrc/blend_forward.cu), the list walk with
the same conservative cull boxes as csrc/project.cu and counts what the instruction-bound kernels pay for:

  * box hits per warp            -> loop iterations of the forward (each: ~21 warp instructions)
  * hits with >= 1 active lane   -> iterations the backward cannot skip (each: ~62 + ~25 warp instructions)
  * active lanes per hit         -> lane utilisation
  * the same for alternative traversals, to rank next-round kernel work with data instead of guesses:
      - "half"  : the 8x4 rectangle split into two 4x4 halves with separate hit lists, one Gaussian per half per
                  iteration (iterations per 32-record chunk = max(|hits L|, |hits R|))
      - "exact" : an exact ellipse-vs-rectangle test instead of the bounding box (upper bound on what better culling buys)
      - "4x8"   : 4-wide x 8-tall rectangles instead of 8x4 (isotropic splats: same)

`cover_masks` restates csrc/binning.cu's per-instance coverage masks, which the shipped kernels cull with; the
tests/test_cover_mask_*.py suites check the device masks and the per-pixel alpha test against it.

Run:  python tools/lane_packing_model.py [--tiles 150] [--gaussians 1000000]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import scenes  # noqa: E402


def cull_half_extents(conic, opacity, radius):
    """hx, hy of csrc/project.cu (double arithmetic, same slack terms); -1 = contributes nowhere."""
    a, b, c = conic[:, 0].astype(np.float64), conic[:, 1].astype(np.float64), conic[:, 2].astype(np.float64)
    op = opacity.astype(np.float64)
    hx = np.full(a.shape, -1.0)
    hy = np.full(a.shape, -1.0)
    ok = op * 255.0 >= 0.999
    reach = radius.astype(np.float64) + 17.0
    eg = 4e-6 * (np.abs(a) + np.abs(c) + 2.0 * np.abs(b)) * reach * reach
    tau = np.log(np.maximum(op * 255.0, 1e-30))
    tau = tau + 1e-3 + 1e-3 * np.abs(tau) + eg
    dc = a * c - b * b
    good = ok & (dc > 0) & (a > 0) & (c > 0)
    hx[good] = np.sqrt(2.0 * tau[good] * c[good] / dc[good]) * 1.0001 + 2e-3
    hy[good] = np.sqrt(2.0 * tau[good] * a[good] / dc[good]) * 1.0001 + 2e-3
    hx[ok & ~good] = 1e30
    hy[ok & ~good] = 1e30
    return hx, hy


def cull_half_extents_f32(conic, opacity, radius):
    """hx, hy as csrc/project.cu stores them: rounded to float32, anything not below 1e30 clamped to 1e30."""
    with np.errstate(over="ignore", invalid="ignore"):
        out = [h.astype(np.float32) for h in cull_half_extents(conic, opacity, radius)]
    return [np.where(h < np.float32(1e30), h, np.float32(1e30)) for h in out]


def cover_masks(xy, conic, hx, hy, tile, grid_x, near_rel=1e-6):
    """Per tile instance, the 8-bit coverage mask of csrc/binning.cu (cover_mask), restated in numpy with the same
    float32 box comparisons and the same float64 operations in the same order: bit w stands for the blend kernels'
    warp w, pixel centres x0..x0+7 by y0..y0+3 with x0 = 16 tx + 8 (w & 1), y0 = 16 ty + 4 (w >> 1).

    xy [n,2] and conic [n,3] float32 as the projection stores them, hx, hy [n] float32 (cull_half_extents_f32), tile [n]
    tile ids.  Returns (mask, box, near), uint8 [n] each: the coverage mask; the box test alone, of which the mask is a
    subset; and the bits whose decision lies within a relative `near_rel` of a threshold (where a last-ulp difference
    in hx, hy between this model and the device can flip the bit)."""
    xy = np.asarray(xy, np.float32)
    gx32, gy32 = xy[:, 0], xy[:, 1]
    hx32, hy32 = np.asarray(hx, np.float32), np.asarray(hy, np.float32)
    gx, gy = gx32.astype(np.float64), gy32.astype(np.float64)
    a, b, c = (np.asarray(conic[:, k], np.float32).astype(np.float64) for k in range(3))
    hx64, hy64 = hx32.astype(np.float64), hy32.astype(np.float64)
    tile = np.asarray(tile, np.int64)
    tx, ty = tile % grid_x, tile // grid_x
    dc = a * c - b * b
    thr_x, thr_y = dc * (hx64 * hx64), dc * (hy64 * hy64)
    culled = ~(hx32 > 0)
    skip = (hx32 >= np.float32(1e30)) | (hy32 >= np.float32(1e30))
    mask, box_all, near = (np.zeros(tile.shape, np.uint8) for _ in range(3))

    def close(x, y):
        return np.abs(x - y) <= near_rel * np.maximum(np.abs(x), np.abs(y))

    with np.errstate(invalid="ignore", over="ignore"):
        for w in range(8):
            x0, y0 = tx * 16 + (w & 1) * 8, ty * 16 + (w >> 1) * 4
            fx0, fx1, fy0, fy1 = (v.astype(np.float32) for v in (x0, x0 + 7, y0, y0 + 3))
            lx, rx, ly, ry = gx32 + hx32, gx32 - hx32, gy32 + hy32, gy32 - hy32
            box = (lx >= fx0) & (rx <= fx1) & (ly >= fy0) & (ry <= fy1)
            box_near = (close(lx, fx0) | close(rx, fx1) | close(ly, fy0) | close(ry, fy1))
            u0, u1 = gx - (x0 + 7.0), gx - x0
            v0, v1 = gy - (y0 + 3.0), gy - y0
            inside = (u0 <= 0) & (u1 >= 0) & (v0 <= 0) & (v1 >= 0)
            hv, hu = (v0 > 0) | (v1 < 0), (u0 > 0) | (u1 < 0)
            v = np.where(v0 > 0, v0, v1)
            bv = b * v
            d = np.maximum(np.maximum(a * u0 + bv, -(a * u1 + bv)), 0.0)
            sh = d * d + dc * v * v
            u = np.where(u0 > 0, u0, u1)
            bu = b * u
            d = np.maximum(np.maximum(c * v0 + bu, -(c * v1 + bu)), 0.0)
            sv = d * d + dc * u * u
            ell = inside | (hv & (sh <= thr_y)) | (hu & (sv <= thr_x))
            ell_near = (hv & close(sh, thr_y)) | (hu & close(sv, thr_x))
            bit = box & ~culled & (skip | ell)
            mask |= bit.astype(np.uint8) << w
            box_all |= box.astype(np.uint8) << w
            near |= ((box_near | (box & ~skip & ell_near)) & ~culled).astype(np.uint8) << w
    return mask, box_all, near


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=150)
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    sc = scenes.config3(P=args.gaussians)
    o = sc.oracle()
    geo, b = o.geometry(), o.binning()
    xy, co, radii = geo["means2D"], geo["conic_opacity"], geo["radii"]
    hx, hy = cull_half_extents(co[:, :3], co[:, 3], radii)
    ranges, plist = b["ranges"], b["point_list"]
    gx = (sc.w + 15) // 16
    rng = np.random.default_rng(args.seed)
    nonempty = np.nonzero(ranges[:, 1] > ranges[:, 0])[0]
    sample = rng.choice(nonempty, size=min(args.tiles, nonempty.size), replace=False)

    tot = dict(entries=0, fwd_entries=0, hits=0, hits_bwd=0, any_active=0, active_lanes=0, pairs_eval=0,
               half_iters=0, half_iters_bwd=0, half_any=0, exact_hits=0, chunks=0, hits48=0)
    px = np.arange(16, dtype=np.float32)
    for t in sample:
        lo, hi = int(ranges[t, 0]), int(ranges[t, 1])
        ids = plist[lo:hi]
        n = ids.size
        tx, ty = int(t % gx), int(t // gx)
        X = (tx * 16 + px)[None, None, :]                     # [1,1,16]
        Y = (ty * 16 + px)[None, :, None]                     # [1,16,1]
        gxy, gco = xy[ids], co[ids]
        dx = gxy[:, 0][:, None, None] - X                     # float32, as the kernels
        dy = gxy[:, 1][:, None, None] - Y
        power = -0.5 * (gco[:, 0][:, None, None] * dx * dx + gco[:, 2][:, None, None] * dy * dy) - gco[:, 1][:, None, None] * dx * dy
        alpha = np.minimum(0.99, gco[:, 3][:, None, None] * np.exp(np.minimum(power, 0.0)))
        contrib = (power <= 0) & (alpha >= 1.0 / 255.0)                                   # [n,16,16]
        valid = (Y < sc.h) & (X < sc.w)
        contrib &= valid
        # per-pixel termination as the reference: stop before the pair that would push T below 1e-4
        one_m = np.where(contrib, 1.0 - alpha, 1.0).astype(np.float64)
        T_incl = np.cumprod(one_m, axis=0)
        stop = contrib & (T_incl < 1e-4)
        stopped = np.cumsum(stop, axis=0) > 0                                              # from the stopping entry on
        live = contrib & ~stopped
        idx1 = np.arange(1, n + 1)[:, None, None]
        n_contrib = np.max(np.where(live, idx1, 0), axis=0)                                # [16,16]
        done_at = np.where(stopped.any(axis=0), np.argmax(stopped, axis=0) + 1, n)         # entries the pixel looks at
        hxs, hys = hx[ids], hy[ids]
        for w in range(8):
            x0, y0 = tx * 16 + (w & 1) * 8, ty * 16 + (w >> 1) * 4
            sl = (slice(None), slice((w >> 1) * 4, (w >> 1) * 4 + 4), slice((w & 1) * 8, (w & 1) * 8 + 8))
            fwd_n = int(done_at[sl[1], sl[2]].max())          # the forward warp walks until its last pixel is done
            bwd_n = int(n_contrib[sl[1], sl[2]].max())        # the backward warp walks entries < max n_contrib
            box = (gxy[:, 0] + hxs >= x0) & (gxy[:, 0] - hxs <= x0 + 7) & (gxy[:, 1] + hys >= y0) & (gxy[:, 1] - hys <= y0 + 3)
            act = live[sl]                                     # [n,4,8] lanes that blend this entry
            anyact = act.reshape(n, -1).any(axis=1)
            tot["entries"] += n
            tot["fwd_entries"] += fwd_n
            tot["hits"] += int(box[:fwd_n].sum())
            tot["hits_bwd"] += int(box[:bwd_n].sum())
            tot["any_active"] += int((box[:bwd_n] & anyact[:bwd_n]).sum())
            tot["active_lanes"] += int(act[:bwd_n][box[:bwd_n]].sum())
            tot["pairs_eval"] += int(box[:fwd_n].sum()) * 32
            # exact test: does any pixel of the rectangle pass the alpha test (ignoring termination)
            ex = contrib[sl].reshape(n, -1).any(axis=1)
            tot["exact_hits"] += int(ex[:fwd_n].sum())
            # two 4x4 halves with their own boxes
            boxL = (gxy[:, 0] + hxs >= x0) & (gxy[:, 0] - hxs <= x0 + 3) & (gxy[:, 1] + hys >= y0) & (gxy[:, 1] - hys <= y0 + 3)
            boxR = (gxy[:, 0] + hxs >= x0 + 4) & (gxy[:, 0] - hxs <= x0 + 7) & (gxy[:, 1] + hys >= y0) & (gxy[:, 1] - hys <= y0 + 3)
            for limit, key in ((fwd_n, "half_iters"), (bwd_n, "half_iters_bwd")):
                for c0 in range(0, limit, 32):
                    c1 = min(limit, c0 + 32)
                    tot[key] += max(int(boxL[c0:c1].sum()), int(boxR[c0:c1].sum()))
                    if key == "half_iters":
                        tot["chunks"] += 1
            actL = act[:, :, :4].reshape(n, -1).any(axis=1)
            actR = act[:, :, 4:].reshape(n, -1).any(axis=1)
            tot["half_any"] += int((boxL[:bwd_n] & actL[:bwd_n]).sum()) + int((boxR[:bwd_n] & actR[:bwd_n]).sum())
        # 4 wide x 8 tall rectangles
        for w in range(8):
            x0, y0 = tx * 16 + (w & 3) * 4, ty * 16 + (w >> 2) * 8
            fwd_n = int(done_at[(w >> 2) * 8:(w >> 2) * 8 + 8, (w & 3) * 4:(w & 3) * 4 + 4].max())
            box = (gxy[:, 0] + hxs >= x0) & (gxy[:, 0] - hxs <= x0 + 3) & (gxy[:, 1] + hys >= y0) & (gxy[:, 1] - hys <= y0 + 7)
            tot["hits48"] += int(box[:fwd_n].sum())

    scale = ranges.shape[0] / 1.0     # informational only
    nt = sample.size
    per = lambda k: tot[k] / (nt * 8)
    print(f"workload: config3, P={sc.P}, R={o.R}, tiles sampled {nt} of {nonempty.size} non-empty")
    print(f"per warp (mean over {nt * 8} warps):")
    print(f"  list entries in the tile                      {per('entries'):9.1f}")
    print(f"  entries walked before the warp is done (fwd)  {per('fwd_entries'):9.1f}")
    print(f"  box hits, forward  (8x4 rectangle)            {per('hits'):9.1f}")
    print(f"  box hits, backward (entries < max n_contrib)  {per('hits_bwd'):9.1f}")
    print(f"  ... with at least one blending lane           {per('any_active'):9.1f}   ({100 * tot['any_active'] / max(tot['hits_bwd'], 1):.1f} % of the backward hits)")
    print(f"  blending lanes per backward hit               {tot['active_lanes'] / max(tot['hits_bwd'], 1):9.2f} of 32")
    print(f"  exact ellipse-vs-rectangle hits (fwd bound)   {per('exact_hits'):9.1f}   ({100 * tot['exact_hits'] / max(tot['hits'], 1):.1f} % of the box hits)")
    print(f"  4x8 rectangles instead of 8x4: box hits       {per('hits48'):9.1f}")
    print(f"  two 4x4 halves: iterations, forward           {per('half_iters'):9.1f}   ({100 * tot['half_iters'] / max(tot['hits'], 1):.1f} % of today's)")
    print(f"  two 4x4 halves: iterations, backward          {per('half_iters_bwd'):9.1f}   ({100 * tot['half_iters_bwd'] / max(tot['hits_bwd'], 1):.1f} % of today's)")
    print(f"  two 4x4 halves: (half, Gaussian) reductions   {per('half_any'):9.1f}   ({100 * tot['half_any'] / max(tot['any_active'], 1):.1f} % of today's per-warp reductions)")
    tiles_total = nonempty.size
    print("extrapolated to the image (x non-empty tiles x 8 warps):")
    print(f"  forward iterations  {per('hits') * tiles_total * 8 / 1e6:7.2f} M   backward iterations {per('hits_bwd') * tiles_total * 8 / 1e6:7.2f} M"
          f"   surviving pairs {per('any_active') * tiles_total * 8 / 1e6:7.2f} M")


if __name__ == "__main__":
    main()
