"""CPU suite for the adversarial scenes (scenes.adversarial): the C oracle pinned against the float64 brute-force
composite on each scene's small variant, and -- on the full-size scenes the GPU suite renders -- assertions that each
scene really sits on the edge it is built for, measured with the oracle's geometry and binning.  A scene that
silently stopped exercising its edge would let a wrong cull box or sort pass the GPU tests."""
import math

import numpy as np
import pytest

import scenes
from test_oracle_cpu import check_oracle_backward, check_oracle_forward

SMALL = scenes.adversarial(small=True)
FULL = scenes.adversarial()


@pytest.mark.parametrize("name", sorted(SMALL))
def test_oracle_matches_bruteforce_on_adversarial(name):
    sc = SMALL[name]()
    check_oracle_forward(sc)
    check_oracle_backward(sc)


def _geometry(name):
    sc = FULL[name]()
    o = sc.oracle()
    return sc, o, o.geometry()


def test_needles_are_ill_conditioned():
    """2D condition numbers above 100 (after the 0.3 px^2 low-pass), many of them at 45 degrees where the conic's
    off-diagonal term is as large as the diagonal ones."""
    sc, o, geo = _geometry("needles")
    vis = geo["radii"] > 0
    a, b, c = (geo["conic_opacity"][vis, i].astype(np.float64) for i in range(3))
    root = np.sqrt(((a - c) / 2) ** 2 + b * b)
    cond = ((a + c) / 2 + root) / ((a + c) / 2 - root)
    assert (cond > 100).sum() >= 200, (cond > 100).sum()
    assert (cond > 3e3).sum() >= 50, (cond > 3e3).sum()
    assert ((cond > 100) & (np.abs(b) > 0.9 * np.sqrt(a * c))).sum() >= 100
    assert geo["radii"].max() > max(sc.w, sc.h) // 2
    # some centred outside the image
    m = geo["means2D"][vis]
    assert ((m[:, 0] < 0) | (m[:, 0] > sc.w - 1) | (m[:, 1] < 0) | (m[:, 1] > sc.h - 1)).sum() >= 20


def test_threshold_opacity_sits_on_the_alpha_threshold():
    sc, o, geo = _geometry("threshold_opacity")
    vis = geo["radii"] > 0
    op = sc.opacities.numpy().reshape(-1)
    f = np.float32(1.0 / 255.0)
    # float32(1/255) and both neighbours
    for v in (np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))):
        assert (vis & (op == v)).sum() >= 50
    # a band of op * 255 in [0.995, 1.01] on both sides of 1
    o255 = op.astype(np.float64) * 255.0
    assert (vis & (o255 >= 0.995) & (o255 < 1.0)).sum() >= 300 and (vis & (o255 > 1.0) & (o255 <= 1.01)).sum() >= 300
    # below 1/255 (cull half-extent -1) and centred strictly inside a warp's 8x4 rectangle: staged, alpha-rejected
    m = geo["means2D"].astype(np.float64)
    fx, fy = np.mod(m[:, 0], 8.0), np.mod(m[:, 1], 4.0)
    staged = vis & (o255 < 0.999) & (fx >= 1) & (fx <= 6) & (fy >= 1) & (fy <= 2) & (m[:, 0] < sc.w) & (m[:, 1] < sc.h)
    assert staged.sum() >= 500, staged.sum()


def test_near_giants_are_huge_and_frustum_clamped():
    sc, o, geo = _geometry("near_giants")
    vis = geo["radii"] > 0
    t = sc.means3D.numpy().astype(np.float64)            # identity view: camera coordinates
    clamped = (np.abs(t[:, 0] / t[:, 2]) > 1.3 * sc.tanfovx) | (np.abs(t[:, 1] / t[:, 2]) > 1.3 * sc.tanfovy)
    giant = vis & (geo["radii"] > 1000)
    assert (giant & clamped).sum() >= 30, (giant & clamped).sum()
    near = vis & (t[:, 2] <= 0.3)
    assert near.sum() >= 100 and (near & (geo["radii"] > 100)).sum() >= 100
    assert (near & (geo["radii"] > 1000)).sum() >= 10
    at_plane = np.flatnonzero(t[:, 2] == np.float32(0.2000001))          # just past the near plane's 0.2f
    assert at_plane.size >= 1 and vis[at_plane].all()
    # every clamped giant's centre is off the image, yet its tile rectangle reaches it
    m = geo["means2D"][giant & clamped]
    assert np.all((m[:, 0] < 0) | (m[:, 0] > sc.w) | (m[:, 1] < 0) | (m[:, 1] > sc.h))


@pytest.mark.parametrize("name", ["translucent_stack", "translucent_crossing"])
def test_translucent_stacks_have_long_chains(name):
    sc, o, geo = _geometry(name)
    r, b = o.render(), o.binning()
    per_tile = b["ranges"][:, 1].astype(np.int64) - b["ranges"][:, 0]
    assert per_tile.min() >= 1000, per_tile.min()
    nc = r["n_contrib"]
    assert nc.max() > 1000, nc.max()
    if name == "translucent_stack":
        assert (nc > 1000).mean() > 0.5 and r["final_T"].min() > 1e-3          # nothing saturates
    else:
        # T crosses 1e-4 (early termination) at list positions spread over many 128-record ring stages, and crosses
        # 0.5 (median depth) in some pixels but not all
        sat = r["final_T"] < 2e-4
        assert sat.mean() > 0.1 and (~sat).mean() > 0.1
        stages = np.unique(nc[sat] // 128)
        assert stages.size >= 6 and stages.min() <= 2, stages
        crossed = r["depth"][0] != 15.0
        assert crossed.mean() > 0.2 and (~crossed).sum() >= 20, crossed.mean()


def _tie_groups(depths, vis):
    """Index lists of the visible Gaussians sharing one depth, one list per depth shared by at least two."""
    d = depths.view(np.uint32)
    idx = np.flatnonzero(vis)
    _, inv, cnt = np.unique(d[idx], return_inverse=True, return_counts=True)
    return [idx[inv == g] for g in np.flatnonzero(cnt >= 2)]


@pytest.mark.parametrize("name,tile", [("depth_ties_70k", 4096), ("depth_ties_20k", 2048)])
def test_depth_ties_span_sort_tiles(name, tile):
    """Three depths shared by thousands of Gaussians each, so ties cross many onesweep tiles of the depth sort
    (4096 keys above 64K items, 2048 below), and depth pairs one ulp apart in reverse index order."""
    sc, o, geo = _geometry(name)
    vis = geo["radii"] > 0
    assert (sc.P > (64 << 10)) == (tile == 4096)
    groups = _tie_groups(geo["depths"], vis)
    big = [g for g in groups if g.size >= 1000]
    assert len(big) == 3
    for g in big:
        assert np.unique(g // tile).size >= 3 and np.unique(g // tile).size >= sc.P // tile
    # ties of the tile sort too: the same (tile | depth) key many times in one tile's list
    keys = o.binning()["keys"]
    assert (keys[1:] == keys[:-1]).sum() >= 1000
    # one-ulp pairs, the nearer Gaussian at the higher index
    d = geo["depths"].view(np.uint32).astype(np.int64)
    order = np.lexsort((np.arange(sc.P), d))
    order = order[vis[order]]
    step = np.diff(d[order])
    ulp = np.flatnonzero(step == 1)
    assert ulp.size >= 1000 and (order[ulp] > order[ulp + 1]).sum() >= 1000


def test_depth_span_moves_every_digit():
    """Depth keys from 0.2000001 to 1e5: all four 8-bit digits of the float bits vary, so no radix pass is a no-op."""
    sc, o, geo = _geometry("depth_span")
    vis = geo["radii"] > 0
    assert vis.sum() >= 0.99 * sc.P and sc.P > (64 << 10)
    d = geo["depths"][vis]
    assert d.min() <= np.float32(0.2000001) * (1 + 1e-6) and d.max() > 5e4
    u = d.view(np.uint32)
    for p in range(3):
        assert np.unique((u >> (8 * p)) & 0xFF).size >= 64, p
    assert np.unique(u >> 24).size >= 8          # sign and top exponent bits: 0.2 .. 1e5 spans 2^-3 .. 2^17
    # one-ulp pairs, the nearer Gaussian at the higher index: a sort that ignored the low bits would misorder them
    d = geo["depths"].view(np.uint32).astype(np.int64)
    order = np.lexsort((np.arange(sc.P), d))
    order = order[vis[order]]
    ulp = np.flatnonzero(np.diff(d[order]) == 1)
    assert (order[ulp] > order[ulp + 1]).sum() >= 1000


@pytest.mark.parametrize("wh", scenes.TINY_SIZES)
def test_tiny_grids(wh):
    w, h = wh
    sc, o, geo = _geometry("tiny_%dx%d" % wh)
    assert (sc.w, sc.h) == (w, h)
    assert o.tiles == math.ceil(w / 16) * math.ceil(h / 16)
    vis = geo["radii"] > 0
    assert vis.sum() >= 20 and (vis & (geo["radii"] > 3 * max(w, h))).sum() >= 3
    r = o.render()
    assert r["n_contrib"].max() >= 5


def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _fma32(x, y, z):
    """float32 fma: the product of two float32 is exact in float64, so one rounding of the sum (then to float32)."""
    return _f32(np.float64(x) * np.float64(y) + np.float64(z))


def _culled_blended_pairs(sc, geo, keep_eg=True, keep_tau_slack=True):
    """(Gaussian, pixel) pairs the reference blends (its float32 `power` and alpha >= 1/255 test, forward.cu) that the
    blend kernels' warp-rectangle box test would skip, with the box of project.cu -- optionally without its `eg`
    float-error term or its 1e-3 tau slacks.  Only the first warp column / row beyond each side of the box is
    examined: those hold the culled pixels nearest the alpha ellipse.  Pairs within 1e-6 (relative) of the alpha
    threshold are left out, so a last-ulp expf difference cannot decide a count."""
    radii = geo["radii"]
    co, m = geo["conic_opacity"], geo["means2D"]
    thr = np.float64(np.float32(1.0 / 255.0))
    gx, gy = (sc.w + 15) // 16, (sc.h + 15) // 16
    lost = 0
    for i in np.flatnonzero(radii > 0):
        a, b, c, op = (np.float64(v) for v in co[i])
        if op * 255.0 < 0.999 or not (a * c - b * b > 0 and a > 0 and c > 0):
            continue
        reach = float(radii[i]) + 17.0
        tau = np.log(op * 255.0)
        tau += (1e-3 + 1e-3 * abs(tau) if keep_tau_slack else 0.0)
        tau += (4e-6 * (abs(a) + abs(c) + 2 * abs(b)) * reach * reach if keep_eg else 0.0)
        dc = a * c - b * b
        with np.errstate(invalid="ignore"):          # tau < 0 without the slacks: NaN, which the kernel makes 1e30
            hx = np.nan_to_num(_f32(np.sqrt(2 * tau * c / dc) * 1.0001 + 2e-3), nan=1e30)
            hy = np.nan_to_num(_f32(np.sqrt(2 * tau * a / dc) * 1.0001 + 2e-3), nan=1e30)
        mx, my = np.float32(m[i, 0]), np.float32(m[i, 1])
        r = float(radii[i])
        tx0, ty0 = min(gx, max(0, int(_f32((mx - r) / 16)))), min(gy, max(0, int(_f32((my - r) / 16))))
        tx1, ty1 = min(gx, max(0, int(_f32((mx + r + 15) / 16)))), min(gy, max(0, int(_f32((my + r + 15) / 16))))
        X0, X1, Y0, Y1 = 16 * tx0, min(sc.w, 16 * tx1) - 1, 16 * ty0, min(sc.h, 16 * ty1) - 1
        right, left = _f32(mx + hx), _f32(mx - hx)
        down, up = _f32(my + hy), _f32(my - hy)
        cols = [8 * (np.floor(right / 8) + 1), 8 * (np.ceil((left - 7) / 8) - 1) + 7]
        rows = [4 * (np.floor(down / 4) + 1), 4 * (np.ceil((up - 3) / 4) - 1) + 3]
        px, py = [], []
        for x in cols:
            if X0 <= x <= X1:
                ys = np.arange(Y0, Y1 + 1)
                px.append(np.full(ys.size, x)), py.append(ys)
        for y in rows:
            if Y0 <= y <= Y1:
                xs = np.arange(X0, X1 + 1)
                px.append(xs), py.append(np.full(xs.size, y))
        if not px:
            continue
        px, py = np.concatenate(px).astype(np.float32), np.concatenate(py).astype(np.float32)
        dx, dy = _f32(mx - px), _f32(my - py)
        sxy = _fma32(dx, _f32(dx * co[i, 0]), _f32(dy * _f32(dy * co[i, 2])))
        power = _fma32(sxy, np.float32(-0.5), -_f32(dy * _f32(dx * co[i, 1])))
        alpha = np.minimum(op * np.exp(power.astype(np.float64)), 0.99)
        lost += int(((power <= 0) & (alpha >= thr * (1 + 1e-6))).sum())
    return lost


@pytest.mark.parametrize("name", ["box_edge_needles", "needles", "threshold_opacity", "near_giants",
                                  "translucent_crossing"])
def test_cull_box_holds_every_blended_pair(name):
    """Emulating the kernels' box test and the reference's float32 alpha test: the box of project.cu skips no pair
    the reference blends.  Without the box's `eg` term it would on box_edge_needles -- the scene that makes that term
    necessary.  Without the 1e-3 tau slacks it would not on any scene: `eg` >= 4e-6 (|a|+|c|+2|b|) reach^2 is over
    ten times the rounding bound of the float32 `power` over the tile rectangle, so the slacks are a second margin
    that no input can reach."""
    sc, o, geo = _geometry(name)
    assert _culled_blended_pairs(sc, geo) == 0
    assert _culled_blended_pairs(sc, geo, keep_tau_slack=False) == 0
    if name == "box_edge_needles":
        assert _culled_blended_pairs(sc, geo, keep_eg=False) >= 3
