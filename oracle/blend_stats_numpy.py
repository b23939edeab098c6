"""Numpy restatement of the blend statistics of csrc/blend_forward.cu's stats walk (sb_blend_stats; TEST
INFRASTRUCTURE ONLY), over the C oracle's projection and tile lists (oracle.Oracle).

Per pixel it walks the tile's list front to back as oracle_render does (splat_oracle.c): skip when power > 0 or
alpha = min(o exp(power), 0.99) < 1/255; test_T = T (1 - alpha); test_T < 1e-4 ENDS the walk at that Gaussian,
otherwise the Gaussian BLENDS with weight alpha T and T = test_T.  Float32 with each operation rounded as the kernel
writes it; fma is evaluated in float64 and rounded once (a rare double rounding is covered by the window below).

Threshold flags.  The GPU's expf and this file's exp differ by up to ~2.5 ulp, so a pair whose alpha or test_T sits
near a threshold may decide the other way on the GPU.  Relative error bounds:
  alpha:   EPS_ALPHA = 2e-6 (expf <= 2.5 ulp = 3e-7, the opacity multiply 1 ulp = 6e-8, a one-ulp power from the
           emulated fma at |power| <= 5.6 (alpha >= 1/255 needs it) = 7e-7; summed 1.1e-6, doubled).
  T:       grows along the walk: each blend adds (alpha / (1 - alpha)) EPS_ALPHA (the error of 1 - alpha) plus one
           rounding 2^-23, so every pixel carries its own bound err_T.
A pair is NEAR when |alpha - 1/255| <= EPS_ALPHA / 255, or when |test_T - 1e-4| <= err 1e-4 with err the bound of
test_T.  The Gaussian of a near pair is FLAGGED: its counts may differ from the GPU's.  What a flip does to the rest of
the walk:
  * at the alpha threshold, the pair blends on one side only, so T differs by the factor 1 - alpha ~ 1 - 1/255 for the
    rest of the walk: err_T grows by alpha / (1 - alpha), and later test_T decisions within that window are near;
  * at the test_T threshold, one side ends the walk here and the other blends, leaving T within err of 1e-4, so the
    next Gaussian that surely passes the alpha test (alpha >= (1 + EPS_ALPHA) / 255) ends it there: test_T <= 1e-4
    (1 + err)(1 - 1/255) < 1e-4.  Every Gaussian the list reaches up to and including that one with
    alpha >= (1 - EPS_ALPHA) / 255 is flagged; after it both walks are over.
Every other Gaussian's counts are exact, and its max_weight agrees within `max_weight_tol`, the largest absolute
error bound (EPS_ALPHA + err_T + 2^-23) alpha T over its blended pairs."""
import numpy as np

EPS_ALPHA = 2e-6
_F = np.float32
_A_MIN = _F(1.0) / _F(255.0)
_T_MIN = _F(0.0001)
_ULP = 2.0 ** -23


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(_F)


def blend_stats(oracle):
    """dict(blended uint32 [P], ended uint32 [P], max_weight float32 [P], flagged bool [P], max_weight_tol float64 [P])
    of one render of `oracle` (an oracle.Oracle)."""
    geo, binning = oracle.geometry(), oracle.binning()
    P, W, H = oracle.P, oracle.W, oracle.H
    xy, co = geo["means2D"].astype(_F), geo["conic_opacity"].astype(_F)
    plist, ranges = binning["point_list"], binning["ranges"]
    gx = (W + 15) // 16
    blended = np.zeros(P, np.uint64)
    ended = np.zeros(P, np.uint64)
    maxw = np.zeros(P, _F)
    tol = np.zeros(P, np.float64)
    flagged = np.zeros(P, bool)
    ly, lx = np.divmod(np.arange(256), 16)
    for t in range(ranges.shape[0]):
        lo, hi = int(ranges[t, 0]), int(ranges[t, 1])
        if hi <= lo:
            continue
        px, py = (t % gx) * 16 + lx, (t // gx) * 16 + ly
        inside = (px < W) & (py < H)
        pxf, pyf = px[inside].astype(_F), py[inside].astype(_F)
        n = pxf.shape[0]
        T = np.ones(n, _F)
        err_T = np.zeros(n)
        done = np.zeros(n, bool)
        open_ = np.zeros(n, bool)                # a test_T flip may let the walk reach the next sure pass
        for k in range(lo, hi):
            g = int(plist[k])
            dx, dy = xy[g, 0] - pxf, xy[g, 1] - pyf
            sxy = _fma(dx, dx * co[g, 0], dy * (dy * co[g, 2]))
            power = _fma(sxy, np.full(n, -0.5, _F), -(dy * (dx * co[g, 1])))
            ok = ~(power > 0)
            with np.errstate(over="ignore", invalid="ignore"):
                alpha = np.minimum(co[g, 3] * np.exp(power.astype(np.float64)).astype(_F), _F(0.99))
            a64 = alpha.astype(np.float64)
            passed = ok & ~(alpha < _A_MIN)
            could = ok & (a64 >= float(_A_MIN) * (1.0 - EPS_ALPHA))
            sure = ok & (a64 >= float(_A_MIN) * (1.0 + EPS_ALPHA))
            test_T = T * (_F(1.0) - alpha)
            live = ~done
            act = live & passed
            end = act & (test_T < _T_MIN)
            bl = act & ~end
            with np.errstate(divide="ignore", invalid="ignore"):
                step = np.where(ok, a64 / (1.0 - a64), 0.0)
            near_a = live & ok & (np.abs(a64 - float(_A_MIN)) <= EPS_ALPHA * float(_A_MIN))
            err_test = err_T + step * EPS_ALPHA + _ULP
            near_t = act & (np.abs(test_T.astype(np.float64) - float(_T_MIN)) <= err_test * float(_T_MIN))
            if np.any(near_a | near_t | (open_ & could)):
                flagged[g] = True
            open_ = (open_ & ~sure) | near_t
            if bl.any():
                w = alpha[bl] * T[bl]
                blended[g] += int(bl.sum())
                maxw[g] = max(maxw[g], w.max())
                tol[g] = max(tol[g], float(((EPS_ALPHA + err_T[bl] + _ULP) * w).max()))
                err_T[bl] += step[bl] * EPS_ALPHA + _ULP
            err_T[near_a] += step[near_a]
            if end.any():
                ended[g] += int(end.sum())
            T = np.where(bl, test_T, T)
            done |= end
    return dict(blended=blended.astype(np.uint32), ended=ended.astype(np.uint32), max_weight=maxw, flagged=flagged,
                max_weight_tol=tol)
