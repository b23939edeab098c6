"""Brute-force dense PyTorch alpha-composite (float64 by default) -- TEST INFRASTRUCTURE ONLY.

An independent second statement of the reference operator's semantics (SURVEY.md Appendix A,
reference files X/cuda_rasterizer/forward.cu:74-393, auxiliary.h:41-56, rasterizer_impl.cu:70-138)
written as dense [P, H*W] tensor algebra; ``torch.autograd`` supplies the backward, which pins
oracle/splat_oracle.c's hand-written backward (itself restating X/cuda_rasterizer/backward.cu).
It is BASELINE.json config[0]'s "brute-force PyTorch alpha-composite on CPU" ground truth.

Faithfulness points (SURVEY.md section 8c): tile-rectangle mask (a Gaussian only reaches pixels of
tiles inside its getRect rectangle); per-pixel order = ascending (depth, index); the pair that would
push T below 1e-4 is not blended and ends the pixel; pixel centres at integer coordinates; the
min(0.99, .) clamp passes gradient straight through (backward.cu:501-531); depth output = median
depth with default 15.0 and no gradient.
"""
import math

import torch


def _quat_to_rot(q):
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    # rows of the conventional rotation matrix Rc (== GLM R transposed in storage); used as M = S * R
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).reshape(-1, 3, 3)
    return R


def render(means3D, colors, opacities, scales, rotations, *, width, height, tanfovx, tanfovy, bg,
           viewmatrix, projmatrix, scale_modifier=1.0, means2D=None, dtype=torch.float64, rows=None,
           frozen_clamp=False):
    """Returns dict(color [3,H,W], depth [1,H,W], final_T [H,W], n_contrib [H,W], radii [P]).

    frozen_clamp=True: the backward of a Gaussian outside the 1.3 x tanfov frustum is the reference's (the clamped
    coordinate is a constant); by default autograd differentiates through the clamp, as the CPU loop fixtures
    (tests/golden/offline) were recorded.  The forward is the same either way.

    rows=(r0, r1): composite only image rows [r0, r1) (pixels are independent), returning images of height
    r1-r0 -- lets a caller walk a large image in bands with bounded memory (bench.py's brute-force timing).

    viewmatrix / projmatrix: [4,4] tensors exactly as the reference stores them (w2c transposed,
    full projection transposed), i.e. p_view = p4 @ viewmatrix.
    """
    dev = means3D.device
    P = means3D.shape[0]
    W, H = int(width), int(height)
    f = lambda t: t.to(dtype)
    m, col, op, sc, q = f(means3D), f(colors), f(opacities).reshape(-1), f(scales), f(rotations)
    V, PM, bgc = f(viewmatrix).reshape(4, 4), f(projmatrix).reshape(4, 4), f(bg).reshape(3)
    ones = torch.ones(P, 1, dtype=dtype, device=dev)
    p4 = torch.cat([m, ones], 1)
    t = (p4 @ V)[:, :3]                       # transformPoint4x3
    hom = p4 @ PM                             # transformPoint4x4
    p_w = 1.0 / (hom[:, 3] + 1e-7)
    proj = hom[:, :2] * p_w[:, None]
    depth = t[:, 2]
    in_front = depth.detach() > 0.2

    # 3D covariance Sigma = M^T M with M = S * R (GLM column-major: M[c][r] = s_r R[c][r])
    Rg = _quat_to_rot(q)                      # Rg[n, c, r] == GLM R[c][r]
    s = sc * scale_modifier
    M = Rg * s[:, None, :]                    # M[n, c, r]
    Sigma = torch.einsum('nrk,nck->ncr', M, M)    # Sigma[c][r] = sum_k M[r][k] M[c][k]

    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    tz = t[:, 2]
    txc = torch.clamp(t[:, 0] / tz, -limx, limx) * tz
    tyc = torch.clamp(t[:, 1] / tz, -limy, limy) * tz
    if frozen_clamp:
        # a coordinate clamped to the 1.3 x tanfov frustum is a constant to the reference's backward: no gradient to
        # it (x_grad_mul = 0) and none through its clamped value to tz (dL/dtz differentiates J with t.x held fixed),
        # backward.cu computeCov2DCUDA
        txz, tyz = (t[:, 0] / tz).detach(), (t[:, 1] / tz).detach()
        txc = torch.where((txz < -limx) | (txz > limx), txc.detach(), t[:, 0])
        tyc = torch.where((tyz < -limy) | (tyz > limy), tyc.detach(), t[:, 1])
    zero = torch.zeros_like(tz)
    # J (GLM columns): J[0] = (fx/tz, 0, -fx tx/tz^2), J[1] = (0, fy/tz, -fy ty/tz^2), J[2] = 0
    J = torch.stack([torch.stack([fx / tz, zero, -(fx * txc) / (tz * tz)], -1),
                     torch.stack([zero, fy / tz, -(fy * tyc) / (tz * tz)], -1),
                     torch.stack([zero, zero, zero], -1)], 1)          # J[n, c, r]
    Wm = torch.stack([V[0, 0], V[1, 0], V[2, 0], V[0, 1], V[1, 1], V[2, 1], V[0, 2], V[1, 2], V[2, 2]]).reshape(3, 3)
    # Wm[c][r] = GLM W[c][r] = view[c + 4 r] where view flat index k = V[k // 4, k % 4]
    # GLM product (A*B)[c][r] = sum_k A[k][r] B[c][k]
    T = torch.einsum('kr,nck->ncr', Wm, J)
    Tt = T.transpose(1, 2)
    St = Sigma.transpose(1, 2)
    A = torch.einsum('nkr,nck->ncr', Tt, St)
    cov = torch.einsum('nkr,nck->ncr', A, T)
    cxx, cxy, cyy = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = cxx * cyy - cxy * cxy
    det_ok = det.detach() != 0
    det_safe = torch.where(det_ok, det, torch.ones_like(det))
    con_x, con_y, con_z = cyy / det_safe, -cxy / det_safe, cxx / det_safe
    mid = 0.5 * (cxx + cyy)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    radius = torch.ceil(3.0 * torch.sqrt(torch.maximum(lam, mid - (lam - mid)))).detach()
    px = ((proj[:, 0] + 1.0) * W - 1.0) * 0.5
    py = ((proj[:, 1] + 1.0) * H - 1.0) * 0.5
    gx, gy = (W + 15) // 16, (H + 15) // 16
    pxd, pyd = px.detach(), py.detach()
    x0 = torch.clamp(torch.trunc((pxd - radius) / 16), 0, gx)
    y0 = torch.clamp(torch.trunc((pyd - radius) / 16), 0, gy)
    x1 = torch.clamp(torch.trunc((pxd + radius + 15) / 16), 0, gx)
    y1 = torch.clamp(torch.trunc((pyd + radius + 15) / 16), 0, gy)
    visible = in_front & det_ok & (((x1 - x0) * (y1 - y0)) > 0)
    radii = torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int32)

    if means2D is not None:  # gradient sink in the reference's NDC-scaled units (backward.cu:452-453,545-546)
        px = px + 0.5 * W * f(means2D)[:, 0]
        py = py + 0.5 * H * f(means2D)[:, 1]

    # per-pixel order: ascending (float32 depth bits, index) -- stable sort on the float32 depth
    order = torch.sort(depth.detach().to(torch.float32), stable=True).indices
    order = order[visible[order]]
    n = order.numel()
    r0, r1 = (0, H) if rows is None else (int(rows[0]), int(rows[1]))
    ys, xs = torch.meshgrid(torch.arange(r0, r1, device=dev), torch.arange(W, device=dev), indexing='ij')
    pixx, pixy = xs.reshape(-1).to(dtype), ys.reshape(-1).to(dtype)
    tilex, tiley = (xs.reshape(-1) // 16).to(dtype), (ys.reshape(-1) // 16).to(dtype)
    H = r1 - r0                     # from here on H is the band height (outputs are band-sized)
    HW = H * W
    if n == 0:
        color = bgc[:, None].expand(3, HW).reshape(3, H, W).clone()
        return dict(color=color, depth=torch.full((1, H, W), 15.0, dtype=dtype, device=dev),
                    final_T=torch.ones(H, W, dtype=dtype, device=dev),
                    n_contrib=torch.zeros(H, W, dtype=torch.int64, device=dev), radii=radii)

    o = order
    dx = px[o][:, None] - pixx[None, :]
    dy = py[o][:, None] - pixy[None, :]
    power = -0.5 * (con_x[o][:, None] * dx * dx + con_z[o][:, None] * dy * dy) - con_y[o][:, None] * dx * dy
    raw = op[o][:, None] * torch.exp(torch.clamp(power, max=0.0))
    alpha = raw + (torch.clamp(raw, max=0.99) - raw).detach()       # straight-through clamp
    in_rect = (tilex[None, :] >= x0[o][:, None]) & (tilex[None, :] < x1[o][:, None]) & \
              (tiley[None, :] >= y0[o][:, None]) & (tiley[None, :] < y1[o][:, None])
    valid = in_rect & (power.detach() <= 0) & (alpha.detach() >= 1.0 / 255.0)
    a = torch.where(valid, alpha, torch.zeros_like(alpha))
    one_m = 1.0 - a
    T_incl = torch.cumprod(one_m, 0)
    T_excl = torch.cat([torch.ones(1, HW, dtype=dtype, device=dev), T_incl[:-1]], 0)
    test_T = T_excl * one_m
    term = valid & (test_T.detach() < 1e-4)
    killed = torch.cumsum(term.to(torch.int32), 0) > 0
    contrib = valid & ~killed
    w = torch.where(contrib, a * T_excl, torch.zeros_like(a))        # alpha_i * T_i
    color = torch.einsum('np,nc->cp', w, col[o])
    final_T = torch.prod(torch.where(contrib, one_m, torch.ones_like(one_m)), 0)
    color = color + bgc[:, None] * final_T[None, :]
    idx1 = torch.arange(1, n + 1, device=dev)[:, None]
    # n_contrib counts positions in the pixel's TILE list (forward.cu:334,379): rank among in-rect entries
    tile_rank = torch.cumsum(in_rect.to(torch.int64), 0)
    n_contrib = torch.max(torch.where(contrib, tile_rank, torch.zeros_like(tile_rank)), 0).values
    cross = contrib & (T_excl.detach() > 0.5) & (test_T.detach() < 0.5)
    first = torch.where(cross, idx1, torch.full_like(idx1, n + 1)).expand(n, HW).min(0).values
    dsorted = depth.detach()[o].to(torch.float32).to(dtype)
    D = torch.where(first <= n, dsorted[torch.clamp(first - 1, max=n - 1)], torch.full((HW,), 15.0, dtype=dtype, device=dev))
    return dict(color=color.reshape(3, H, W), depth=D.reshape(1, H, W), final_T=final_T.reshape(H, W),
                n_contrib=n_contrib.reshape(H, W), radii=radii)
