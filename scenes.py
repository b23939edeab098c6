"""Synthetic scenes and cameras for BASELINE.json's configs (SURVEY.md section 8d).

Shared by tests/, bench.py, __graft_entry__.smoke() and tests/golden/make_golden.py.  Everything is
generated on the CPU with a seeded ``torch.Generator`` so the GPU box, this container and the golden
fixtures all see bit-identical inputs.  No dataset access (Replica / TUM are not available offline);
`write_replica_sequence` renders a synthetic sequence on the GPU and writes it in Replica's on-disk layout.
"""
import math

import numpy as np
import torch


def camera_matrices(w, h, fx, fy, cx, cy, w2c=None, near=0.01, far=100.0):
    """Float32 (viewmatrix, projmatrix, campos) exactly as R/utils/recon_helpers.py:4-27 builds them
    (w2c transposed; full projection = w2c^T @ opengl_proj^T), computed on the CPU."""
    w2c = torch.eye(4) if w2c is None else torch.as_tensor(w2c, dtype=torch.float32)
    w2c = w2c.float()
    cam_center = torch.inverse(w2c)[:3, 3]
    view = w2c.unsqueeze(0).transpose(1, 2)
    opengl_proj = torch.tensor([[2 * fx / w, 0.0, -(w - 2 * cx) / w, 0.0],
                                [0.0, 2 * fy / h, -(h - 2 * cy) / h, 0.0],
                                [0.0, 0.0, far / (far - near), -(far * near) / (far - near)],
                                [0.0, 0.0, 1.0, 0.0]]).float().unsqueeze(0).transpose(1, 2)
    full_proj = view.bmm(opengl_proj)
    return view.contiguous(), full_proj.contiguous(), cam_center.contiguous()


class Scene:
    """Inputs of one raster call in the operator's own parametrisation (post-exp scales,
    post-sigmoid opacities, normalised quaternions), as CPU float32 tensors."""

    def __init__(self, name, w, h, fx, fy, cx, cy, means3D, colors, opacities, scales, rotations,
                 w2c=None, bg=(0.0, 0.0, 0.0)):
        self.name, self.w, self.h = name, int(w), int(h)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.means3D, self.colors, self.opacities = means3D.float(), colors.float(), opacities.float().reshape(-1, 1)
        self.scales, self.rotations = scales.float(), rotations.float()
        self.view, self.proj, self.campos = camera_matrices(w, h, fx, fy, cx, cy, w2c)
        self.bg = torch.tensor(bg, dtype=torch.float32)
        self.tanfovx, self.tanfovy = w / (2 * fx), h / (2 * fy)

    @property
    def P(self):
        return self.means3D.shape[0]

    def settings(self, cls, device):
        """Build a GaussianRasterizationSettings-like NamedTuple of class `cls` on `device`."""
        return cls(image_height=self.h, image_width=self.w, tanfovx=self.tanfovx, tanfovy=self.tanfovy,
                   bg=self.bg.to(device), scale_modifier=1.0, viewmatrix=self.view.to(device),
                   projmatrix=self.proj.to(device), sh_degree=0, campos=self.campos.to(device), prefiltered=False)

    def inputs(self, device, requires_grad=False):
        d = dict(means3D=self.means3D, colors_precomp=self.colors, opacities=self.opacities, scales=self.scales,
                 rotations=self.rotations)
        out = {k: v.to(device).clone().requires_grad_(requires_grad) for k, v in d.items()}
        out["means2D"] = torch.zeros_like(out["means3D"], requires_grad=requires_grad)
        return out

    def oracle_cam(self):
        from oracle import oracle as O
        return O.make_cam(self.w, self.h, self.tanfovx, self.tanfovy, self.bg.numpy(), self.view.numpy().reshape(-1),
                          self.proj.numpy().reshape(-1))

    def oracle(self):
        from oracle import oracle as O
        return O.Oracle(self.oracle_cam(), self.means3D.numpy(), self.colors.numpy(), self.opacities.numpy(),
                        self.scales.numpy(), self.rotations.numpy())


def _rand(gen, *shape):
    return torch.rand(*shape, generator=gen)


def config1(seed=0, P=256, w=64, h=64, bg=(0.0, 0.0, 0.0)):
    """BASELINE config[0]: 256 mixed isotropic/anisotropic Gaussians, 64x64, fx=fy=64 (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)
    fx = fy = 64.0 * w / 64.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u = -4.0 + (w + 8.0) * _rand(g, P)
    v = -4.0 + (h + 8.0) * _rand(g, P)
    means = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    s = 0.5 + 5.5 * _rand(g, P, 3)
    half = P // 2
    s[:half] = s[:half, :1]
    scales = s * z[:, None] / fx
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    q[:half] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    opac = torch.sigmoid(1.5 * torch.randn(P, generator=g))
    col = _rand(g, P, 3)
    return Scene("config1", w, h, fx, fy, cx, cy, means, col, opac, scales, q, bg=bg)


REPLICA = dict(w=1200, h=680, fx=600.0, fy=600.0, cx=599.5, cy=339.5)      # R/configs/data/replica.yaml
TUM_FR1 = dict(w=640, h=480, fx=517.3, fy=516.5, cx=318.6, cy=255.3)       # R/configs/data/TUM/freiburg1_desk.yaml


def config3(seed=2, P=1_000_000, cam=REPLICA, sigma_px=(0.7, 2.5), zr=(1.0, 5.0)):
    """BASELINE config[2]: P isotropic Gaussians, Replica intrinsics, sigma_px~U(0.7,2.5), z~U(1,5),
    opacity~U(.05,.95), colour~U(0,1) (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)
    w, h, fx, fy, cx, cy = cam["w"], cam["h"], cam["fx"], cam["fy"], cam["cx"], cam["cy"]
    z = zr[0] + (zr[1] - zr[0]) * _rand(g, P)
    u, v = w * _rand(g, P), h * _rand(g, P)
    means = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    sig = sigma_px[0] + (sigma_px[1] - sigma_px[0]) * _rand(g, P)
    scales = (sig * z / fx)[:, None].repeat(1, 3)
    q = torch.zeros(P, 4)
    q[:, 0] = 1.0
    opac = 0.05 + 0.9 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("config3_%d" % P, w, h, fx, fy, cx, cy, means, col, opac, scales, q)


def room(seed=1, P=50_000, cam=REPLICA, anisotropic=False, w2c=None):
    """BASELINE config[1]-like "room": points on the faces of a 6x4x3 m box around the camera plus
    clutter, sigma ~1.5-3 px, opacity 0.9 (SURVEY.md 8d config 2); also used for TUM-sized scenes."""
    g = torch.Generator().manual_seed(seed)
    w, h, fx, fy, cx, cy = cam["w"], cam["h"], cam["fx"], cam["fy"], cam["cx"], cam["cy"]
    n_wall = int(P * 0.85)
    face = torch.randint(0, 6, (n_wall,), generator=g)
    a, b = _rand(g, n_wall) * 2 - 1, _rand(g, n_wall) * 2 - 1
    half = torch.tensor([3.0, 2.0, 1.5])
    pts = torch.zeros(n_wall, 3)
    for f in range(6):
        m = face == f
        ax = f // 2
        sgn = 1.0 if f % 2 else -1.0
        o = [i for i in range(3) if i != ax]
        pts[m, ax] = sgn * half[ax]
        pts[m, o[0]] = a[m] * half[o[0]]
        pts[m, o[1]] = b[m] * half[o[1]]
    clutter = (torch.rand(P - n_wall, 3, generator=g) * 2 - 1) * half * 0.8
    pts = torch.cat([pts, clutter], 0)
    # camera at the origin looking down +z (x right, y down), as SplaTAM's first frame
    z = pts[:, 2].clamp(min=0.05)
    sig = 1.5 + 1.5 * _rand(g, P)
    base = sig * z.abs().clamp(min=0.3) / fx
    if anisotropic:
        scales = base[:, None] * (0.4 + 1.6 * _rand(g, P, 3))
        q = torch.randn(P, 4, generator=g)
        q = q / q.norm(dim=1, keepdim=True)
    else:
        scales = base[:, None].repeat(1, 3)
        q = torch.zeros(P, 4)
        q[:, 0] = 1.0
    opac = torch.full((P,), 0.9)
    col = 0.5 + 0.5 * torch.sin(pts * 3.0 + torch.tensor([0.0, 2.0, 4.0]))
    return Scene("room_%d" % P, w, h, fx, fy, cx, cy, pts, col, opac, scales, q, w2c=w2c)


def _surface_depth(u, v):
    """Smooth synthetic depth map (metres) standing in for a Replica / TUM depth frame."""
    return 2.5 + 0.8 * torch.sin(u / 130.0) * torch.cos(v / 90.0) + 0.3 * torch.sin(u / 23.0 + v / 31.0)


def view_filling(seed=12, cam=REPLICA, P=None, stride=1, anisotropic=False, w2c=None, opacity=(0.45, 0.6), margin=0,
                 cover=False):
    """A map that FILLS the view the way SplaTAM's maps do: one Gaussian per pixel of the first frame,
    back-projected through the depth map, sigma_world = depth / f (one pixel std on screen), logit opacity ~ 0
    (R/scripts/splatam.py:67-118,120-157,196-203: get_pointcloud + initialize_params with the "projective"
    mean_sq_dist), plus -- when P exceeds the pixel count -- further Gaussians at random sub-pixel positions of the
    same surface with sizes 0.8-1.3 px, standing in for the back-projections that later keyframes add
    (R/scripts/splatam.py:378-420).  Every Gaussian is in view, so num_rendered ~ 2 x P and every tile list is
    hundreds of entries long -- unlike `room`, where ~97 % of the Gaussians lie outside the frustum."""
    g = torch.Generator().manual_seed(seed)
    w, h, fx, fy, cx, cy = cam["w"], cam["h"], cam["fx"], cam["fy"], cam["cx"], cam["cy"]
    # margin > 0 extends the surface beyond the image borders (pixels), so a moving camera keeps seeing a covered view
    vv, uu = torch.meshgrid(torch.arange(-margin, h + margin, stride, dtype=torch.float32),
                            torch.arange(-margin, w + margin, stride, dtype=torch.float32), indexing="ij")
    u, v = uu.reshape(-1), vv.reshape(-1)
    n_grid = u.numel()
    P = n_grid if P is None else int(P)
    if P < n_grid:
        keep = torch.randperm(n_grid, generator=g)[:P].sort().values
        u, v = u[keep], v[keep]
        # cover: a map with fewer Gaussians than pixels still fills the view (as a map built at a lower densification
        # resolution does): splat size grows with the pixel spacing
        size = torch.full((P,), math.sqrt(n_grid / P) if cover else 1.0)
    else:
        extra = P - n_grid
        u = torch.cat([u, -margin + (w + 2 * margin) * _rand(g, extra)])
        v = torch.cat([v, -margin + (h + 2 * margin) * _rand(g, extra)])
        size = torch.cat([torch.ones(n_grid), 0.8 + 0.5 * _rand(g, extra)])
    z = _surface_depth(u, v) * (1.0 + 0.004 * torch.randn(P, generator=g))
    means = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    base = size * z / ((fx + fy) / 2.0)
    if anisotropic:
        scales = base[:, None] * (0.5 + 1.0 * _rand(g, P, 3))
        q = torch.randn(P, 4, generator=g)
        q = q / q.norm(dim=1, keepdim=True)
    else:
        scales = base[:, None].repeat(1, 3)
        q = torch.zeros(P, 4)
        q[:, 0] = 1.0
    opac = opacity[0] + (opacity[1] - opacity[0]) * _rand(g, P)
    col = 0.5 + 0.5 * torch.sin(means * 6.0 + torch.tensor([0.0, 2.0, 4.0]))
    return Scene("view_filling_%d" % P, w, h, fx, fy, cx, cy, means, col, opac, scales, q, w2c=w2c)


def edge_cases(seed=5, w=97, h=45):
    """Ragged image size (not a multiple of 16), Gaussians behind / on the near plane, far off-screen,
    huge and sub-pixel splats, opacity below 1/255, exact depth ties, non-zero background, and a
    non-identity view matrix."""
    g = torch.Generator().manual_seed(seed)
    P = 300
    fx = fy = 80.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 0.5 + 3.0 * _rand(g, P)
    u, v = -30 + (w + 60) * _rand(g, P), -30 + (h + 60) * _rand(g, P)
    means = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    means[:10, 2] = -1.0                      # behind the camera
    means[10:14, 2] = 0.2                     # exactly on the near plane (culled: z <= 0.2)
    means[14:18, 2] = 0.2000001               # just inside
    means[20:40, 2] = 2.0                     # exact depth ties -> order by index
    s = (0.3 + 4 * _rand(g, P, 3)) * z[:, None] / fx
    s[40:44] *= 40.0                          # huge splats covering the whole image
    s[44:50] *= 0.01                          # sub-pixel
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    opac = _rand(g, P)
    opac[50:56] = 0.003                       # below 1/255: never contributes
    opac[56:60] = 1.0
    col = _rand(g, P, 3)
    ang = 0.1
    w2c = torch.tensor([[math.cos(ang), 0, math.sin(ang), 0.05], [0, 1, 0, -0.02],
                        [-math.sin(ang), 0, math.cos(ang), 0.1], [0, 0, 0, 1]], dtype=torch.float32)
    return Scene("edge", w, h, fx, fy, cx, cy, means, col, opac, s, q, w2c=w2c, bg=(0.2, 0.5, 0.7))


def dense_opaque(seed=7, P=4000, w=128, h=96):
    """Many near-opaque overlapping splats so pixels saturate (T < 1e-4) and the early-out paths run."""
    g = torch.Generator().manual_seed(seed)
    fx = fy = 100.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 2.0 * _rand(g, P)
    u, v = w * _rand(g, P), h * _rand(g, P)
    means = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    s = (3.0 + 5.0 * _rand(g, P, 3)) * z[:, None] / fx
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    opac = 0.9 + 0.1 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("dense", w, h, fx, fy, cx, cy, means, col, opac, s, q)


# ---- adversarial scenes: inputs built to sit on the edges of the blend kernels' cull boxes (project.cu), the
# two-level depth/tile sort (binning.cu, radix_sort.cu) and the backward's contributor windows.  Every generator
# takes `small=True` for a variant the float64 brute-force composite (oracle/bruteforce_torch.py) can afford.

def _unproject(u, v, z, fx, fy, cx, cy):
    """World = camera coordinates (identity w2c) of pixel (u, v) at depth z."""
    return torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)


def _quat_z(theta):
    """Rotation by `theta` about the camera axis: an in-image rotation of the splat."""
    return torch.stack([torch.cos(theta / 2), torch.zeros_like(theta), torch.zeros_like(theta), torch.sin(theta / 2)], 1)


def _random_quat(g, n):
    q = torch.randn(n, 4, generator=g)
    return q / q.norm(dim=1, keepdim=True)


def needles(seed=31, small=False):
    """Needle-like splats, 2D condition numbers up to ~1e4 (box_edge_needles goes to 1e6, for its forward only):
    a third long needles at 45 / 135 degrees (where the
    conic's off-diagonal term is largest and the float evaluation of `power` cancels hardest), a third at uniform
    in-image angles, a third with random 3D rotations; opacity 0.9-0.999 (largest tau), centres up to 12 px outside
    the image."""
    g = torch.Generator().manual_seed(seed)
    w, h, P = (48, 32, 60) if small else (256, 192, 600)
    fx = fy = w * 0.625
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u, v = -12 + (w + 24) * _rand(g, P), -12 + (h + 24) * _rand(g, P)
    k = P // 3
    long_px = torch.cat([(w / 16) + (w / 5) * _rand(g, k), 4.0 + (w / 6) * _rand(g, P - k)])
    # 10:1 .. 1000:1 in 3D; the small variant stops at ~30:1, past which the float32 conic (the reference's and
    # the oracle's) departs from the float64 brute-force composite by more than ulp-level noise
    ratio = 10.0 ** (1.0 + (0.5 if small else 2.0) * _rand(g, P))
    s_px = torch.stack([long_px, long_px / ratio, long_px / ratio], 1)
    theta = torch.where(torch.arange(P) % 2 == 0, torch.tensor(math.pi / 4), torch.tensor(3 * math.pi / 4))
    theta[k:] = math.pi * _rand(g, P - k)
    q = _quat_z(theta)
    q[2 * k:] = _random_quat(g, P - 2 * k)
    opac = 0.9 + 0.099 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("needles" + ("_small" if small else ""), w, h, fx, fy, cx, cy, _unproject(u, v, z, fx, fy, cx, cy),
                 col, opac, s_px * z[:, None] / fx, q)


def threshold_opacity(seed=32, small=False):
    """Opacities within a hair of 1/255, where tau = ln(255 op) ~ 0: half with op*255 in [0.995, 1.01], a tenth
    cycling through float32(1/255) and its two neighbours, and three tenths BELOW 1/255 (cull half-extent -1,
    "contributes nowhere") centred inside one warp's 8x4 pixel rectangle, where they are still staged and only the
    alpha test rejects them; plus a tenth of ordinary splats.  Sizes 2-12 px, some anisotropic."""
    g = torch.Generator().manual_seed(seed)
    w, h, P = (48, 32, 160) if small else (128, 96, 4000)
    fx = fy = 100.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u, v = w * _rand(g, P), h * _rand(g, P)
    n_band, n_exact, n_below = P // 2, P // 10, 3 * P // 10
    opac = 0.2 + 0.6 * _rand(g, P)
    opac[:n_band] = ((0.995 + 0.015 * _rand(g, n_band).double()) / 255.0).float()
    f = np.float32(1.0 / 255.0)
    near = torch.tensor([np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))], dtype=torch.float32)
    opac[n_band:n_band + n_exact] = near[torch.arange(n_exact) % 3]
    b0, b1 = n_band + n_exact, n_band + n_exact + n_below
    opac[b0:b1] = ((0.99 + 0.009 * _rand(g, n_below).double()) / 255.0).float()
    # centres strictly inside a warp's rectangle [x0, x0+7] x [y0, y0+3] (the box test passes with half-extent -1)
    wx = torch.randint(0, w // 8, (n_below,), generator=g) * 8
    wy = torch.randint(0, h // 4, (n_below,), generator=g) * 4
    u[b0:b1] = wx + 1.0 + 5.0 * _rand(g, n_below)
    v[b0:b1] = wy + 1.0 + 1.0 * _rand(g, n_below)
    sig = 2.0 + 10.0 * _rand(g, P)
    s_px = sig[:, None] * (1.0 + 3.0 * (_rand(g, P, 3) * (torch.arange(P) % 2 == 0)[:, None]))
    q = _random_quat(g, P)
    col = _rand(g, P, 3)
    return Scene("threshold_opacity" + ("_small" if small else ""), w, h, fx, fy, cx, cy,
                 _unproject(u, v, z, fx, fy, cx, cy), col, opac, s_px * z[:, None] / fx, q)


def near_giants(seed=33, small=False):
    """Splats just inside the near plane (z in (0.2, 0.3]) with radii of hundreds to thousands of pixels, and giants
    far outside the frustum (|x/z| or |y/z| beyond 1.3 tanfov, so the Jacobian is clamped) whose tile rectangles
    still reach the image; low opacities so the layers behind them still show, over a bed of ordinary splats."""
    g = torch.Generator().manual_seed(seed)
    w, h = (48, 32) if small else (128, 96)
    n_near, n_out, n_bed = (12, 12, 36) if small else (120, 120, 360)
    P = n_near + n_out + n_bed
    fx = fy = 100.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u, v = w * _rand(g, P), h * _rand(g, P)
    z[:n_near] = 0.3 - 0.0999 * _rand(g, n_near)
    z[0] = 0.2000001                                           # the float just above the near plane's 0.2f
    # outside: 0.4 .. 20 image widths off one side of the frustum
    o = slice(n_near, n_near + n_out)
    side = torch.randint(0, 4, (n_out,), generator=g)
    off = (0.4 + 19.6 * _rand(g, n_out) ** 2) * w
    along_u, along_v = w * _rand(g, n_out), h * _rand(g, n_out)
    u[o] = torch.where(side == 0, -off, torch.where(side == 1, w + off, along_u))
    v[o] = torch.where(side == 2, -off, torch.where(side == 3, h + off, along_v))
    z[o] = 0.25 + 2.0 * _rand(g, n_out)
    sig = 1.0 + 3.0 * _rand(g, P)
    sig[:n_near] = 50.0 + 600.0 * _rand(g, n_near)
    sig[o] = off * (0.4 + 0.8 * _rand(g, n_out))
    s_px = sig[:, None] * (0.5 + _rand(g, P, 3))
    q = _random_quat(g, P)
    opac = 0.3 + 0.6 * _rand(g, P)
    opac[:n_near + n_out] = 0.01 + 0.2 * _rand(g, n_near + n_out)
    col = _rand(g, P, 3)
    return Scene("near_giants" + ("_small" if small else ""), w, h, fx, fy, cx, cy,
                 _unproject(u, v, z, fx, fy, cx, cy), col, opac, s_px * z[:, None] / fx, q)


def translucent_stack(seed=34, small=False, crossing=False):
    """Thousands of translucent splats (opacity 0.01-0.05) over a few tiles: tile lists of thousands of entries and
    per-pixel contributor chains past 1000 list positions, many ring stages long.  `crossing=True` ramps the opacity
    across the image (0.01 at the left edge, 0.5 at the right) so that T crosses 0.5 (median depth) and 1e-4 (early
    termination) at widely varied list positions."""
    g = torch.Generator().manual_seed(seed)
    w, h, P = (32, 16, 900) if small else (64, 32, 5000)
    fx = fy = 64.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u, v = -4 + (w + 8) * _rand(g, P), -4 + (h + 8) * _rand(g, P)
    sig = 1.5 + 2.5 * _rand(g, P)
    s_px = sig[:, None] * (0.6 + 0.8 * _rand(g, P, 3))
    q = _random_quat(g, P)
    opac = 0.01 + 0.04 * _rand(g, P)
    if crossing:
        opac = 0.01 + 0.49 * (u.clamp(0, w) / w) ** 2 * (0.5 + _rand(g, P))
    col = _rand(g, P, 3)
    return Scene("translucent_" + ("crossing" if crossing else "stack") + ("_small" if small else ""), w, h, fx, fy,
                 cx, cy, _unproject(u, v, z, fx, fy, cx, cy), col, opac, s_px * z[:, None] / fx, q)


def depth_ties(seed=35, small=False, P=70_000):
    """Depth-sort ties: P > 64K (the depth sort's 4096-key tiles) or below it (2048-key tiles).  A third of the
    Gaussians share one of three depths, spread over the whole index range so every tie group spans many sort
    tiles; a third come in pairs of depths one ulp apart, the nearer one at the higher index; the rest are random.
    Identity view, so a mean's z IS its float32 depth key."""
    g = torch.Generator().manual_seed(seed)
    if small:
        P //= 200
    w, h = (32, 32) if small else (256, 128)
    fx = fy = float(w)
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    kind = torch.randint(0, 3, (P,), generator=g)
    z = 1.0 + 3.0 * _rand(g, P)
    tied = torch.tensor([1.5, 2.0, 3.25])[torch.randint(0, 3, (P,), generator=g)]
    z = torch.where(kind == 0, tied, z)
    pair = (kind == 1).nonzero().reshape(-1)
    pair = pair[:pair.numel() // 2 * 2].reshape(-1, 2)
    zn = z.numpy()
    zn[pair[:, 0].numpy()] = np.nextafter(zn[pair[:, 1].numpy()], np.float32(np.inf))
    z = torch.from_numpy(zn)
    u, v = w * _rand(g, P), h * _rand(g, P)
    sig = 0.7 + 1.3 * _rand(g, P)
    s_px = sig[:, None].repeat(1, 3)
    q = torch.zeros(P, 4)
    q[:, 0] = 1.0
    opac = 0.05 + 0.5 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("depth_ties_%d" % P, w, h, fx, fy, cx, cy, _unproject(u, v, z, fx, fy, cx, cy), col, opac,
                 s_px * z[:, None] / fx, q)


def depth_span(seed=36, small=False, P=70_000):
    """Depths log-uniform from 0.2000001 to 1e5, so all four 8-bit digit passes of the depth sort move keys; every
    tenth depth is repeated one ulp LOWER at the next index, so keys that differ only in their lowest bits occur in
    the opposite order to their indices."""
    g = torch.Generator().manual_seed(seed)
    if small:
        P = 300
    w, h = (32, 32) if small else (256, 128)
    fx = fy = float(w)
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = torch.exp(math.log(0.2000001) + (math.log(1e5) - math.log(0.2000001)) * _rand(g, P).double()).float()
    z[0] = 0.2000001
    zn = z.numpy()
    zn[1::10] = np.nextafter(zn[0::10][:zn[1::10].size], np.float32(0))
    z = torch.from_numpy(zn)
    u, v = w * _rand(g, P), h * _rand(g, P)
    sig = 0.7 + 1.3 * _rand(g, P)
    s_px = sig[:, None].repeat(1, 3)
    q = torch.zeros(P, 4)
    q[:, 0] = 1.0
    opac = 0.05 + 0.5 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("depth_span_%d" % P, w, h, fx, fy, cx, cy, _unproject(u, v, z, fx, fy, cx, cy), col, opac,
                 s_px * z[:, None] / fx, q)


TINY_SIZES = [(1, 1), (16, 16), (17, 1), (1, 33), (15, 15), (31, 17)]


def tiny(w, h, seed=37, small=False):
    """A W x H image (one tile, 1-pixel-wide or -tall, W or H = 1 or 15 mod 16) with a few dozen Gaussians, a sixth
    of them larger than the image.  Small enough that `small` changes nothing."""
    g = torch.Generator().manual_seed(seed + 100 * w + h)
    P = 36
    fx = fy = 20.0
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    z = 1.0 + 3.0 * _rand(g, P)
    u, v = -3 + (w + 6) * _rand(g, P), -3 + (h + 6) * _rand(g, P)
    sig = 0.3 + 3.0 * _rand(g, P)
    sig[:P // 6] = 2.0 * max(w, h) + 10.0 * _rand(g, P // 6)
    s_px = sig[:, None] * (0.5 + _rand(g, P, 3))
    q = _random_quat(g, P)
    opac = 0.05 + 0.9 * _rand(g, P)
    col = _rand(g, P, 3)
    return Scene("tiny_%dx%d" % (w, h), w, h, fx, fy, cx, cy, _unproject(u, v, z, fx, fy, cx, cy), col, opac,
                 s_px * z[:, None] / fx, q, bg=(0.1, 0.6, 0.3))


def box_edge_needles(seed=38, small=False):
    """Needles whose x-extreme pixel sits just outside the blend kernels' cull box as it would be WITHOUT its float
    error term (project.cu: `eg`), where only rounding in the float32 evaluation of `power` decides whether the
    reference blends it.  Each needle has a 2D condition number of ~1e5-1e6 (long axis 150-400 px, short axes
    1e-6 of it, so the 0.3 px^2 low-pass sets the width), opacity 0.99 and an in-image angle of 30-60 degrees.

    The float32 conic of such a needle is far from its float64 value (det cancels), so the placement uses the
    projected geometry itself: a first projection (C oracle, bit-identical to the reference's) gives each needle's
    conic, which does not depend on where the needle is moved within the image; the centre is then put 0-0.03 px
    left of the point where the box without `eg` ends at a warp rectangle's first column, on the row of the alpha
    ellipse's x-extreme point."""
    g = torch.Generator().manual_seed(seed)
    w = h = 192 if small else 512
    P = 24 if small else 64
    f = w * 0.78
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    op = 0.99
    z = 1.0 + 2.0 * _rand(g, P)
    long_px = (150.0 + 250.0 * _rand(g, P)) * (0.15 if small else 1.0)
    theta = math.pi / 6 + math.pi / 6 * _rand(g, P)
    col = 8.0 * torch.floor((0.55 * w + 0.35 * w * _rand(g, P)) / 8)
    row = torch.floor(0.55 * h + 0.35 * h * _rand(g, P))
    delta = 0.03 * _rand(g, P).double()
    thin = 0.1 if small else 1e-6      # the small variant stays within reach of the float64 brute force
    s3 = torch.stack([long_px, long_px * thin, long_px * thin], 1) * z[:, None] / f
    q = _quat_z(theta)
    rgb = _rand(g, P, 3)
    opac = torch.full((P,), op)
    name = "box_edge_needles" + ("_small" if small else "")
    first = Scene(name, w, h, f, f, cx, cy, _unproject(col - 0.8 * long_px, row, z, f, f, cx, cy), rgb, opac, s3, q)
    co = torch.from_numpy(first.oracle().geometry()["conic_opacity"]).double()
    a, b, c = co[:, 0], co[:, 1], co[:, 2]
    tau = math.log(255.0 * float(np.float32(op)))
    hx = (torch.sqrt(2 * (tau + 1e-3 + 1e-3 * tau) * c / (a * c - b * b)) * 1.0001 + 2e-3).float().double()
    u = col.double() - hx - delta
    v = row.double() + b * (col.double() - u) / c          # x-extreme of q = tau: c dy + b dx = 0, dx = u - col
    # the projection puts world (u, v) at pixel (u - 0.5, v - 0.5) (ndc_to_pix of the reference's camera matrices)
    means = _unproject(u + 0.5, v + 0.5, z.double(), f, f, cx, cy).float()
    return Scene(name, w, h, f, f, cx, cy, means, rgb, opac, s3, q)


def adversarial(small=False):
    """name -> scene factory of every adversarial scene (the full-size ones unless `small`)."""
    d = {"needles": lambda: needles(small=small), "box_edge_needles": lambda: box_edge_needles(small=small),
         "threshold_opacity": lambda: threshold_opacity(small=small),
         "near_giants": lambda: near_giants(small=small), "translucent_stack": lambda: translucent_stack(small=small),
         "translucent_crossing": lambda: translucent_stack(small=small, crossing=True),
         "depth_ties_70k": lambda: depth_ties(small=small), "depth_ties_20k": lambda: depth_ties(small=small, P=20_000),
         "depth_span": lambda: depth_span(small=small)}
    for w, h in TINY_SIZES:
        d["tiny_%dx%d" % (w, h)] = (lambda w=w, h=h: tiny(w, h, small=small))
    return d


def write_replica_sequence(dst, num_frames, device, seed=14, cam=REPLICA, png_depth_scale=6553.5, quality=95):
    """Writes a sequence in Replica's on-disk layout (results/frame<t>.jpg, results/depth<t>.png, traj.txt of c2w
    rows) under `dst`: the frames are rendered on `device` from a view-filling surface (`view_filling`) along
    `slam.look_trajectory`, colour as JPEG and depth as a 16-bit PNG at `png_depth_scale`, depth as a sensor reports it
    (alpha-normalised, 0 where the silhouette is below 0.9).  Returns the ground-truth w2c matrices [T,4,4] (CPU)."""
    import os
    from PIL import Image
    import splatam_b200 as S
    from splatam_b200 import mapping as M, slam
    gen = view_filling(seed=seed, cam=cam, margin=48, opacity=(0.85, 0.95))
    rs = gen.settings(S.GaussianRasterizationSettings, device)
    gt = dict(means3D=gen.means3D, rgb_colors=gen.colors, unnorm_rotations=gen.rotations,
              logit_opacities=torch.logit(gen.opacities.clamp(0.02, 0.98)), log_scales=torch.log(gen.scales[:, :1]))
    gt = {k: v.to(device).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(num_frames, device)
    os.makedirs(os.path.join(dst, "results"), exist_ok=True)
    w2cs, traj = [], []
    for t in range(num_frames):
        f = slam.render_frame(gt, rots, trans, t, rs)
        depth = torch.where(f["sil"] > 0.9, f["depth"] / f["sil"].clamp(min=1e-6), torch.zeros_like(f["depth"]))
        rgb = (f["im"].clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).cpu().numpy()
        raw = (depth[0] * png_depth_scale).round().clamp(0, 65535).cpu().numpy().astype(np.uint16)
        Image.fromarray(rgb).save(os.path.join(dst, "results", "frame%06d.jpg" % t), quality=quality)
        Image.fromarray(raw).save(os.path.join(dst, "results", "depth%06d.png" % t))
        w2c = M.camera_w2c(rots[..., t], trans[..., t])[0].detach().double().cpu()
        w2cs.append(w2c)
        traj.append(" ".join("%.17g" % v for v in torch.linalg.inv(w2c).reshape(-1).tolist()))
    with open(os.path.join(dst, "traj.txt"), "w") as fh:
        fh.write("\n".join(traj) + "\n")
    return torch.stack(w2cs)


def algorithmic_bytes(P, R, w, h):
    """B_algo of SURVEY.md section 8(d) / BASELINE.md section 4, bytes per fwd+bwd render."""
    tiles = ((w + 15) // 16) * ((h + 15) // 16)
    n, msb = tiles, 0
    # getHigherMsb (rasterizer_impl.cu:35-50)
    msb, step = 16, 16
    while step > 1:
        step //= 2
        msb = msb + step if (n >> msb) else msb - step
    if n >> msb:
        msb += 1
    passes = (32 + msb + 7) // 8
    return 180 * P + (72 + 24 * passes) * R + 44 * h * w
