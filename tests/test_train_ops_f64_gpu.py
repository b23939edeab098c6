"""GPU: the training-step kernels (csrc/train_ops.cu, csrc/prepare.cu) against float64 restatements of the same
operations (oracle/train_ops_torch.py, checked against the reference's own Python by test_train_ops_oracle_cpu.py).

Bound rule, per compared quantity: error(kernel, float64) <= max(floor, 2 x error(float32 oracle, float64)), with
floors of 1e-6 relative for scalar losses and 1e-6 L2-relative for fields; element-wise, the fraction of entries off
by more than 1e-4 (relative error floored at 1e-3 of the largest entry) is at most twice the float32 oracle's.  The
float32 oracle always runs on the CPU: on the GPU cuDNN would run its convolutions in TF32.  Every measured pair is
printed as one `f64err` JSON line."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import train_ops_torch as O
from util import l2_rel, rel_err

pytestmark = pytest.mark.gpu

F32, F64 = torch.float32, torch.float64


def _np(t):
    return t.detach().to("cpu", F64).numpy().reshape(-1)


def _report(name, **kv):
    print("f64err " + json.dumps(dict(name=name, **{k: float(v) for k, v in kv.items()})))


def check_scalar(name, k, c, r, floor=1e-6):
    k, c, r = (float(torch.as_tensor(v).detach()) for v in (k, c, r))
    den = max(abs(r), 1e-30)
    ek, ec = abs(k - r) / den, abs(c - r) / den
    _report(name, kernel=ek, f32=ec)
    assert ek <= max(floor, 2 * ec), (name, ek, ec, k, r)


def _frac_off(a, r):
    if not np.any(r):
        return float(np.mean(a != 0))
    return float(np.mean(rel_err(a, r, 1e-3) > 1e-4))


def check_field(name, k, c, r, floor=1e-6):
    k, c, r = _np(k), _np(c), _np(r)
    assert k.shape == r.shape, name
    lk, lc = l2_rel(k, r), l2_rel(c, r)
    fk, fc = _frac_off(k, r), _frac_off(c, r)
    _report(name, kernel=lk, f32=lc, frac_kernel=fk, frac_f32=fc)
    assert lk <= max(floor, 2 * lc), (name, lk, lc)
    assert fk <= 2 * fc, (name, fk, fc)


# ---- image loss -------------------------------------------------------------------------------------------------

EDGE_SHAPES = [(1, 1, 1), (1, 3, 2), (1, 5, 200), (1, 200, 5)]                 # smaller than the 11x11 window
TILE_SHAPES = [(1, 7, 31), (1, 8, 32), (1, 9, 33), (3, 17, 41), (3, 18, 42), (3, 19, 43)]   # 32x8 output tiles
FAMILIES = ["random", "correlated", "constant", "smooth", "saturated", "outside", "equal"]


def images(family, shape, seed=0):
    """(x, y) float32 CPU images of one input family."""
    g = torch.Generator().manual_seed(seed)
    C, H, W = shape
    r = lambda: torch.rand(*shape, generator=g)
    if family == "random":
        return r(), r()
    if family == "correlated":
        y = r()
        return (y + 0.2 * torch.randn(*shape, generator=g)).clamp(0, 1), y
    if family == "constant":        # zero variance inside: C2 dominates, E[x^2] - mu^2 cancels completely
        return torch.full(shape, 0.3), torch.full(shape, 0.7)
    if family == "smooth":          # low-frequency content, as rendered walls are
        v, u = torch.meshgrid(torch.arange(H, dtype=F64) / max(H, 1), torch.arange(W, dtype=F64) / max(W, 1),
                              indexing="ij")
        ph = torch.arange(C, dtype=F64).reshape(C, 1, 1)
        y = 0.5 + 0.3 * torch.sin(2 * math.pi * (0.7 * u + 0.4 * v) + ph)
        x = y + 0.05 * torch.cos(2 * math.pi * (0.3 * u - 0.9 * v) + 2 * ph)
        return x.float(), y.float()
    if family == "saturated":
        return (r() > 0.5).float(), (r() > 0.3).float()
    if family == "outside":         # renders are not clamped
        return 0.5 + 1.5 * torch.randn(*shape, generator=g), 2.0 * r() - 0.5
    if family == "equal":
        y = r()
        return y.clone(), y
    raise ValueError(family)


def _noncontig(t, dev):
    """`t` on `dev` as a non-contiguous view (W-major storage)."""
    return t.transpose(-1, -2).contiguous().to(dev).transpose(-1, -2)


def run_image_loss(x, y, w_l1, w_ssim, go, dev, ref_dev=None):
    """(loss, grad) of the kernel (non-contiguous inputs), the float32 oracle (CPU) and the float64 oracle (on
    `ref_dev`, the GPU by default)."""
    ref_dev = dev if ref_dev is None else ref_dev
    from splatam_b200.train_ops import image_loss
    a = _noncontig(x, dev).requires_grad_(True)
    assert not a.is_contiguous() or min(x.shape[1:]) == 1
    lk = image_loss(a, _noncontig(y, dev), w_l1, w_ssim)
    (lk * go).backward()
    c = x.clone().requires_grad_(True)
    lc = O.image_loss(c, y, w_l1, w_ssim, dtype=F32)
    (lc * go).backward()
    r = x.to(ref_dev, F64).requires_grad_(True)
    lr = O.image_loss(r, y.to(ref_dev), w_l1, w_ssim, dtype=F64)
    (lr * go).backward()
    return (lk, a.grad), (lc, c.grad), (lr, r.grad)


def _check_image_loss(tag, x, y, w, dev, go=1.7):
    (lk, gk), (lc, gc), (lr, gr) = run_image_loss(x, y, w[0], w[1], go, dev)
    assert torch.isfinite(lk) and torch.isfinite(gk).all(), tag
    check_scalar(tag + ":loss", lk, lc, lr)
    check_field(tag + ":grad", gk, gc, gr)


@pytest.mark.parametrize("family", FAMILIES[:-1])
@pytest.mark.parametrize("shape", EDGE_SHAPES + TILE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_image_loss_small_shapes(shape, family, cuda_device):
    x, y = images(family, shape, seed=sum(shape))
    _check_image_loss("image_loss/%s/%s" % ("x".join(map(str, shape)), family), x, y, (0.8, 0.2), cuda_device)


@pytest.mark.parametrize("shape,family", [((3, 680, 1200), "correlated"), ((3, 1200, 680), "correlated"),
                                          ((3, 680, 1200), "smooth"), ((1, 680, 1200), "outside")],
                         ids=["680x1200", "1200x680", "680x1200-smooth", "C1-680x1200-outside"])
def test_image_loss_full_size(shape, family, cuda_device):
    x, y = images(family, shape, seed=3)
    _check_image_loss("image_loss/%s/%s" % ("x".join(map(str, shape)), family), x, y, (0.8, 0.2), cuda_device)


@pytest.mark.parametrize("w", [(0.8, 0.2), (1.0, 0.0), (0.0, 1.0)], ids=str)
@pytest.mark.parametrize("shape", [(3, 45, 97), (1, 9, 33)], ids=lambda s: "x".join(map(str, s)))
def test_image_loss_weights(shape, w, cuda_device):
    x, y = images("correlated", shape, seed=11)
    _check_image_loss("image_loss/%s/w=%s" % ("x".join(map(str, shape)), w), x, y, w, cuda_device, go=-0.35)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 200), (3, 19, 43), (3, 90, 130)], ids=lambda s: "x".join(map(str, s)))
def test_image_loss_equal_images(shape, cuda_device):
    """x == y: the L1 term is exactly zero, the loss is w_ssim (1 - S) with S within bound of 1, and the gradient --
    zero in exact arithmetic -- is no larger than the float32 oracle's rounding noise allows."""
    x, y = images("equal", shape, seed=5)
    w_ssim = 0.2
    (lk, gk), (lc, gc), (lr, gr) = run_image_loss(x, y, 0.8, w_ssim, 1.0, cuda_device)
    assert float(lr) == 0.0
    s_k, s_c = 1.0 - float(lk) / w_ssim, 1.0 - float(lc) / w_ssim
    check_scalar("image_loss/%s/equal:S" % "x".join(map(str, shape)), s_k, s_c, 1.0)
    # the scale a gradient of this loss has: that of a correlated pair of the same shape
    xs, ys = images("correlated", shape, seed=5)
    scale = float(run_image_loss(xs, ys, 0.8, w_ssim, 1.0, cuda_device)[2][1].norm())
    nk, nc = float(gk.norm()), float(gc.norm())
    _report("image_loss/%s/equal:grad_norm" % "x".join(map(str, shape)), kernel=nk / scale, f32=nc / scale)
    assert nk <= max(1e-6 * scale, 2 * nc), (nk, nc, scale)


@pytest.mark.parametrize("where", [(0, 20, 40), (2, 0, 0), (1, 44, 96), (0, 3, 90)], ids=str)
def test_image_loss_nan_pixel(where, cuda_device):
    """One NaN pixel: the loss is NaN, and the gradient is NaN on exactly the oracle's pixels -- the 21x21 box around
    the NaN, clipped to the image, in its channel -- and finite elsewhere."""
    x, y = images("correlated", (3, 45, 97), seed=9)
    c, i, j = where
    x[c, i, j] = float("nan")
    (lk, gk), _, (lr, gr) = run_image_loss(x, y, 0.8, 0.2, 1.0, cuda_device, ref_dev="cpu")
    assert torch.isnan(lk) and torch.isnan(lr)
    box = torch.zeros(3, 45, 97, dtype=torch.bool)
    box[c, max(i - 10, 0):i + 11, max(j - 10, 0):j + 11] = True
    assert torch.equal(torch.isnan(gr), box)
    assert torch.equal(torch.isnan(gk).cpu(), box)
    assert torch.isfinite(gk[~box.to(gk.device)]).all()


# ---- masked L1 --------------------------------------------------------------------------------------------------

MASK_SIZES = [(67, 131), (1, 528 * 256 - 1), (352, 384), (1, 528 * 256 + 1), (680, 1200)]   # 352*384 = 528*256
MASK_KINDS = ["mixed", "all_in", "all_out", "nan_depth_sq", "sil_at_threshold", "gt_zero_negative"]
SIL = 0.99


def depth_case(kind, H, W, seed=0):
    """(depth_sil [3,H,W], gt_depth [1,H,W], im, gt_im), float32 CPU, for one edge of get_loss's mask."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)
    ds = torch.empty(3, H, W)
    ds[0] = 0.5 + 2.0 * r(H, W)
    ds[1] = 0.95 + 0.1 * r(H, W)                      # silhouette around the 0.99 threshold
    ds[2] = ds[0] ** 2 + 0.01 * r(H, W)
    gt = 0.5 + 2.0 * r(1, H, W)
    im, gt_im = r(3, H, W), r(3, H, W)
    pick = lambda p: r(H, W) < p
    if kind == "mixed":
        ds[0][pick(0.01)] = float("nan")
        gt[0][pick(0.05)] = 0.0
    elif kind == "all_in":
        ds[1] = 1.0
    elif kind == "all_out":
        gt.zero_()
    elif kind == "nan_depth_sq":                      # only the uncertainty (depth^2 - depth^2) is NaN
        ds[2][pick(0.2)] = float("nan")
    elif kind == "sil_at_threshold":                  # strict >: exactly at the (float32) threshold is out
        at = pick(0.3)
        ds[1][at] = torch.tensor(SIL, dtype=F32)
        ds[1][pick(0.1) & ~at] = torch.nextafter(torch.tensor(SIL, dtype=F32), torch.tensor(2.0))
    elif kind == "gt_zero_negative":
        gt[0][pick(0.2)] = 0.0
        gt[0][pick(0.2)] = -0.5
        gt[0][pick(0.05)] = -0.0
    return ds, gt, im, gt_im


@pytest.mark.parametrize("site", ["mapping", "tracking"])
@pytest.mark.parametrize("kind", MASK_KINDS)
@pytest.mark.parametrize("size", MASK_SIZES, ids=lambda s: "%dx%d" % s)
def test_masked_l1(size, kind, site, cuda_device):
    """Both call sites: mapping (mean depth L1, no image) and tracking (silhouette mask, sums, with image)."""
    from splatam_b200.train_ops import masked_l1
    dev = cuda_device
    H, W = size
    ds, gt, im, gt_im = depth_case(kind, H, W, seed=H + W)
    tracking = site == "tracking"
    kw = dict(sil_thres=SIL, use_sil=tracking, depth_mean=not tracking)
    gd, gi = 2.0, 0.5

    def run(dev_, dtype, kernel):
        a = ds.to(dev_, dtype, copy=True).requires_grad_(True)
        b = im.to(dev_, dtype, copy=True).requires_grad_(True)
        if kernel:
            ld, li = masked_l1(a, gt.to(dev_), b if tracking else None, gt_im.to(dev_) if tracking else None, **kw)
        else:
            ld, li = O.masked_l1(a, gt.to(dev_), b if tracking else None, gt_im.to(dev_) if tracking else None,
                                 dtype=dtype, **kw)
        (gd * ld + (gi * li if tracking else 0.0)).backward()
        return ld, li, a.grad, (b.grad if tracking else None)

    k, c, r = run(dev, F32, True), run("cpu", F32, False), run("cpu", F64, False)
    tag = "masked_l1/%dx%d/%s/%s" % (H, W, kind, site)
    if kind == "all_out":
        if tracking:
            assert float(k[0]) == 0.0 and float(k[1]) == 0.0
        else:
            assert torch.isnan(k[0]) and torch.isnan(r[0])
        assert float(k[2].abs().max()) == 0.0 and (k[3] is None or float(k[3].abs().max()) == 0.0)
        return
    # the mask: exactly the oracle's pixels carry a depth gradient
    assert torch.equal(k[2][0].cpu() != 0, r[2][0] != 0), tag
    assert float(k[2][1:].abs().max()) == 0.0
    check_scalar(tag + ":depth", k[0], c[0], r[0])
    check_field(tag + ":grad_depth_sil", k[2], c[2], r[2])
    if tracking:
        check_scalar(tag + ":im", k[1], c[1], r[1])
        check_field(tag + ":grad_im", k[3], c[3], r[3])


# ---- Gaussian preparation and the camera-pose gradient ----------------------------------------------------------

OFFSET = torch.tensor([50.0, -20.0, 10.0])      # ScanNet-scale world coordinates
W2C0 = torch.tensor([[0.999, 0.01, -0.02, -0.1], [-0.01, 1.0, 0.0, 0.05], [0.02, -0.01, 0.999, 0.3],
                     [0.0, 0.0, 0.0, 1.0]])
CAMERAS = {"near_identity": ([1.0, 2e-4, -3e-4, 1e-4], [0.01, -0.02, 0.005]),
           "far": ([0.6, -0.5, 0.4, 0.3], [0.8, -1.5, 2.0]),
           "unnormalised": ([1.8, -1.5, 1.2, 0.9], [0.3, 0.2, -0.4])}       # norm 3


def gaussians(P, aniso, offset, seed=0, extreme=False):
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s: torch.randn(*s, generator=g)
    gs = dict(means3D=mk(P, 3) * 2 + (OFFSET if offset else 0.0), unnorm_rotations=mk(P, 4),
              logit_opacities=mk(P, 1), log_scales=mk(P, 3 if aniso else 1) * 0.3 - 3.0)
    if extreme:     # F.normalize's clamp branch and a tiny norm, saturated sigmoid, exp at +-20
        q = gs["unnorm_rotations"]
        q[0::4] *= 1e-13 / q[0::4].norm(dim=1, keepdim=True)
        q[1::4] *= 1e-6 / q[1::4].norm(dim=1, keepdim=True)
        gs["logit_opacities"][0::3] = 30.0
        gs["logit_opacities"][1::3] = -30.0
        gs["log_scales"][0::5] = 20.0
        gs["log_scales"][1::5] = -20.0
    return gs


def camera(name, dtype=F32):
    q, t = CAMERAS[name]
    return torch.tensor([q], dtype=dtype), torch.tensor([t], dtype=dtype)


def upstream(P, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(P, n, generator=g) for n in (3, 4, 1, 3, 3)]


GKEYS = ("means3D", "unnorm_rotations", "logit_opacities", "log_scales")
OUT_NAMES = ("means_cam", "rotations", "opacities", "scales3", "depth_sil_colors")


def compare_prepare(tag, gs, rot, tran, ups, camgrad, dev):
    """prepare_gaussians with rel_w2c / cam_rot as leaves (the pose built from the camera in float64 and rounded once)
    and, with camgrad, mapping.fused_rendervars through camera_w2c: every output and every gradient."""
    from splatam_b200 import mapping as M
    from splatam_b200.prepare import prepare_gaussians
    rel64, cr64 = O.camera_pose(rot, tran)
    rel32, cr32 = rel64.float(), cr64.float()

    def run(dev_, dtype, kernel):
        p = {k: v.to(dev_, dtype, copy=True).requires_grad_(True) for k, v in gs.items()}
        rel = rel32.to(dev_, dtype, copy=True).requires_grad_(camgrad)
        cr = cr32.to(dev_, dtype, copy=True).requires_grad_(camgrad)
        f = prepare_gaussians if kernel else (lambda *a: O.prepare(*a, dtype=dtype))
        outs = f(*[p[k] for k in GKEYS], rel, cr, W2C0.to(dev_))
        sum((o * w.to(dev_, o.dtype)).sum() for o, w in zip(outs, ups)).backward()
        grads = {k: p[k].grad for k in GKEYS}
        if camgrad:
            grads["rel_w2c"] = rel.grad[:3] if rel.grad is not None else torch.zeros(3, 4)
            grads["cam_rot"] = cr.grad if cr.grad is not None else torch.zeros(1, 4)
        return outs, grads

    k, c, r = run(dev, F32, True), run("cpu", F32, False), run(dev, F64, False)
    for name, a, b, d in zip(OUT_NAMES, k[0], c[0], r[0]):
        check_field("%s:%s" % (tag, name), a, b, d)
    for name in k[1]:
        check_field("%s:g_%s" % (tag, name), k[1][name], c[1][name], r[1][name])
    if not camgrad:
        return

    # mapping.fused_rendervars through camera_w2c: the gradients of the camera's own parameters
    def run_cam(dev_, dtype, kernel):
        rots = rot.to(dev_, dtype, copy=True).reshape(1, 4, 1).requires_grad_(True)
        trans = tran.to(dev_, dtype, copy=True).reshape(1, 3, 1).requires_grad_(True)
        g = {k: v.to(dev_) for k, v in gs.items()}
        if kernel:
            params = dict(g, cam_unnorm_rots=rots, cam_trans=trans, rgb_colors=torch.zeros_like(g["means3D"]))
            rgb, dep = M.fused_rendervars(params, 0, W2C0.to(dev_), camera_grad=True)
            outs = (rgb["means3D"], rgb["rotations"], rgb["opacities"], rgb["scales"], dep["colors_precomp"])
        else:
            outs = O.prepare_from_camera(*[g[k] for k in GKEYS], rots[..., 0], trans[..., 0], W2C0.to(dev_), dtype)
        sum((o * w.to(dev_, o.dtype)).sum() for o, w in zip(outs, ups)).backward()
        return rots.grad, trans.grad

    k, c, r = run_cam(dev, F32, True), run_cam("cpu", F32, False), run_cam(dev, F64, False)
    check_field(tag + ":g_cam_unnorm_rots", k[0], c[0], r[0])
    check_field(tag + ":g_cam_trans", k[1], c[1], r[1])


PREP_CASES = [(P, aniso, camgrad, cam, offset) for P in (1, 255, 256, 257, 100_003, 816_000) for aniso in (False, True)
              for camgrad, cam, offset in ((True, "far", True), (False, "near_identity", False))]
PREP_CASES += [(257, True, True, "unnormalised", False), (100_003, False, True, "near_identity", True)]


@pytest.mark.parametrize("P,aniso,camgrad,cam,offset", PREP_CASES,
                         ids=["P%d-%s-%s-%s-%s" % (P, "aniso" if a else "iso", "cam" if c else "nocam", cam,
                                                   "offset" if o else "origin") for P, a, c, cam, o in PREP_CASES])
def test_prepare_random_upstream(P, aniso, camgrad, cam, offset, cuda_device):
    compare_prepare("prepare/P%d/%s/%s/%s/%s" % (P, "aniso" if aniso else "iso", camgrad, cam, offset),
                    gaussians(P, aniso, offset, seed=P), *camera(cam), upstream(P, P + 1), camgrad, cuda_device)


@pytest.mark.parametrize("aniso", [False, True], ids=["iso", "aniso"])
def test_prepare_extreme_values(aniso, cuda_device):
    """Quaternions of norm 1e-13 (F.normalize's clamp) and 1e-6, logits +-30, log-scales +-20."""
    P = 4000
    compare_prepare("prepare/extreme/%s" % aniso, gaussians(P, aniso, True, seed=7, extreme=True), *camera("far"),
                    upstream(P, 8), True, cuda_device)


@pytest.fixture(scope="module")
def tracking_upstream(cuda_device):
    """The real backward of SplaTAM's tracking loss at 816k Gaussians: a fused render of view_filling(seed=12) at a
    pose 0.05 deg / 1 mm from the one that rendered the target -- converged tracking, where the pose sums cancel most.
    Returns (gaussians, the upstream gradients of the five prepared tensors, camera quaternion, translation)."""
    import scenes
    import splatam_b200 as S
    from splatam_b200 import mapping as M
    from splatam_b200.train_ops import masked_l1
    dev = cuda_device
    sc = scenes.view_filling(seed=12)
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gs = dict(means3D=sc.means3D, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.02, 0.98)), log_scales=torch.log(sc.scales[:, :1]))
    w2c0 = torch.eye(4, device=dev)

    def render(q, t):
        p = {k: v.to(dev) for k, v in gs.items()}
        p.update(rgb_colors=sc.colors.to(dev), cam_unnorm_rots=torch.tensor(q, device=dev).reshape(1, 4, 1),
                 cam_trans=torch.tensor(t, device=dev).reshape(1, 3, 1).requires_grad_(True))
        rgb, dep = M.fused_rendervars(p, 0, w2c0, camera_grad=True)
        outs = [rgb["means3D"], rgb["rotations"], rgb["opacities"], rgb["scales"], dep["colors_precomp"]]
        for o in outs if torch.is_grad_enabled() else []:
            o.retain_grad()
        im, ds, _, _ = S.GaussianRasterizer(cam).forward_fused(
            means3D=rgb["means3D"], means2D=rgb["means2D"], opacities=rgb["opacities"],
            colors_precomp=rgb["colors_precomp"], colors_extra=dep["colors_precomp"], scales=rgb["scales"],
            rotations=rgb["rotations"])
        return outs, im, ds

    q0, t0 = [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0]
    q1, t1 = [1.0, 4e-4, -3e-4, 2e-4], [0.001, -0.0005, 0.0007]
    with torch.no_grad():
        _, im, ds = render(q0, t0)
    outs, im1, ds1 = render(q1, t1)
    ld, li = masked_l1(ds1, ds[0:1].detach(), im1, im.detach(), sil_thres=SIL, use_sil=True, depth_mean=False)
    (0.5 * li + ld).backward()
    ups = [o.grad.detach().cpu() for o in outs]
    assert all(torch.isfinite(u).all() for u in ups) and float(ups[0].abs().max()) > 0
    return {k: v.detach().cpu() for k, v in gs.items()}, ups, torch.tensor([q1]), torch.tensor([t1])


@pytest.mark.parametrize("offset", [False, True], ids=["origin", "offset"])
def test_prepare_pose_gradient_of_converged_tracking(tracking_upstream, offset, cuda_device):
    """816k Gaussians with upstream gradients from a real tracking backward; with `offset` the map (and the camera
    translation that keeps it in view) is moved to ScanNet-scale coordinates, which the translation column of the pose
    gradient has to cancel."""
    gs, ups, q, t = tracking_upstream
    gs = dict(gs)
    if offset:      # R (p + o) + (t - R o) = R p + t: the same camera-frame map
        gs["means3D"] = gs["means3D"] + OFFSET
        R = O.camera_pose(q, t)[0][:3, :3]
        t = (t.double() - (R @ OFFSET.double())).float().reshape(1, 3)
    compare_prepare("prepare/tracking816k/%s" % ("offset" if offset else "origin"), gs, q, t, ups, True, cuda_device)


# ---- fused Adam -------------------------------------------------------------------------------------------------

def _ordered(a):
    i = a.detach().cpu().contiguous().view(torch.int32).to(torch.int64)
    return torch.where(i < 0, -(i & 0x7FFFFFFF), i)


def ulps(a, b):
    """Per-element distance in float32 units in the last place; NaN == NaN (and +-inf equal to itself) is 0."""
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    d = (_ordered(a) - _ordered(b)).abs()
    both_nan = torch.isnan(a) & torch.isnan(b)
    d[both_nan] = 0
    d[torch.isnan(a) ^ torch.isnan(b)] = 1 << 40
    return d


def ulps_of_scale(a, b, old):
    """|a - b| in units of the last place of the operands' scale max(|a|, |b|, |old|): an update that cancels most of
    its old value (p - lr m / sqrt(v) near 0) is rounded at the scale of its operands, not of its result.  NaN == NaN
    and inf == inf count as 0."""
    a, b, old = (t.detach().cpu().double() for t in (a, b, old))
    scale = torch.maximum(torch.maximum(a.abs(), b.abs()), old.abs()).nan_to_num(0.0, 0.0, 0.0).float()
    ulp = (torch.nextafter(scale, torch.tensor(float("inf"))) - scale).double().clamp_min(2.0 ** -149)
    d = ((a - b).abs() / ulp).nan_to_num(0.0, 0.0, 0.0)
    same = (torch.isnan(a) & torch.isnan(b)) | (torch.isinf(a) & (a == b))
    d[same] = 0.0
    d[torch.isnan(a) ^ torch.isnan(b)] = float("inf")
    return d


def torch_adam_step(p, g, m, v, t, sizes, lrs, betas=(0.9, 0.999), eps=1e-15):
    """One float32 torch.optim.Adam step (CPU) from the state (p, m, v, t): returns the new (p, m, v)."""
    ps = [x.clone().requires_grad_(True) for x in torch.split(p.cpu(), sizes)]
    opt = torch.optim.Adam([{"params": [x], "lr": lr} for x, lr in zip(ps, lrs)], lr=0.0, betas=betas, eps=eps,
                           foreach=False)
    for x, gx, mx, vx in zip(ps, *(torch.split(a.cpu(), sizes) for a in (g, m, v))):
        x.grad = gx.clone()
        opt.state[x] = dict(step=torch.tensor(float(t)), exp_avg=mx.clone(), exp_avg_sq=vx.clone())
    opt.step()
    return (torch.cat([x.detach() for x in ps]), torch.cat([opt.state[x]["exp_avg"] for x in ps]),
            torch.cat([opt.state[x]["exp_avg_sq"] for x in ps]))


# The moments agree within 1 ulp.  For the parameter, torch's CPU addcdiv rounds lr_t * m, then the quotient, then the
# sum (3 roundings); the kernel, like torch's CUDA addcdiv, rounds m / denom and the fused multiply-add (2).  The two
# differ by at most 1.5 ulps of the update plus 1 ulp of the result, and the update is at most twice the operands'
# scale (it cancels p at most): 4 ulps of that scale.
ULPS = dict(p=4, m=1, v=1)

LAYOUTS = {
    "16segs_some_empty": [0, 5, 250, 0, 256, 1, 0, 257, 3, 0, 1000, 7, 0, 2, 511, 0],
    "ends_255_256_257": [255, 1, 1, 300],
    "ends_256_257": [256, 1, 254],
    "n1": [1],
    "n2": [1, 1],
    "n1023": [1023],
    "n1025": [512, 513],
    "n65537": [65536, 1],
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_adam_segment_layouts_match_torch_steps(layout, cuda_device):
    """Each step, started from the kernel's own state, is within ULPS (of the operands' scale) of float32
    torch.optim.Adam's step (CPU) in the parameters and both moments; every segment gets its own learning rate."""
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    sizes = LAYOUTS[layout]
    lrs = [1e-3 * (k + 1) for k in range(len(sizes))]
    n = sum(sizes)
    g = torch.Generator().manual_seed(len(sizes) * 1000 + n)
    flat, grad = torch.randn(n, generator=g).to(dev), torch.zeros(n, device=dev)
    opt = FusedAdam(flat, grad, sizes, lrs, eps=1e-15)
    worst = 0
    for t in range(1, 7):
        gr = torch.randn(n, generator=g) * 10.0 ** torch.randint(-4, 2, (n,), generator=g).float()
        p0, m0, v0 = flat.cpu(), opt.m.cpu(), opt.v.cpu()
        grad.copy_(gr.to(dev))
        opt.step()
        rp, rm, rv = torch_adam_step(p0, gr, m0, v0, t - 1, sizes, lrs)
        for name, a, b, old in (("p", flat, rp, p0), ("m", opt.m, rm, m0), ("v", opt.v, rv, v0)):
            d = float(ulps_of_scale(a, b, old).max()) if n else 0.0
            worst = max(worst, d)
            assert d <= ULPS[name], (layout, t, name, d)
    _report("adam/layout/%s" % layout, max_ulps=worst)


def test_adam_rejects_17_segments(cuda_device):
    """17 segments: FusedAdam refuses them, and so does the C ABI, before anything is launched."""
    import ctypes
    from splatam_b200 import _lib
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    flat, grad = torch.ones(17, device=dev), torch.ones(17, device=dev)
    with pytest.raises(ValueError):
        FusedAdam(flat, grad, [1] * 17, [1e-3] * 17)
    m, v = torch.zeros(17, device=dev), torch.zeros(17, device=dev)
    ends = (ctypes.c_uint32 * 17)(*range(1, 18))
    lrs = (ctypes.c_double * 17)(*([1e-3] * 17))
    with pytest.raises(_lib.SplatamB200Error, match="SB_ERR_BAD_ARG"):
        _lib.call("sb_adam_step", flat, grad, m, v, 17, ends, lrs, 17, 1, 0.9, 0.999, 1e-15, device=dev)
    clock = torch.zeros(64, dtype=torch.int32, device=dev)
    with pytest.raises(_lib.SplatamB200Error, match="SB_ERR_BAD_ARG"):
        _lib.call("sb_adam_step_guarded", flat, grad, m, v, 17, ends, lrs, 17, clock, None, 0.9, 0.999, 1e-15,
                  device=dev)
    torch.cuda.synchronize(dev)
    assert float(flat.min()) == 1.0 and float(flat.max()) == 1.0 and float(m.abs().max()) == 0.0
    assert int(clock.abs().max()) == 0


def _adam_problem(sizes=(3000, 0, 7001, 999, 9000), steps=30, seed=4):
    g = torch.Generator().manual_seed(seed)
    sizes, n = list(sizes), sum(sizes)
    lrs = [1e-4, 1e-3, 2.5e-3, 5e-2, 1e-3]
    init = torch.randn(n, generator=g)
    mag = 10.0 ** (-6.0 + 8.0 * torch.rand(n, generator=g))          # gradients spanning 1e-6 .. 1e2
    grads = [torch.randn(n, generator=g) * mag for _ in range(steps)]
    return sizes, lrs, init, grads


def test_adam_30_steps_against_float64(cuda_device):
    """30 steps, gradients from 1e-6 to 1e2, eps = 1e-15, a learning-rate change halfway: parameters and moments
    against torch.optim.Adam in float64, with float32 torch.optim.Adam (CPU) as the comparator."""
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    sizes, lrs, init, grads = _adam_problem()
    flat, grad = init.to(dev), torch.zeros_like(init, device=dev)
    opt = FusedAdam(flat, grad, sizes, lrs, eps=1e-15)
    change = {15: (2, 4e-4)}
    for i, gr in enumerate(grads):
        if i in change:
            opt.set_lr(*change[i])
        grad.copy_(gr.to(dev))
        opt.step()
    c = O.adam(init, grads, sizes, lrs, lr_changes=change, dtype=F32)
    r = O.adam(init, grads, sizes, lrs, lr_changes=change, dtype=F64)
    for name, a, b, d in zip(("params", "exp_avg", "exp_avg_sq"), (flat, opt.m, opt.v), c[:3], r[:3]):
        check_field("adam/30steps:" + name, a, b, d)
    # the parameter update itself, where lr * m / sqrt(v) is small against the parameter
    check_field("adam/30steps:update", flat.cpu().double() - init.double(), c[0].double() - init.double(), r[0] - init.double())


SKIP = [0, 1, 0, 0, 1, 1, 0, 0, 0, 1, 0, 1, 1, 1, 0, 0]


@pytest.mark.parametrize("flag", [1.0, -2.5, float("inf")], ids=["one", "negative", "inf"])
def test_adam_guarded_equals_unguarded_over_applied_steps(flag, cuda_device):
    """Guarded steps with the skip pattern: the moments are bit-equal to unguarded steps over only the applied
    gradients, the parameters within 1 ulp per applied step (the device pow of the bias corrections against the host's),
    applied_steps() counts both, and step() after step_guarded() goes on from the device clock."""
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    sizes, lrs, init, grads = _adam_problem((1000, 0, 2001, 999, 1000), steps=len(SKIP) + 1, seed=6)
    fa, ga = init.to(dev), torch.zeros(5000, device=dev)
    fb, gb = init.to(dev), torch.zeros(5000, device=dev)
    a, b = FusedAdam(fa, ga, sizes, lrs), FusedAdam(fb, gb, sizes, lrs)
    flagt = torch.zeros(1, device=dev)
    worst, applied = 0, 0
    for gr, s in zip(grads, SKIP):
        ga.copy_(gr.to(dev))
        flagt.fill_(flag if s else 0.0)
        a.step_guarded(flagt)
        if not s:
            gb.copy_(gr.to(dev))
            b.step()
            applied += 1
        assert torch.equal(a.m, b.m) and torch.equal(a.v, b.v)
        d = int(ulps(fa, fb).max())
        worst = max(worst, d)
        assert d <= applied, (applied, d)
    assert a.applied_steps() == (SKIP.count(0), SKIP.count(1))
    ga.copy_(grads[-1].to(dev)); gb.copy_(grads[-1].to(dev))
    a.step(); b.step()
    assert a.applied_steps() == (SKIP.count(0) + 1, SKIP.count(1))
    assert torch.equal(a.m, b.m) and torch.equal(a.v, b.v) and int(ulps(fa, fb).max()) <= applied + 1
    _report("adam/guarded/%s" % flag, max_ulps=worst)


@pytest.mark.parametrize("mode", ["plain", "guarded"])
def test_adam_resume_is_bit_equal(mode, cuda_device):
    """FusedAdam(step=t, exp_avg=m, exp_avg_sq=v) continued from a saved state is bit-equal to an uninterrupted run."""
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    sizes, lrs, init, grads = _adam_problem((1000, 0, 1000, 500, 500), steps=10, seed=7)
    zero = torch.zeros(1, device=dev)

    def steps(opt, g, gs):
        for gr in gs:
            g.copy_(gr.to(dev))
            opt.step_guarded(zero) if mode == "guarded" else opt.step()

    fa, ga = init.to(dev), torch.zeros(3000, device=dev)
    a = FusedAdam(fa, ga, sizes, lrs)
    steps(a, ga, grads)
    fb, gb = init.to(dev), torch.zeros(3000, device=dev)
    b = FusedAdam(fb, gb, sizes, lrs)
    steps(b, gb, grads[:4])
    t = b.applied_steps()[0]
    fc, gc = fb.clone(), torch.zeros(3000, device=dev)
    c = FusedAdam(fc, gc, sizes, lrs, exp_avg=b.m.clone(), exp_avg_sq=b.v.clone(), step=t)
    steps(c, gc, grads[4:])
    assert torch.equal(fa, fc) and torch.equal(a.m, c.m) and torch.equal(a.v, c.v)
    assert c.applied_steps()[0] == a.applied_steps()[0] == 10


@pytest.mark.parametrize("edge", ["zero", "denormal", "huge", "nan"])
def test_adam_element_edges(edge, cuda_device):
    """Zero gradient: the element is unchanged.  Denormal gradients; 1e21 gradients, where (1 - b2) g g overflows and
    v becomes inf; a NaN gradient changes only its own element.  Each step within ULPS (of the operands' scale) of
    torch, NaN == NaN."""
    from splatam_b200.train_ops import FusedAdam
    dev = cuda_device
    n, sizes, lrs = 1000, [600, 400], [1e-3, 5e-3]
    g = torch.Generator().manual_seed(12)
    flat, grad = torch.randn(n, generator=g).to(dev), torch.zeros(n, device=dev)
    opt = FusedAdam(flat, grad, sizes, lrs)
    idx = torch.tensor([0, 1, 599, 600, 601, 999, 333])
    for t in range(1, 5):
        gr = torch.randn(n, generator=g)
        if edge == "zero":
            gr[idx] = 0.0
        elif edge == "denormal":
            gr[idx] = torch.tensor([1e-40, -1e-41, 1e-45, -1e-45, 3e-39, 1e-44, -2e-40])
        elif edge == "huge":
            gr[idx] = torch.tensor([1e21, -1e21, 3e20, -1e22, 1e21, 1e21, -1e21])
        else:
            gr[idx[:3]] = float("nan")
        p0, m0, v0 = flat.cpu(), opt.m.cpu(), opt.v.cpu()
        grad.copy_(gr.to(dev))
        opt.step()
        rp, rm, rv = torch_adam_step(p0, gr, m0, v0, t - 1, sizes, lrs)
        for name, a, b, old in (("p", flat, rp, p0), ("m", opt.m, rm, m0), ("v", opt.v, rv, v0)):
            d = float(ulps_of_scale(a, b, old).max())
            assert d <= ULPS[name], (edge, t, name, d)
        if edge == "zero":
            assert torch.equal(flat.cpu()[idx], p0[idx])
        if edge == "huge":
            assert torch.isinf(opt.v.cpu()[idx[[0, 1, 3, 4, 5, 6]]]).all()
        if edge == "nan":
            bad = torch.zeros(n, dtype=torch.bool)
            bad[idx[:3]] = True
            assert torch.isnan(flat.cpu()[bad]).all() and torch.isfinite(flat.cpu()[~bad]).all()
