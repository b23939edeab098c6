"""GPU: the fused glue / loss kernels (csrc/prepare.cu, csrc/train_ops.cu) against outputs of the reference's OWN
Python (tests/golden/glue/ref_glue.npz, generated from R/utils/slam_helpers.py, R/utils/slam_external.py and the
unmodified get_loss of R/scripts/splatam.py), and loop-level tests against what the UNMODIFIED get_loss /
initialize_optimizer computed over the reference extension (tests/golden/reference/loops.npz).  Where the reference's
Python is installed (oracle/_ref/SplaTAM, oracle/reference.py), the same get_loss also runs through this repo's drop-in
alias."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, digest

pytestmark = pytest.mark.gpu
FIX = os.path.join(GOLDEN, "glue", "ref_glue.npz")
LOOPS = os.path.join(GOLDEN, "reference", "loops.npz")     # tests/golden/make_golden_reference.py
UPDATE_KEYS = ("means3D", "rgb_colors", "logit_opacities", "log_scales")


@pytest.fixture(scope="module")
def fx():
    return np.load(FIX)


def _t(a, dev):
    return torch.from_numpy(np.asarray(a)).to(dev)


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("aniso", [False, True])
@pytest.mark.parametrize("camgrad", [False, True])
def test_fused_glue_matches_reference_python(fx, aniso, camgrad, cuda_device):
    """prepare_gaussians == transform_to_frame + transformed_params2rendervar + transformed_params2depthplussilhouette
    (R/utils/slam_helpers.py:124-139,196-304): values and every gradient incl. the camera pose."""
    from splatam_b200 import mapping as M
    dev = cuda_device
    tag = "glue_%s_%s_" % ("aniso" if aniso else "iso", "cam" if camgrad else "nocam")
    keys = ["means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales", "cam_unnorm_rots", "cam_trans"]
    p = {k: _t(fx[tag + "in_" + k], dev).clone().requires_grad_(True) for k in keys}
    t = int(fx[tag + "time_idx"])
    rgb, dep = M.fused_rendervars(p, t, _t(fx["glue_w2c0"], dev), camera_grad=camgrad)
    outs = [rgb["means3D"], rgb["rotations"], rgb["opacities"], rgb["scales"], dep["colors_precomp"]]
    for name, o in zip(["means3D", "rotations", "opacities", "scales", "depth_colors"], outs):
        assert torch.allclose(o, _t(fx[tag + "out_" + name], dev), rtol=1e-5, atol=1e-6), name
    assert rgb["colors_precomp"] is p["rgb_colors"]
    w = [_t(fx[tag + "w%d" % i], dev) for i in range(5)]
    loss = sum((o * wi).sum() for o, wi in zip(outs, w)) + 0.5 * sum(
        (o * wi).sum() for o, wi in zip([dep["means3D"], dep["rotations"], dep["opacities"], dep["scales"]], w))
    loss.backward()
    for k in ["means3D", "unnorm_rotations", "logit_opacities", "log_scales"] + (["cam_unnorm_rots", "cam_trans"] if camgrad else []):
        assert _rel(p[k].grad, _t(fx[tag + "grad_" + k], dev)) < 1e-4, k


@pytest.mark.parametrize("i", [0, 1, 2])
def test_fused_image_loss_matches_reference_python(fx, i, cuda_device):
    """image_loss == 0.8 l1_loss_v1 + 0.2 (1 - calc_ssim) of the reference (slam_external.py:66-97)."""
    from splatam_b200.train_ops import image_loss
    dev = cuda_device
    tag = "ssim%d_" % i
    gt = _t(fx[tag + "gt"], dev)
    a = _t(fx[tag + "im"], dev).clone().requires_grad_(True)
    ls = image_loss(a, gt, 0.0, 1.0)
    ls.backward()
    assert abs(float(ls.detach()) - (1.0 - float(fx[tag + "ssim"]))) < 2e-6
    assert _rel(a.grad, -_t(fx[tag + "dssim"], dev)) < 5e-4
    b = _t(fx[tag + "im"], dev).clone().requires_grad_(True)
    l1 = image_loss(b, gt, 1.0, 0.0)
    l1.backward()
    assert abs(float(l1.detach()) - float(fx[tag + "l1"])) < 2e-6
    assert torch.allclose(b.grad, _t(fx[tag + "dl1"], dev), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("mode", ["mapping", "tracking"])
def test_fused_losses_match_reference_get_loss(fx, mode, cuda_device):
    """The fused loss kernels on the renders the fixture holds == loss and dLoss/d(renders) of the UNMODIFIED
    get_loss (R/scripts/splatam.py:214-347): masks (valid depth, NaN, silhouette > 0.99), L1 sums / means, SSIM,
    weights im 0.5 / depth 1.0."""
    from splatam_b200.train_ops import image_loss, masked_l1
    dev = cuda_device
    im = _t(fx["loss_im"], dev).clone().requires_grad_(True)
    ds = _t(fx["loss_depth_sil"], dev).clone().requires_grad_(True)
    gt_im, gt_d = _t(fx["loss_gt_im"], dev), _t(fx["loss_gt_depth"], dev)
    if mode == "mapping":
        l_depth, _ = masked_l1(ds, gt_d, depth_mean=True)
        loss = 0.5 * image_loss(im, gt_im, 0.8, 0.2) + 1.0 * l_depth
    else:
        l_depth, l_im = masked_l1(ds, gt_d, im, gt_im, sil_thres=0.99, use_sil=True, depth_mean=False)
        loss = 0.5 * l_im + 1.0 * l_depth
    loss.backward()
    tag = "loss_%s_" % mode
    ref = float(fx[tag + "loss"])
    assert abs(float(loss.detach()) - ref) < 3e-6 * max(1.0, abs(ref)), (float(loss.detach()), ref)
    assert _rel(im.grad, _t(fx[tag + "d_im"], dev)) < 2e-4
    assert _rel(torch.nan_to_num(ds.grad), _t(fx[tag + "d_ds"], dev)) < 1e-5


# ---- loop level: the reference's own Python, unmodified, over both operators ------------------------------------

def _loop_problem(dev, P=40_000):
    sc = scenes.view_filling(seed=31, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5), stride=1)
    g = torch.Generator().manual_seed(5)
    gauss = sc.splatam_params()
    rots = torch.zeros(1, 4, 2); rots[:, 0] = 1.0
    rots[0, 1:, 1] = torch.tensor([0.004, -0.003, 0.002])
    trans = torch.zeros(1, 3, 2); trans[0, :, 1] = torch.tensor([0.010, -0.006, 0.008])
    params = {k: v.to(dev) for k, v in dict(gauss, cam_unnorm_rots=rots, cam_trans=trans).items()}
    gt_im = torch.rand(3, sc.h, sc.w, generator=g).to(dev)
    gt_d = (1.0 + 2.0 * torch.rand(1, sc.h, sc.w, generator=g)).to(dev)
    gt_d[0, :4] = 0.0
    return sc, params, gt_im, gt_d


def _run_get_loss(R, sc, params, gt_im, gt_d, mode, dev):
    cam = R.recon_helpers.setup_camera(sc.w, sc.h, np.array([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1.0]]),
                                       np.eye(4))
    p = {k: torch.nn.Parameter(v.clone().contiguous()) for k, v in params.items()}
    P = p["means3D"].shape[0]
    variables = dict(max_2D_radius=torch.zeros(P, device=dev), means2D_gradient_accum=torch.zeros(P, device=dev),
                     denom=torch.zeros(P, device=dev))
    curr = dict(cam=cam, im=gt_im, depth=gt_d, id=1, intrinsics=None, w2c=torch.eye(4, device=dev), iter_gt_w2c_list=None)
    tracking = mode == "tracking"
    loss, variables, wl = R.splatam.get_loss(p, curr, variables, 1, dict(im=0.5, depth=1.0), use_sil_for_loss=tracking,
                                             sil_thres=0.99, use_l1=True, ignore_outlier_depth_loss=False,
                                             tracking=tracking, mapping=not tracking)
    loss.backward()
    return float(loss.detach()), {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in p.items()}, variables, p


def loss_keys(mode):
    return ["cam_unnorm_rots", "cam_trans"] if mode == "tracking" else ["means3D", "rgb_colors", "logit_opacities", "log_scales"]


def stock_mapping_iterations(R, sc, params, gt_im, gt_d, dev):
    """Five iterations of the reference's mapping inner loop with its stock optimizer; returns (losses, params)."""
    from splatam_b200 import mapping as M
    lrs = dict(M.ShardedMapper.DEFAULT_LRS, cam_unnorm_rots=0.0, cam_trans=0.0)
    p = {k: torch.nn.Parameter(v.clone().contiguous()) for k, v in params.items()}
    opt = R.splatam.initialize_optimizer(p, lrs, tracking=False)
    cam = R.recon_helpers.setup_camera(sc.w, sc.h, np.array([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1.0]]), np.eye(4))
    P = p["means3D"].shape[0]
    variables = dict(max_2D_radius=torch.zeros(P, device=dev), means2D_gradient_accum=torch.zeros(P, device=dev),
                     denom=torch.zeros(P, device=dev))
    curr = dict(cam=cam, im=gt_im, depth=gt_d, id=1, intrinsics=None, w2c=torch.eye(4, device=dev), iter_gt_w2c_list=None)
    losses = []
    for _ in range(5):
        loss, variables, _ = R.splatam.get_loss(p, curr, variables, 1, dict(im=0.5, depth=1.0), False, 0.99, True, False,
                                                mapping=True)
        loss.backward()
        with torch.no_grad():
            opt.step()
            opt.zero_grad(set_to_none=True)
        losses.append(float(loss.detach()))
    return losses, p


@pytest.mark.parametrize("mode", ["mapping", "tracking"])
def test_unmodified_get_loss_through_the_drop_in_alias(mode, cuda_device):
    """SURVEY.md section 4 item 4: get_loss (R/scripts/splatam.py:214-347) + transform_to_frame / rendervars
    (R/utils/slam_helpers.py) + setup_camera (R/utils/recon_helpers.py:4-27), none of them modified, as they ran over
    the reference extension (loss, `seen` / max_2D_radius bit for bit, gradients on a seeded sample of the seen
    Gaussians); where the reference's Python is installed, the same unmodified code once more with
    `diff_gaussian_rasterization` = this repo's alias package; then this repo's fused mapping / tracking loss (fused
    glue + two-set render + fused loss kernels) against the reference."""
    import refsrc
    import splatam_b200 as S
    import splatam_b200.compat.diff_gaussian_rasterization as alias
    from splatam_b200 import mapping as M
    dev = cuda_device
    sc, params, gt_im, gt_d = _loop_problem(dev)
    z = np.load(LOOPS)
    lr, idx, keys = float(z[mode + "_loss"]), torch.from_numpy(z[mode + "_index"]), loss_keys(mode)
    gr = {k: torch.from_numpy(z["%s_grad_%s" % (mode, k)]) for k in keys}

    def pick(g, k):
        g = g.detach().cpu()
        return g if k.startswith("cam_") else g[idx]
    if refsrc.available():
        R_ours = refsrc.load(alias)
        assert R_ours.splatam.Renderer is S.GaussianRasterizer
        lo, go, vo, _ = _run_get_loss(R_ours, sc, params, gt_im, gt_d, mode, dev)
        assert abs(lo - lr) < 1e-5 * abs(lr), (lo, lr)
        assert digest(vo["seen"].cpu().numpy()) == str(z[mode + "_digest_seen"])
        assert digest(vo["max_2D_radius"].cpu().numpy()) == str(z[mode + "_digest_max_2D_radius"])
        for k in keys:
            assert _rel(pick(go[k], k), gr[k]) < 1e-4, (k, _rel(pick(go[k], k), gr[k]))
    # this repo's fused formulation of the same loss
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    frame = dict(id=1, cam=sc.settings(S.GaussianRasterizationSettings, dev), w2c=torch.eye(4, device=dev), im=gt_im, depth=gt_d)
    if mode == "mapping":
        lf, _ = M.mapping_loss(p, frame, M.default_render, fused_loss=True)
    else:
        lf, _ = M.tracking_loss(p, frame, M.default_render, fused=True)
    lf.backward()
    assert abs(float(lf.detach()) - lr) < 2e-5 * abs(lr), (float(lf.detach()), lr)
    for k in keys:
        assert _rel(pick(p[k].grad, k), gr[k]) < 2e-4, (k, _rel(pick(p[k].grad, k), gr[k]))


def test_unmodified_mapping_iterations_with_stock_optimizer(cuda_device):
    """Five iterations of the reference's mapping inner loop -- get_loss(mapping=True), backward, the stock
    initialize_optimizer (R/scripts/splatam.py:160-166) -- with the reference extension (its losses and, on a seeded
    sample of 512 Gaussians, its parameter updates are stored in tests/golden/reference/loops.npz) and with this repo's
    ShardedMapper (fused path): losses follow each other and the parameters end up the same."""
    import splatam_b200 as S
    from splatam_b200 import mapping as M
    dev = cuda_device
    sc, params, gt_im, gt_d = _loop_problem(dev)
    z = np.load(LOOPS)
    ref_losses, idx = z["stock_losses"].tolist(), torch.from_numpy(z["stock_index"]).to(dev)
    gauss = {k: params[k] for k in M.GAUSSIAN_KEYS}
    m = M.ShardedMapper(gauss, params["cam_unnorm_rots"], params["cam_trans"], seed=3, fused=True)
    frame = dict(id=1, cam=sc.settings(S.GaussianRasterizationSettings, dev), w2c=torch.eye(4, device=dev), im=gt_im, depth=gt_d)
    our_losses = [m.step([frame])[0] for _ in range(5)]
    assert np.allclose(our_losses, ref_losses, rtol=1e-3), (our_losses, ref_losses)
    # Adam with eps = 1e-15 turns every gradient element into a step of ~lr whatever its size, so elements whose
    # gradient is float noise (all of unnorm_rotations for isotropic Gaussians; a few elsewhere) move by +-lr in
    # BOTH implementations with uncorrelated signs.  Compare the UPDATES of the parameters that carry signal.
    for k in UPDATE_KEYS:
        du, dr = (m.g.params[k].detach() - params[k])[idx], torch.from_numpy(z["stock_update_" + k]).to(dev)
        assert float((du - dr).norm() / dr.norm()) < 0.05, (k, float((du - dr).norm() / dr.norm()))
