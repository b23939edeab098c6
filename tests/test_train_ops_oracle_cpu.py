"""CPU: the float64 restatements of the training ops (oracle/train_ops_torch.py), which tests/test_train_ops_f64_gpu.py
holds the kernels to, against the reference's own Python (tests/golden/glue/ref_glue.npz: calc_ssim / l1_loss_v1,
the unmodified get_loss with preset renders, transform_to_frame + both rendervars), against autograd's numerical
gradient, and in float32 against mapping.calc_ssim."""
import os

import numpy as np
import pytest
import torch

from oracle import train_ops_torch as O
from util import GOLDEN, l2_rel

FIX = os.path.join(GOLDEN, "glue", "ref_glue.npz")
F64 = torch.float64


@pytest.fixture(scope="module")
def fx():
    return np.load(FIX)


def _t(a):
    return torch.from_numpy(np.asarray(a))


def _rel(a, b):
    return abs(float(torch.as_tensor(a).detach()) - float(b)) / max(abs(float(b)), 1e-30)


@pytest.mark.parametrize("i", [0, 1, 2])
def test_ssim_and_l1_match_reference_python(fx, i):
    """The fixture is float32: its SSIM and L1 lie within ~1e-7 of float64, its gradients within a few 1e-7."""
    tag = "ssim%d_" % i
    im, gt = _t(fx[tag + "im"]), _t(fx[tag + "gt"])
    x = im.to(F64).requires_grad_(True)
    s = O.ssim(x, gt)
    s.backward()
    assert _rel(s, fx[tag + "ssim"]) < 1e-6
    assert l2_rel(x.grad.numpy(), fx[tag + "dssim"]) < 1e-5
    x = im.to(F64).requires_grad_(True)
    l1 = O.image_loss(x, gt, 1.0, 0.0)
    l1.backward()
    assert _rel(l1, fx[tag + "l1"]) < 1e-6
    assert np.array_equal(x.grad.numpy().astype(np.float32), fx[tag + "dl1"])     # sign / n: exact in both


@pytest.mark.parametrize("mode", ["mapping", "tracking"])
def test_losses_match_reference_get_loss(fx, mode):
    """mapping: 0.5 (0.8 L1 + 0.2 (1 - SSIM)) + masked mean depth L1; tracking: 0.5 masked RGB L1 sum + masked depth
    L1 sum over the silhouette-masked pixels -- loss, weighted terms and gradients."""
    im = _t(fx["loss_im"]).to(F64).requires_grad_(True)
    ds32 = _t(fx["loss_depth_sil"])
    ds = ds32.to(F64).requires_grad_(True)
    gt_im, gt_d = _t(fx["loss_gt_im"]), _t(fx["loss_gt_depth"])
    if mode == "mapping":
        w_im = 0.5 * O.image_loss(im, gt_im, 0.8, 0.2)
        w_depth = 1.0 * O.masked_l1(ds, gt_d, depth_mean=True)[0]
    else:
        ld, li = O.masked_l1(ds, gt_d, im, gt_im, sil_thres=0.99, use_sil=True, depth_mean=False)
        w_im, w_depth = 0.5 * li, 1.0 * ld
    loss = w_im + w_depth
    loss.backward()
    tag = "loss_%s_" % mode
    assert _rel(loss, fx[tag + "loss"]) < 1e-6
    assert _rel(w_im, fx[tag + "w_im"]) < 1e-6 and _rel(w_depth, fx[tag + "w_depth"]) < 1e-6
    assert l2_rel(im.grad.numpy(), fx[tag + "d_im"]) < 1e-5
    assert l2_rel(torch.nan_to_num(ds.grad).numpy(), fx[tag + "d_ds"]) < 1e-5
    # the mask is the reference's: exactly the entries with a non-zero depth gradient
    assert np.array_equal(torch.nan_to_num(ds.grad[0]).numpy() != 0, fx[tag + "d_ds"][0] != 0)


@pytest.mark.parametrize("aniso", [False, True])
@pytest.mark.parametrize("camgrad", [False, True])
def test_prepare_matches_reference_python(fx, aniso, camgrad):
    tag = "glue_%s_%s_" % ("aniso" if aniso else "iso", "cam" if camgrad else "nocam")
    keys = ["means3D", "unnorm_rotations", "logit_opacities", "log_scales", "cam_unnorm_rots", "cam_trans"]
    p = {k: _t(fx[tag + "in_" + k]).to(F64).requires_grad_(True) for k in keys}
    t = int(fx[tag + "time_idx"])
    rot, tran = p["cam_unnorm_rots"][..., t], p["cam_trans"][..., t]
    if not camgrad:
        rot, tran = rot.detach(), tran.detach()
    outs = O.prepare_from_camera(p["means3D"], p["unnorm_rotations"], p["logit_opacities"], p["log_scales"], rot, tran,
                                 _t(fx["glue_w2c0"]))
    for name, o in zip(["means3D", "rotations", "opacities", "scales", "depth_colors"], outs):
        ref = fx[tag + "out_" + name]
        assert np.abs(o.detach().numpy() - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max()), name
    w = [_t(fx[tag + "w%d" % i]) for i in range(5)]
    # both raster calls consume means / rotations / opacities / scales: weights 1.0 (RGB) + 0.5 (depth)
    loss = sum(((1.5 if i < 4 else 1.0) * o * wi).sum() for i, (o, wi) in enumerate(zip(outs, w)))
    loss.backward()
    for k in keys[:4] + (keys[4:] if camgrad else []):
        assert l2_rel(p[k].grad.numpy(), fx[tag + "grad_" + k]) < 1e-5, k


def test_prepare_pose_leaves_match_camera_chain():
    """prepare() with rel_w2c / cam_rot as leaves, chained by hand through camera_pose, equals prepare_from_camera."""
    g = torch.Generator().manual_seed(5)
    P = 300
    args = [torch.randn(P, 3, generator=g, dtype=F64) * 2, torch.randn(P, 4, generator=g, dtype=F64),
            torch.randn(P, 1, generator=g, dtype=F64), torch.randn(P, 3, generator=g, dtype=F64) * 0.3 - 3]
    w2c0 = torch.eye(4, dtype=F64)
    rot = torch.tensor([[0.9, -0.1, 0.2, 0.05]], dtype=F64, requires_grad=True)
    tran = torch.tensor([[-0.3, 0.1, 0.2]], dtype=F64, requires_grad=True)
    ws = [torch.randn(P, 3 if i != 1 and i != 2 else (4 if i == 1 else 1), generator=g, dtype=F64) for i in range(5)]
    loss = lambda outs: sum((o * w).sum() for o, w in zip(outs, ws))
    loss(O.prepare_from_camera(*args, rot, tran, w2c0)).backward()
    ga = rot.grad.clone(), tran.grad.clone()
    rel, cr = O.camera_pose(rot.detach(), tran.detach())
    rel.requires_grad_(True); cr.requires_grad_(True)
    loss(O.prepare(*args, rel, cr, w2c0)).backward()
    rot2, tran2 = rot.detach().clone().requires_grad_(True), tran.detach().clone().requires_grad_(True)
    rel2, cr2 = O.camera_pose(rot2, tran2)
    torch.autograd.backward([rel2, cr2], [rel.grad, cr.grad])
    assert torch.allclose(rot2.grad, ga[0], rtol=1e-12, atol=1e-14) and torch.allclose(tran2.grad, ga[1], rtol=1e-12)


@pytest.mark.parametrize("shape", [(1, 5, 7), (2, 12, 13)])
def test_image_loss_gradcheck(shape):
    g = torch.Generator().manual_seed(6)
    x = torch.rand(*shape, generator=g, dtype=F64).requires_grad_(True)
    y = torch.rand(*shape, generator=g, dtype=F64).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b: O.image_loss(a, b, 0.8, 0.2), (x, y))


@pytest.mark.parametrize("shape", [(3, 45, 97), (1, 11, 7), (3, 64, 80), (1, 1, 1)])
def test_float32_oracle_equals_calc_ssim(shape):
    """In float32 the restatement is mapping.calc_ssim op for op: value and gradient are equal."""
    from splatam_b200.mapping import calc_ssim
    g = torch.Generator().manual_seed(7)
    y = torch.rand(*shape, generator=g)
    x0 = (y + 0.2 * torch.randn(*shape, generator=g)).clamp(0, 1)
    a, b = x0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
    sa, sb = O.ssim(a, y, torch.float32), calc_ssim(b, y)
    sa.backward(); sb.backward()
    assert torch.equal(sa, sb) and torch.equal(a.grad, b.grad)


def test_masked_l1_empty_mask():
    """No pixel in the mask: NaN mean, zero sums, exactly zero gradients (torch's empty boolean index)."""
    ds = torch.rand(3, 4, 5, dtype=F64, requires_grad=True)
    im = torch.rand(3, 4, 5, dtype=F64, requires_grad=True)
    gt_d = torch.zeros(1, 4, 5)
    ld, li = O.masked_l1(ds, gt_d, im, torch.rand(3, 4, 5), depth_mean=True)
    assert torch.isnan(ld) and float(li) == 0.0
    (ld + li).backward()
    assert torch.equal(ds.grad, torch.zeros_like(ds)) and torch.equal(im.grad, torch.zeros_like(im))


def test_adam_oracle_is_torch_adam_with_skips_and_resume():
    """Skipped gradients leave no trace; a run resumed from its state equals an uninterrupted one."""
    g = torch.Generator().manual_seed(8)
    sizes, lrs = [5, 0, 7], [1e-2, 1e-3, 3e-3]
    init = torch.randn(12, generator=g, dtype=F64)
    grads = [torch.randn(12, generator=g, dtype=F64) for _ in range(6)]
    skip = [0, 1, 0, 0, 1, 0]
    a = O.adam(init, grads, sizes, lrs, skip=skip, lr_changes={3: (2, 1e-4)})
    b = O.adam(init, [gr for gr, s in zip(grads, skip) if not s], sizes, lrs, lr_changes={2: (2, 1e-4)})
    assert a[3] == b[3] == 4 and all(torch.equal(u, v) for u, v in zip(a[:3], b[:3]))
    h = O.adam(init, grads[:2], sizes, lrs)
    c = O.adam(h[0], grads[2:], sizes, lrs, state=(h[3], h[1], h[2]))
    d = O.adam(init, grads, sizes, lrs)
    assert c[3] == d[3] == 6 and all(torch.equal(u, v) for u, v in zip(c[:3], d[:3]))
