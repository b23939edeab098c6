"""BASELINE config[1]-style tracking loop on the GPU: SplaTAM's tracking inner loop (camera-only Adam, silhouette-
masked L1 sums) run with (a) the fused path, (b) the plain two-call path through this repo's operator and
(c) the unmodified reference extension (its run is stored in tests/golden/reference/loops.npz) -- the three must
recover the same pose."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN

pytestmark = pytest.mark.gpu


def _setup(dev, Settings, P=50_000):
    sc = scenes.room(seed=1, P=P, cam=dict(w=400, h=224, fx=200.0, fy=200.0, cx=199.5, cy=111.5))
    cam = sc.settings(Settings, dev)
    gauss = sc.splatam_params()
    gauss = {k: v.to(dev) for k, v in gauss.items()}
    return sc, cam, gauss


def _pose_params(dev, rot1, tran1):
    rots = torch.zeros(1, 4, 2); rots[:, 0] = 1.0
    trans = torch.zeros(1, 3, 2)
    rots[0, :, 1] = torch.tensor(rot1); trans[0, :, 1] = torch.tensor(tran1)
    return rots.to(dev), trans.to(dev)


TRUE_ROT, TRUE_TRAN = [1.0, 0.004, -0.003, 0.002], [0.010, -0.006, 0.008]     # ~0.5 deg, ~1 cm


def _problem(dev):
    """The map and the target RGB-D frame, rendered at the true pose with this repo's operator."""
    import splatam_b200 as S
    from splatam_b200 import mapping as M
    sc, cam, gauss = _setup(dev, S.GaussianRasterizationSettings)
    with torch.no_grad():
        r, t = _pose_params(dev, TRUE_ROT, TRUE_TRAN)
        p = dict(gauss, cam_unnorm_rots=r, cam_trans=t)
        rgb, dep = M.fused_rendervars(p, 1, torch.eye(4, device=dev), camera_grad=False)
        im, ds, _, _ = S.GaussianRasterizer(cam).forward_fused(
            means3D=rgb["means3D"], means2D=rgb["means2D"], opacities=rgb["opacities"], colors_precomp=rgb["colors_precomp"],
            colors_extra=dep["colors_precomp"], scales=rgb["scales"], rotations=rgb["rotations"])
        frame = dict(id=1, cam=cam, w2c=torch.eye(4, device=dev), im=im.clone(), depth=ds[0:1].clone())
    return sc, gauss, frame


def _run(sc, gauss, frame, dev, render, fused, settings_cls=None):
    from splatam_b200 import mapping as M
    fr = dict(frame)
    if settings_cls is not None:
        fr["cam"] = sc.settings(settings_cls, dev)
    r0, t0 = _pose_params(dev, [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0])    # start from the previous frame's pose
    p = dict({k: v.detach() for k, v in gauss.items()}, cam_unnorm_rots=r0, cam_trans=t0)
    losses = M.track_frame(p, fr, render=render, num_iters=40, fused=fused)
    q = torch.nn.functional.normalize(p["cam_unnorm_rots"][0, :, 1].detach(), dim=0).cpu().numpy()
    return losses, q, p["cam_trans"][0, :, 1].detach().cpu().numpy()


def reference_run(ref, dev):
    """The plain tracking loop over the reference extension `ref` (stored by tests/golden/make_golden_reference.py)."""
    sc, gauss, frame = _problem(dev)
    render = lambda settings, **rv: ref.GaussianRasterizer(raster_settings=settings)(**rv)
    losses, q, t = _run(sc, gauss, frame, dev, render, False, ref.GaussianRasterizationSettings)
    return dict(losses=np.array(losses[:8]), q=q, t=t)


def test_tracking_recovers_pose_and_matches_reference(cuda_device):
    dev = cuda_device
    true_rot, true_tran = TRUE_ROT, TRUE_TRAN
    sc, gauss, frame = _problem(dev)
    lf, qf, tf = _run(sc, gauss, frame, dev, None, True)
    lp, qp, tp = _run(sc, gauss, frame, dev, None, False)
    tq = np.array(true_rot) / np.linalg.norm(true_rot)
    assert lf[-1] < 0.2 * lf[0], (lf[0], lf[-1])
    assert np.abs(qf - tq).max() < 2e-3 and np.abs(tf - np.array(true_tran)).max() < 4e-3, (qf, tf)
    # fused and plain paths follow the same trajectory
    # (the silhouette-masked L1 sums are discontinuous in the pose, so trajectories are compared tightly only
    # over the first iterations; afterwards 1-ulp differences flip mask pixels and the small end losses drift)
    assert np.allclose(lf[:8], lp[:8], rtol=1e-3), max(abs(a - b) / b for a, b in zip(lf[:8], lp[:8]))
    assert np.abs(qf - qp).max() < 1e-3 and np.abs(tf - tp).max() < 2e-3
    z = np.load(os.path.join(GOLDEN, "reference", "loops.npz"))
    lr_, qr, tr = z["tracking_run_losses"], z["tracking_run_q"], z["tracking_run_t"]
    assert np.allclose(lp[:8], lr_[:8], rtol=1e-3), max(abs(a - b) / b for a, b in zip(lp[:8], lr_[:8]))
    assert np.abs(qp - qr).max() < 1e-3 and np.abs(tp - tr).max() < 2e-3
