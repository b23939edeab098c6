"""ICP pose initialisation without a GPU: the numpy restatement (oracle/icp_numpy.py) recovers known motions of an
analytic scene and rejects a degenerate one, its Jacobian is the derivative of its residual, the C-ABI entry points
check their arguments, and the product path refuses CPU tensors."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import icp_scene as S
import scenes
from oracle import icp_numpy as O
from util import bits_equal, cpu_render
from splatam_b200 import _lib, slam

H, W = 240, 320
PREV = S.rigid(S.rot((1, 1, 0), 3), (0.05, 0.02, -0.1))
MOTIONS = [((0, 1, 0), 5, (0.1, 0, 0)), ((0, 1, 0), -5, (0.1, 0, 0)), ((1, 0, 0), 5, (0, 0.1, 0)),
           ((0, 0, 1), 5, (0, 0, 0.1)), ((1, 2, -1), 4, (-0.06, 0.05, 0.06)), ((0.3, -1, 0.5), 2, (0.02, 0.0, -0.03))]


def _errors(w2c, truth):
    e = np.asarray(w2c, np.float64) @ np.linalg.inv(truth)
    return np.abs(e[:3, 3]).max(), Rotation.from_matrix(e[:3, :3]).magnitude()


@pytest.mark.parametrize("axis,deg,t", MOTIONS)
def test_oracle_recovers_rigid_motions(axis, deg, t):
    """Three orthogonal planes and a sphere; the frame moved by up to 10 cm and 5 degrees from the map's view, and
    the guess is the map's pose (no velocity): the ICP pose is within 0.1 mm and 1e-4 rad of the truth."""
    K = S.intrinsics(H, W)
    cur = S.rigid(S.rot(axis, deg), t) @ PREV
    guess = PREV.astype(np.float32)
    out, st, _ = O.align(S.depth_sil(PREV, K, H, W), S.depth(cur, K, H, W), K, guess, guess)
    dt, dr = _errors(out, cur)
    assert st[0] == 1.0 and st[5] >= O.MIN_PIVOT_RATIO and st[2] < 1e-3, st[:8]
    assert dt <= 1e-4 and dr <= 1e-4, (dt, dr)


def test_jacobian_matches_finite_differences():
    """r(xi) = n.(exp(xi) p - q) has the derivative [p x n, n] at xi = 0 (float64 throughout)."""
    rng = np.random.default_rng(4)
    for _ in range(20):
        p, q = rng.normal(size=3) + [0, 0, 3], rng.normal(size=3) + [0, 0, 3]
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        r = lambda xi: n @ (O.exp_se3(xi) @ np.append(p, 1.0) - q)
        J = np.concatenate([np.cross(p, n), n])
        fd = np.array([(r(1e-6 * e) - r(-1e-6 * e)) / 2e-6 for e in np.eye(6)])
        assert np.allclose(fd, J, rtol=0, atol=1e-7), (fd, J)
    # the oracle's per-pixel Jacobian is that formula in float32
    K = S.intrinsics(60, 80)
    lv = O.pyramid(S.depth_sil(PREV, K, 60, 80), S.depth(PREV, K, 60, 80), K)
    _, _, Jf, _ = O.associate(lv[0], np.eye(4)[:3], 0)
    assert len(Jf) > 1000 and np.all(np.isfinite(Jf))


def test_single_plane_is_rejected_and_the_guess_kept():
    """A single plane leaves three degrees of freedom free: the conditioning test rejects the pose and the guess
    comes back bit for bit."""
    K = S.intrinsics(120, 160)
    plane = dict(planes=((2, 3.0),), sphere=False)
    prev = np.eye(4)
    cur = S.rigid(S.rot((0, 1, 0), 1), (0.02, 0.0, 0.01))
    guess = S.rigid(np.eye(3), (0.01, 0.0, 0.0)).astype(np.float32)
    out, st, _ = O.align(S.depth_sil(prev, K, 120, 160, **plane), S.depth(cur, K, 120, 160, **plane), K,
                         prev.astype(np.float32), guess)
    assert st[0] == 0.0 and st[5] < O.MIN_PIVOT_RATIO, st[:8]
    assert bits_equal(out, guess)


def test_abi_symbols_and_argument_checks():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_icp_workspace_bytes(680, 1200, ctypes.byref(n)) == 0
    assert n.value >= (4 * 11 + 1) * 680 * 1200                  # level 0: 11 float maps and the association codes
    assert lib.sb_icp_workspace_bytes(3, 100, ctypes.byref(n)) == 1
    assert lib.sb_icp_workspace_bytes(100, 0, ctypes.byref(n)) == 1
    assert lib.sb_icp_workspace_bytes(100, 100, None) == 1
    it = (ctypes.c_int * 3)(10, 5, 4)
    bad_it = (ctypes.c_int * 3)(10, -1, 4)
    d = 1                                                          # non-null dummy pointers, never dereferenced
    args = lambda **kw: [kw.get(k, v) for k, v in dict(
        h=45, w=97, ds=d, dd=d, fx=50.0, fy=50.0, cx=48.0, cy=22.0, prev=d, init=d, it=it, ws=d, nb=1 << 30, out=d,
        st=d, stream=None).items()]
    assert lib.sb_icp_align(*args(ds=None)) == 1
    assert lib.sb_icp_align(*args(st=None)) == 1
    assert lib.sb_icp_align(*args(it=None)) == 1
    assert lib.sb_icp_align(*args(it=bad_it)) == 1
    assert lib.sb_icp_align(*args(fx=0.0)) == 1
    assert lib.sb_icp_align(*args(cy=float("nan"))) == 1
    assert lib.sb_icp_align(*args(h=2)) == 1
    assert lib.sb_icp_align(*args(nb=16)) == 2                     # SB_ERR_WORKSPACE
    assert lib.sb_icp_export(45, 97, d, 1 << 30, 3, d, d, d, d, d, d, None) == 1
    assert lib.sb_icp_export(45, 97, d, 16, 0, d, d, d, d, d, d, None) == 2


def test_align_refuses_cpu_tensors():
    from splatam_b200 import icp
    ds, dd, eye = torch.zeros(2, 8, 8), torch.zeros(8, 8), torch.eye(4)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        icp.align(ds, dd, np.eye(3), eye, eye)


def _cpu_run(**kw):
    import splatam_b200 as SB
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(SB.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(3, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(3)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    torch.manual_seed(1); np.random.seed(1)
    return slam.run_slam(gt, frames, cam, render=cpu_render, fused=False, tracking_iters=2, mapping_iters=1,
                         keyframe_every=1, window=2, intrinsics=K, **kw)


def test_run_slam_icp_needs_cuda_and_a_known_mode():
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        _cpu_run(pose_init="icp")
    with pytest.raises(ValueError, match="pose_init"):
        _cpu_run(pose_init="icp_odometry")


def test_constant_velocity_equals_the_default():
    torch.set_num_threads(4)
    a, b = _cpu_run(), _cpu_run(pose_init="constant_velocity")
    assert "icp" not in a and "icp" not in b
    for k in ("rots", "trans"):
        assert bits_equal(a[k].numpy(), b[k].numpy()), k
    for k in a["gauss"]:
        assert bits_equal(a["gauss"][k].numpy(), b["gauss"][k].numpy()), k
    assert a["psnr"] == b["psnr"]
