"""RGB-D ICP and the photometric health check without a GPU: the numpy restatement (oracle/rgbd_icp_numpy.py) has the
derivative of its residual as its Jacobian, aligns a textured plane that depth alone cannot, reduces to
oracle/icp_numpy.py bit for bit at weight 0; the C-ABI entry points check their arguments, the product path refuses
CPU tensors, and the new settings are validated and off by default."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import icp_scene as S
from oracle import icp_numpy as G
from oracle import rgbd_icp_numpy as O
from util import bits_equal, load
from splatam_b200 import _lib, icp, reloc

H, W = 120, 160
PLANE = dict(planes=((2, 3.0),), sphere=False)


def _texture(w2c, K, depth):
    """RGB [3,H,W] of the world plane z = 3 seen by w2c: grey a smooth function of the back-projected world point."""
    h, w = depth.shape
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    z = depth.astype(np.float64)
    cam = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z, np.ones_like(z)])
    X = np.einsum("ij,jhw->ihw", np.linalg.inv(w2c), cam)
    g = 0.5 + 0.2 * np.sin(3.1 * X[0]) * np.cos(2.3 * X[1]) + 0.1 * np.sin(1.7 * X[0] + 2.9 * X[1])
    return np.stack([g, g, g]).astype(np.float32)


def _plane_views(motion):
    K = S.intrinsics(H, W)
    prev = np.eye(4)
    cur = S.rigid(S.rot(*motion[:2]), motion[2]) @ prev
    md, dd = S.depth(prev, K, H, W, **PLANE), S.depth(cur, K, H, W, **PLANE)
    ds = np.stack([md, (md > 0).astype(np.float32)])
    return K, ds, _texture(prev, K, md), dd, _texture(cur, K, dd), prev, cur


def _errors(w2c, truth):
    e = np.asarray(w2c, np.float64) @ np.linalg.inv(truth)
    return np.abs(e[:3, 3]).max(), np.degrees(Rotation.from_matrix(e[:3, :3]).magnitude())


def test_photometric_jacobian_matches_finite_differences():
    """r(xi) = I(pi(exp(xi) p)) - I_d for a linear image I(u, v) (central differences and bilinear sampling are then
    exact) has the derivative [p x g, g], g = (dpi/dp)^T grad I (float64 throughout)."""
    rng = np.random.default_rng(5)
    K = (200.0, 180.0, 80.0, 60.0)
    for _ in range(20):
        gu, gv, c = rng.normal(size=3) * 0.01
        img = lambda u, v: gu * u + gv * v + c
        p = rng.normal(size=3) * 0.3 + [0, 0, 2.5]

        def r(xi):
            q = G.exp_se3(xi) @ np.append(p, 1.0)
            return img(K[0] * q[0] / q[2] + K[2], K[1] * q[1] / q[2] + K[3])
        J = O.photometric_jacobian(p[:, None], np.array([[gu], [gv]]), K)[0]
        fd = np.array([(r(1e-6 * e) - r(-1e-6 * e)) / 2e-6 for e in np.eye(6)])
        assert np.allclose(fd, J, rtol=1e-6, atol=1e-9), (fd, J)


def test_single_textured_plane():
    """Depth alone rejects a single plane; with its texture the joint system is well conditioned and 10 cm / 5 deg
    motions are recovered to 1 mm and 0.05 deg."""
    for motion in (((0, 1, 0), 5.0, (0.1, 0.0, 0.0)), ((0, 0, 1), 5.0, (0.0, 0.1, 0.0)),
                   ((1, 0, 0), 3.0, (0.05, -0.05, 0.05))):
        K, ds, mrgb, dd, drgb, prev, cur = _plane_views(motion)
        p32 = prev.astype(np.float32)
        _, gst, _ = G.align(ds, dd, K, p32, p32)
        assert gst[0] == 0.0 and gst[5] < G.MIN_PIVOT_RATIO, gst[:8]
        out, st, _ = O.align(ds, mrgb, dd, drgb, K, p32, p32, iters=(20, 10, 10), weight=icp.DEFAULT_WEIGHT)
        dt, dr = _errors(out, cur)
        assert st[0] == 1.0 and st[5] >= G.MIN_PIVOT_RATIO and st[36] >= O.MIN_PAIRS, st[:8]
        assert dt <= 1e-3 and dr <= 0.05, (motion, dt, dr)


def test_weight_zero_reproduces_the_geometric_oracle():
    K = S.intrinsics(60, 80)
    prev = S.rigid(S.rot((1, 1, 0), 3), (0.05, 0.02, -0.1))
    cur = S.rigid(S.rot((0, 1, 0), 2), (0.03, 0.0, 0.02)) @ prev
    ds, dd = S.depth_sil(prev, K, 60, 80), S.depth(cur, K, 60, 80)
    rng = np.random.default_rng(1)
    mrgb, drgb = rng.random((3, 60, 80), np.float32), rng.random((3, 60, 80), np.float32)
    p32 = prev.astype(np.float32)
    a, sa, _ = G.align(ds, dd, K, p32, p32)
    b, sb, lv = O.align(ds, mrgb, dd, drgb, K, p32, p32, weight=0.0)
    assert bits_equal(a, b) and bits_equal(sa, sb[:36])
    assert sb[36] > 0 and np.all(np.isfinite(sb))
    # the grey pyramid averages exactly the depth pyramid's samples: NaN exactly where the depth is 0
    for L in lv:
        assert np.array_equal(np.isnan(L["model_grey"]), L["model_depth"] == 0)


def test_health_ncc_oracle():
    rng = np.random.default_rng(2)
    d = rng.uniform(1, 3, (40, 50)).astype(np.float32)
    ds = np.stack([d, np.ones_like(d)])
    rgb = rng.random((3, 40, 50), np.float32)
    st = O.health_ncc(ds, d, rgb, rgb, 0.05, 0.02, 0.05, 0.5, 0.5)
    assert st[4] == 1.0 and st[5] == 2000 and abs(st[6] - 1.0) < 1e-12
    other = rng.random((3, 40, 50), np.float32)
    st = O.health_ncc(ds, d, rgb, other, 0.05, 0.02, 0.05, 0.5, 0.5)
    assert st[4] == 0.0 and abs(st[6]) < 0.1


def test_abi_argument_checks():
    lib = _lib.load()
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert lib.sb_rgbd_icp_workspace_bytes(680, 1200, ctypes.byref(n)) == 0
    assert lib.sb_icp_workspace_bytes(680, 1200, ctypes.byref(m)) == 0 and n.value > m.value
    assert lib.sb_rgbd_icp_workspace_bytes(3, 100, ctypes.byref(n)) == 1
    assert lib.sb_rgbd_icp_workspace_bytes(100, 100, None) == 1
    it = (ctypes.c_int * 3)(10, 5, 4)
    d = 1
    args = lambda **kw: [kw.get(k, v) for k, v in dict(
        h=45, w=97, ds=d, mrgb=d, dd=d, drgb=d, fx=50.0, fy=50.0, cx=48.0, cy=22.0, prev=d, init=d, it=it, lam=0.05,
        ws=d, nb=1 << 30, out=d, st=d, stream=None).items()]
    for bad in (dict(ds=None), dict(mrgb=None), dict(drgb=None), dict(st=None), dict(it=None), dict(fx=0.0),
                dict(lam=-0.1), dict(lam=float("nan")), dict(lam=float("inf")), dict(h=2)):
        assert lib.sb_rgbd_icp_align(*args(**bad)) == 1, bad
    assert lib.sb_rgbd_icp_align(*args(nb=16)) == 2
    assert lib.sb_rgbd_icp_export(45, 97, d, 1 << 30, 3, d, d, d, d, None) == 1
    assert lib.sb_rgbd_icp_export(45, 97, d, 1 << 30, 0, d, None, d, d, None) == 1
    assert lib.sb_rgbd_icp_export(45, 97, d, 16, 0, d, d, d, d, None) == 2
    h = lambda **kw: [kw.get(k, v) for k, v in dict(
        h=45, w=97, ds=d, fd=d, mrgb=d, frgb=d, ta=0.05, tr=0.02, cov=0.05, inl=0.5, ncc=0.5, scr=d, st=d,
        stream=None).items()]
    for bad in (dict(mrgb=None), dict(frgb=None), dict(scr=None), dict(ncc=1.5), dict(ncc=float("nan")),
                dict(ta=-1.0), dict(h=0)):
        assert lib.sb_track_health_rgb(*h(**bad)) == 1, bad


def test_refuses_cpu_tensors_and_bad_arguments():
    ds, rgb, dd, eye = torch.zeros(2, 8, 8), torch.zeros(3, 8, 8), torch.zeros(8, 8), torch.eye(4)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        icp.align_rgbd(ds, rgb, dd, rgb, np.eye(3), eye, eye)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        reloc._health_rgb_of(ds, rgb, dd, rgb, reloc.config({}))


@pytest.mark.parametrize("bad", [dict(photometric=1), dict(photometric="yes"), dict(min_ncc=1.5),
                                 dict(min_ncc=-2.0), dict(min_ncc=float("nan")), dict(min_ncc=True)])
def test_bad_photometric_settings_raise(bad):
    with pytest.raises(ValueError, match="relocalise"):
        reloc.config(bad)


def test_photometric_settings_default_off():
    cfg = reloc.config({})
    assert cfg["photometric"] is False and cfg["min_ncc"] == reloc.DEFAULTS["min_ncc"]
    assert reloc.config(dict(photometric=True, min_ncc=-1.0))["min_ncc"] == -1.0


def test_pose_init_validation():
    cpu = load("tests/test_icp_cpu.py")
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        cpu._cpu_run(pose_init="rgbd_icp")
    with pytest.raises(ValueError, match="pose_init"):
        cpu._cpu_run(pose_init="rgbd")


def test_tool_flags():
    tool = load("tools/localise_sequence.py")
    a = tool.parse_args(["--record", __file__, "--dataset", "replica", "--basedir", "b", "--sequence", "s",
                         "--photometric", "--pose-init", "rgbd_icp"])
    assert a.photometric and a.pose_init == "rgbd_icp"
