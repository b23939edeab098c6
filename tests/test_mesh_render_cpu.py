"""CPU suite of mesh depth rendering: the rasterizer rule through its numpy restatement (oracle/mesh_render_numpy.py),
the random-view protocol, the depth-L1 arithmetic on hand-built depth maps, and the library's and the tool's argument
checks without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from util import load
from oracle.mesh_render_numpy import mesh_depth
from splatam_b200 import _lib, mesh_eval as E

EYE = np.eye(4, dtype=np.float32)[None]


def _K(fx, cx, fy=None, cy=None):
    return np.array([[fx, 0, cx], [0, fx if fy is None else fy, cx if cy is None else cy], [0, 0, 1]])


def _grid(n, lo, hi, z, jitter=0.0, seed=0):
    """A plane z = z over [lo, hi]^2 of n x n vertices, two triangles per quad (interior vertices jittered)."""
    x, y = np.meshgrid(np.linspace(lo, hi, n), np.linspace(lo, hi, n))
    if jitter:
        g = np.random.default_rng(seed)
        inner = np.zeros((n, n), bool)
        inner[1:-1, 1:-1] = True
        x = x + np.where(inner, g.uniform(-jitter, jitter, x.shape), 0)
        y = y + np.where(inner, g.uniform(-jitter, jitter, y.shape), 0)
    v = np.c_[x.ravel(), y.ravel(), np.full(n * n, z)].astype(np.float32)
    q = np.arange(n - 1)
    i = (q[:, None] * n + q[None, :]).ravel()
    return v, np.concatenate([np.c_[i, i + 1, i + n + 1], np.c_[i, i + n + 1, i + n]])


QUAD = np.float32([[-1, -1, 2], [1, -1, 2], [1, 1, 2], [-1, 1, 2]])
TWO = np.array([[0, 1, 2], [0, 2, 3]])


def test_plane_facing_the_camera_covers_exactly_its_projection():
    d, fid = mesh_depth(QUAD, TWO, EYE, _K(10.0, 7.5, cy=5.5), 12, 16)
    want = np.zeros((12, 16), bool)
    want[1:11, 3:13] = True                                      # u in [2.5, 12.5], v in [0.5, 10.5]
    assert np.array_equal(d[0] > 0, want) and np.array_equal(fid[0] >= 0, want)
    assert np.all(np.abs(d[0][want].view(np.int32) - np.float32(2).view(np.int32)) <= 4)


def test_slanted_plane_matches_the_closed_form():
    v = np.float32([[-3, -3, 0.5], [3, -3, 3.5], [3, 3, 3.5], [-3, 3, 0.5]])    # z = 2 + 0.5 x
    K = _K(20.0, 15.5)
    d, _ = mesh_depth(v, TWO, EYE, K, 32, 32)
    c = np.arange(32)[None, :].repeat(32, 0)
    xn = (c - K[0, 2]) / K[0, 0]
    want = 2.0 / (1.0 - 0.5 * xn)
    assert (d[0] > 0).all()
    assert np.max(np.abs(d[0] - want) / want) < 1e-6


def test_near_plane_clipping():
    # a floor y = 1 from 10 m behind the camera to 200 m ahead: clipped, its visible part fills the lower image
    v = np.float32([[-200, 1, -10], [200, 1, -10], [0, 1, 200]])
    K = _K(20.0, 15.5)
    for f in ([[0, 1, 2]], [[1, 2, 0]], [[2, 1, 0]]):
        d, fid = mesh_depth(v, f, EYE, K, 32, 32, near=0.01)
        assert not (d[0][:16] > 0).any()
        rows = np.arange(16, 32)
        want = K[1, 1] / (rows - K[1, 2])                        # depth of the floor on row r
        assert (fid[0][16:] == 0).all()
        assert np.max(np.abs(d[0][16:] - want[:, None]) / want[:, None]) < 1e-4    # float32 at 200 m
    behind = np.float32([[-1, -1, -1], [1, -1, -2], [0, 1, -0.5]])
    d, fid = mesh_depth(behind, [[0, 1, 2]], EYE, K, 32, 32)
    assert not (d > 0).any() and (fid == -1).all()
    # a triangle whose one vertex lies behind the near plane keeps only the part in front of it
    part = np.float32([[0, 0, -1], [1, -1, 3], [-1, -1, 3]])
    d, _ = mesh_depth(part, [[0, 1, 2]], EYE, K, 32, 32, near=0.5)
    assert (d[0] > 0).any() and d[0][d[0] > 0].min() >= 0.5 * (1 - 1e-6)


def test_both_windings_draw_the_same():
    K = _K(10.0, 7.5, cy=5.5)
    a = mesh_depth(QUAD, TWO, EYE, K, 12, 16)
    b = mesh_depth(QUAD, TWO[:, ::-1], EYE, K, 12, 16)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("jitter", [0.0, 0.006])
def test_a_plane_of_2500_quads_has_no_cracks(jitter):
    # vertices on pixel centres (jitter 0) put shared edges through pixel centres; jitter moves them off
    v, f = _grid(51, -0.5, 0.5, 1.0, jitter=jitter, seed=3)
    assert len(f) == 5000
    d, fid = mesh_depth(v, f, EYE, _K(100.0, 59.0), 118, 118)
    inner = np.zeros((118, 118), bool)
    inner[9:110, 9:110] = True                                   # u in [9, 109]
    assert (d[0][inner] > 0).all() and not (d[0][~inner] > 0).any()
    assert np.array_equal(fid[0] >= 0, inner)


def test_nearest_face_wins_and_ties_go_to_the_lower_index():
    K = _K(10.0, 7.5, cy=5.5)
    far = QUAD * np.float32([1, 1, 1.5])                         # z = 3
    v = np.concatenate([far, QUAD])
    f = np.array([[0, 1, 2], [4, 5, 6]])                         # the far face has the lower index
    d, fid = mesh_depth(v, f, EYE, K, 12, 16)
    both = (fid[0] >= 0) & (d[0] < 2.5)
    assert both.any() and (fid[0][both] == 1).all()
    d, fid = mesh_depth(QUAD, np.array([[0, 1, 2], [0, 2, 1], [0, 1, 2]]), EYE, K, 12, 16)
    assert (fid[0][fid[0] >= 0] == 0).all()


def test_zero_area_and_non_finite_faces_draw_nothing():
    v = np.concatenate([QUAD, np.float32([[np.nan, 0, 2]])])
    d, fid = mesh_depth(v, [[0, 0, 2], [1, 1, 1], [0, 4, 2], [0, 1, 5]], EYE, _K(10.0, 7.5, cy=5.5), 12, 16)
    assert not (d > 0).any() and (fid == -1).all()
    nan_pose = EYE.copy()
    nan_pose[0, 0, 3] = np.nan
    d, _ = mesh_depth(QUAD, TWO, nan_pose, _K(10.0, 7.5, cy=5.5), 12, 16)
    assert not (d > 0).any()


# ---- the random views and the metric -----------------------------------------------------------------------------

def test_depth_views_are_seeded_in_the_box_and_have_no_roll():
    g = np.random.default_rng(0)
    pts = g.uniform([-1, 0, 2], [3, 1, 5], (500, 3)).astype(np.float32)
    a = E.depth_views(pts, 200, seed=7)
    assert a.dtype == np.float32 and a.shape == (200, 4, 4)
    assert np.array_equal(a, E.depth_views(torch.from_numpy(pts), 200, seed=7))
    assert np.array_equal(a[:50], E.depth_views(pts, 50, seed=7))
    assert not np.array_equal(a, E.depth_views(pts, 200, seed=8))
    R, t = a[:, :3, :3].astype(np.float64), a[:, :3, 3].astype(np.float64)
    assert np.allclose(R @ R.transpose(0, 2, 1), np.eye(3), atol=1e-6) and np.allclose(np.linalg.det(R), 1, atol=1e-6)
    centre = -np.einsum("bji,bj->bi", R, t)
    lo, hi = pts.min(0), pts.max(0)
    assert np.all(centre >= lo - 1e-5) and np.all(centre <= hi + 1e-5)
    assert np.all(np.abs(R[:, 0, 1]) < 1e-6)                     # camera x is perpendicular to the map's y
    assert np.all(np.abs(R[:, 2, 1]) < 0.99)                     # no view along +-y
    assert np.all(R[:, 1, 1] > 0)                                # "down" stays on the side of +y


def test_depth_l1_arithmetic_on_hand_built_maps():
    gt = torch.tensor([[[2.0, 2.0], [2.0, 0.0]],                # 3 scored pixels
                       [[1.0, 0.0], [0.0, 0.0]],                # 1 scored pixel: below half, rejected
                       [[4.0, 4.0], [4.0, 4.0]]])
    pred = torch.tensor([[[2.5, 0.0], [1.0, 3.0]],              # errors 0.5, 2 (a hole), 1
                         [[1.0, 1.0], [1.0, 1.0]],
                         [[4.0, 4.0], [4.0, 3.0]]])              # errors 0, 0, 0, 1
    sums = E.depth_sums(pred, gt, gt > 0)
    assert sums.dtype == torch.float64
    assert np.array_equal(sums.numpy(), [[3, 3.5, 2, 1.5], [1, 0, 1, 0], [4, 1, 4, 1]])
    out = E.depth_scores(sums.numpy(), 4, views=10)
    assert out["views_used"] == 2
    assert out["depth_l1"] == pytest.approx((3.5 / 3 + 1 / 4) / 2, rel=1e-15)
    assert out["depth_l1_surface"] == pytest.approx((1.5 / 2 + 1 / 4) / 2, rel=1e-15)
    assert out["hole_ratio"] == pytest.approx(1 / 7, rel=1e-15)
    assert E.depth_scores(sums.numpy(), 4, views=1)["views_used"] == 1
    with pytest.raises(ValueError, match="map's frame"):
        E.depth_scores(sums.numpy()[1:2], 4, views=10)


def test_eval_mesh_depth_views_argument(tmp_path):
    tool = load("tools/eval_mesh.py")
    from splatam_b200 import formats
    mesh = formats.save_mesh_ply(str(tmp_path / "m.ply"), QUAD, np.zeros((4, 3)), TWO)
    ok = ["--mesh", mesh, "--gt-mesh", mesh, "--no-cull"]
    assert tool.parse_args(ok).depth_views == 0
    assert tool.parse_args(ok + ["--depth-views", "5"]).depth_views == 5
    with pytest.raises(SystemExit):
        tool.parse_args(ok + ["--depth-views", "-1"])


# ---- the library and the Python layer without a GPU ----------------------------------------------------------------

def test_mesh_depth_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_mesh_depth_workspace_bytes(10, 2, 8, 8, ctypes.byref(n)) == 0 and n.value >= 8 * 128 + 8 * 21
    for bad in ((0, 1, 8, 8), (10, 0, 8, 8), (10, 1, 0, 8), (10, 1, 8, 0), (10, 2, 1 << 15, 1 << 15),
                (1 << 30, 2, 1, 1)):
        assert lib.sb_mesh_depth_workspace_bytes(*bad, ctypes.byref(n)) == 1, bad
    assert lib.sb_mesh_depth_workspace_bytes(10, 1, 8, 8, None) == 1
    good = [3, 1, 1, 1, 1, 8, 8, 1, 10.0, 10.0, 4.0, 4.0, 0.01, 1, 1 << 20, 1, 1, None]
    for i, val in ((1, None), (3, None), (7, None), (13, None), (15, None), (16, None), (0, 0), (2, 0), (4, 0),
                   (5, 0), (6, 0), (8, 0.0), (9, -1.0), (8, float("nan")), (10, float("inf")), (12, 0.0),
                   (12, -0.01), (12, float("nan"))):
        args = list(good)
        args[i] = val
        assert lib.sb_mesh_depth(*args) == 1, (i, val)
    args = list(good)
    args[14] = 16
    assert lib.sb_mesh_depth(*args) == 2                         # short workspace


def test_mesh_depth_host_checks_and_no_cpu_fallback():
    with pytest.raises(ValueError, match=r"\[0, 4\)"):
        E.MeshDepth(QUAD, [[0, 1, 4]], "cuda:0")
    with pytest.raises(ValueError, match=r"\[0, 4\)"):
        E.MeshDepth(QUAD, [[0, 1, -1]], "cuda:0")
    bad = QUAD.copy()
    bad[3, 0] = np.inf
    with pytest.raises(ValueError, match="finite"):
        E.MeshDepth(bad, TWO, "cuda:0")
    with pytest.raises(ValueError, match="empty"):
        E.MeshDepth(QUAD, np.zeros((0, 3), np.int64), "cuda:0")
    with pytest.raises(ValueError, match="integers"):
        E.MeshDepth(QUAD, np.float32(TWO), "cuda:0")
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.MeshDepth(QUAD, TWO, "cpu")
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.depth_l1((QUAD, TWO), (QUAD, TWO), device="cpu")
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.evaluate_mesh((QUAD, TWO), (QUAD, TWO), device="cpu", depth_views=5)
