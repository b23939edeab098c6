"""GPU suite of mesh depth rendering: sb_mesh_depth bit for bit against the numpy restatement
(oracle/mesh_render_numpy.py) on the meshes where a rasterizer is easiest to get wrong, MeshDepth free of host
synchronisation, and depth_l1 / eval_mesh.py --depth-views end to end on a meshed wall of Gaussians."""
import json

import numpy as np
import pytest
import torch

from util import load, look_at
from oracle.mesh_render_numpy import mesh_depth
from splatam_b200 import _lib, formats
from splatam_b200 import mesh_eval as E
from splatam_b200.mesh import RecordFusion, mesh_record

pytestmark = pytest.mark.gpu


def _K(H, W):
    f = 0.8 * max(H, W)
    return np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]])


def _random_mesh(seed, n_small=3000, n_big=12, nan=True):
    """Tiny triangles in a 1 m cube, a few huge ones through it (screen-filling, crossing the near plane of cameras
    inside the cube), shared-edge strips, repeated vertices (zero area) and a face on a NaN vertex, which MeshDepth
    refuses and the library drops."""
    g = np.random.default_rng(seed)
    c = g.uniform(-0.5, 0.5, (n_small, 1, 3))
    small = c + g.normal(0, 0.01, (n_small, 3, 3))
    big = g.uniform(-3, 3, (n_big, 3, 3))
    strip_v = g.uniform(-0.5, 0.5, (40, 3))
    v = np.concatenate([small.reshape(-1, 3), big.reshape(-1, 3), strip_v, [[np.nan, 0, 0]]]).astype(np.float32)
    nv = len(v)
    f = np.arange(3 * (n_small + n_big)).reshape(-1, 3)
    s0 = 3 * (n_small + n_big)
    strip = np.stack([np.arange(38), np.arange(1, 39), np.arange(2, 40)], 1) + s0
    degenerate = np.array([[0, 0, 1], [5, 5, 5], [nv - 1, 1, 2]] if nan else [[0, 0, 1], [5, 5, 5]])
    return v, np.concatenate([f, strip, degenerate])


def _box():
    """A closed box [-1, 1]^3 of 12 triangles."""
    v = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                  [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]])
    return v, f


def _poses(B, seed, inside=False):
    g = np.random.default_rng(seed)
    out = []
    for b in range(B):
        d = g.normal(size=3)
        r = g.uniform(0.0, 0.4) if inside or b % 3 == 0 else g.uniform(1.0, 2.5)
        # up = -y: image x = y x fwd, these views' camera rolled 180 degrees about the view axis
        out.append(look_at(r * d / np.linalg.norm(d), g.uniform(-0.2, 0.2, 3), up=(0.0, -1.0, 0.0)).astype(np.float32))
    return np.stack(out)


def _check(mesh_v, mesh_f, w2c, H, W, dev, near=0.01):
    K = _K(H, W)
    v = torch.from_numpy(np.ascontiguousarray(mesh_v, np.float32)).to(dev)
    f = torch.from_numpy(np.ascontiguousarray(mesh_f, np.int32)).to(dev)
    w = torch.from_numpy(w2c).to(dev)
    B = w.shape[0]
    with _lib.on_device(dev):
        nb = _lib.nbytes("sb_mesh_depth_workspace_bytes", f.shape[0], B, H, W)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    d = torch.empty(B, H, W, device=dev)
    fid = torch.empty(B, H, W, dtype=torch.int32, device=dev)
    _lib.call("sb_mesh_depth", v.shape[0], v, f.shape[0], f, B, H, W, w, float(K[0, 0]), float(K[1, 1]),
              float(K[0, 2]), float(K[1, 2]), near, ws, nb, d, fid, device=dev)
    want_d, want_f = mesh_depth(mesh_v, mesh_f, w2c, K, H, W, near)
    got_d, got_f = d.cpu().numpy(), fid.cpu().numpy()
    assert np.array_equal(got_d.view(np.int32), want_d.view(np.int32)), (H, W, int((got_d != want_d).sum()))
    assert np.array_equal(got_f, want_f)
    return got_d, got_f


@pytest.mark.parametrize("hw", [(1, 1), (17, 31), (500, 500)])
def test_random_meshes_are_bit_equal_to_the_oracle(cuda_device, hw):
    H, W = hw
    v, f = _random_mesh(1)
    w2c = _poses(6, seed=2)
    w2c[4] = np.nan                                                   # a non-finite pose draws nothing
    d, fid = _check(v, f, w2c, H, W, cuda_device)
    assert not (d[4] > 0).any() and (fid[4] == -1).all()
    if H * W > 1:
        assert (d > 0).mean() > 0.05
        assert ((fid >= 3000) & (fid < 3012)).any()                     # the big triangles drew


def test_camera_inside_a_closed_box(cuda_device):
    v, f = _box()
    w2c = _poses(5, seed=3, inside=True)
    d, _ = _check(v, f, w2c, 64, 80, cuda_device)
    assert (d > 0).all()                                               # no crack and nothing clipped away
    d, _ = _check(v, f, w2c, 64, 80, cuda_device, near=0.5)
    assert (d > 0).all()


def test_a_batch_equals_single_views(cuda_device):
    v, f = _random_mesh(4, nan=False)
    w2c = torch.from_numpy(_poses(8, seed=5)).to(cuda_device)
    m = E.MeshDepth(v, f, cuda_device)
    d8, f8 = m.render(w2c, _K(120, 160), 120, 160)
    for b in range(8):
        d1, f1 = m.render(w2c[b:b + 1], _K(120, 160), 120, 160)
        assert torch.equal(d1[0].view(torch.int32), d8[b].view(torch.int32)) and torch.equal(f1[0], f8[b])


def test_a_hundred_thousand_faces(cuda_device):
    v, f = _random_mesh(6, n_small=100_000, n_big=4)
    _check(v, f, _poses(3, seed=7), 96, 128, cuda_device)


def test_render_has_no_host_synchronisation(cuda_device):
    v, f = _random_mesh(8, nan=False)
    m = E.MeshDepth(v, f, cuda_device)
    w2c = torch.from_numpy(_poses(4, seed=9)).to(cuda_device)
    want = m.render(w2c, _K(50, 60), 50, 60)
    out = (torch.empty_like(want[0]), torch.empty_like(want[1]))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = m.render(w2c, _K(50, 60), 50, 60)
        m.render(w2c, _K(50, 60), 50, 60, out=out)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]) and torch.equal(out[1], want[1])


# ---- end to end: the wall of Gaussians of test_mesh_eval_gpu.py ----------------------------------------------------

WALL_Z = 2.0
REC_W, REC_H = 160, 120
REC_K = np.array([[150.0, 0, 79.5], [0, 150.0, 59.5], [0, 0, 1]], np.float32)
VOXEL = 0.02
# view centres 0.4-0.8 m in front of the observed middle of the wall
VIEW_BOX = np.float32([[-0.3, -0.3, 1.2], [0.3, 0.3, 1.6]])


def _plane(n, drop_checkerboard=False):
    gx, gy = np.meshgrid(np.linspace(-4, 4, n), np.linspace(-4, 4, n))
    gv = np.c_[gx.ravel(), gy.ravel(), np.full(n * n, WALL_Z)].astype(np.float32)
    q = np.arange(n - 1)
    i00 = (q[:, None] * n + q[None, :]).ravel()
    keep = np.ones(len(i00), bool)
    if drop_checkerboard:
        keep = ((q[:, None] + q[None, :]) % 2 == 1).ravel()
    i00 = i00[keep]
    return gv, np.concatenate([np.c_[i00, i00 + 1, i00 + n + 1], np.c_[i00, i00 + n + 1, i00 + n]])


@pytest.fixture(scope="module")
def wall(tmp_path_factory, cuda_device):
    """A wall of flat Gaussians on z = 2 seen by six cameras, its mesh, the frames it was meshed from (rendered
    depth, map-frame w2c) and a ground-truth plane on z = 2, 8 m x 8 m in 2,500 quads (also as a PLY)."""
    g = np.random.default_rng(0)
    xs, ys = np.meshgrid(np.arange(-1.5, 1.5, 0.02), np.arange(-1.2, 1.2, 0.02))
    P = xs.size
    means = np.c_[xs.ravel(), ys.ravel(), np.full(P, WALL_Z)].astype(np.float32)
    gauss = dict(means3D=means, rgb_colors=g.uniform(0.2, 0.8, (P, 3)).astype(np.float32),
                 unnorm_rotations=np.tile(np.float32([1, 0, 0, 0]), (P, 1)),
                 logit_opacities=np.full((P, 1), 6.0, np.float32),
                 log_scales=np.log(np.tile(np.float32([0.015, 0.015, 0.001]), (P, 1))))
    T = 6
    t = np.arange(T)
    rots = np.zeros((1, 4, T), np.float32)
    rots[0, 0] = 1.0
    rots[0, 2] = 0.03 * np.sin(t)
    trans = np.zeros((1, 3, T), np.float32)
    trans[0, 0] = 0.05 * t - 0.1
    trans[0, 2] = 0.1 * np.cos(t)
    d = tmp_path_factory.mktemp("wall_depth")
    record = formats.save_run_record(str(d), gauss, rots, trans, np.zeros(P), REC_K, np.eye(4), REC_W, REC_H,
                                     [np.eye(4)] * T, [0])
    v, c, f, _ = mesh_record(record, VOXEL, device=cuda_device)
    pred = formats.save_mesh_ply(str(d / "mesh.ply"), v, c, f)
    rf = RecordFusion(record, device=cuda_device)
    frames = []
    for k in range(len(rf.ids)):
        rf._frame_into(0, k)
        frames.append(dict(depth=rf.depth_b[0][None].clone(), gt_w2c=rf.w2cs[k].clone()))
    gv, gf = _plane(51)
    gt = formats.save_mesh_ply(str(d / "gt.ply"), gv, np.zeros_like(gv), gf)
    return dict(pred=pred, gt=gt, frames=frames, K=rf.K, mesh=(v, f), gt_mesh=(gv, gf))


def test_identical_meshes_score_zero(cuda_device, wall):
    out = E.depth_l1(wall["gt_mesh"], wall["gt_mesh"], views=20, gt_kept=VIEW_BOX, device=cuda_device)
    assert out["depth_l1"] == 0 and out["depth_l1_surface"] == 0 and out["hole_ratio"] == 0, out
    assert out["views_used"] == 20 and out["views_drawn"] >= 20 and out["render_ms"] > 0 and out["cull_ms"] == 0


def test_meshed_wall_is_within_a_voxel_where_it_has_a_surface(cuda_device, wall):
    out = E.depth_l1(wall["mesh"], wall["gt_mesh"], wall["frames"], wall["K"], views=20, gt_kept=VIEW_BOX,
                     device=cuda_device)
    assert out["views_used"] >= 1 and out["cull_ms"] > 0, out
    assert out["depth_l1_surface"] < VOXEL and out["depth_l1"] >= out["depth_l1_surface"], out
    again = E.depth_l1(wall["mesh"], wall["gt_mesh"], wall["frames"], wall["K"], views=20, gt_kept=VIEW_BOX,
                       device=cuda_device)
    assert again["depth_l1"] == out["depth_l1"] and again["views_drawn"] == out["views_drawn"]


def test_removed_quads_show_as_holes(cuda_device, wall):
    holes = _plane(51, drop_checkerboard=True)
    out = E.depth_l1(holes, wall["gt_mesh"], views=20, gt_kept=VIEW_BOX, device=cuda_device)
    assert abs(out["hole_ratio"] - 0.5) < 0.05 and out["depth_l1_surface"] == 0, out
    assert out["depth_l1"] > 0.5 * 0.4


def test_evaluate_mesh_and_the_tool_report_depth_l1(cuda_device, wall, tmp_path, capsys):
    # a room: the views are centred in the box of the ground-truth samples, which a lone plane leaves flat
    rv, rf = _box()
    room = formats.save_mesh_ply(str(tmp_path / "room.ply"), 2 * rv, np.zeros_like(rv), rf)
    pred, gt = formats.load_mesh_ply(wall["pred"]), formats.load_mesh_ply(room)
    pred, gt = (pred[0], pred[2]), (gt[0], gt[2])
    base = E.evaluate_mesh(pred, gt, samples=50_000, seed=4, device=cuda_device)
    full = E.evaluate_mesh(pred, gt, samples=50_000, seed=4, device=cuda_device, depth_views=5)
    assert {k: full[k] for k in base if not k.endswith("_ms")} == {k: base[k] for k in base if not k.endswith("_ms")}
    assert set(full) - set(base) == {"depth_l1", "depth_l1_surface", "hole_ratio", "depth_views_used",
                                     "depth_views_drawn", "depth_render_ms", "depth_cull_ms"}
    tool = load("tools/eval_mesh.py")
    tool.main(["--mesh", wall["pred"], "--gt-mesh", room, "--no-cull", "--samples", "50000", "--seed", "4",
               "--depth-views", "5"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line["depth_l1_cm"] == 100 * full["depth_l1"] and line["hole_ratio"] == full["hole_ratio"]
    assert line["depth_l1_surface_cm"] == 100 * full["depth_l1_surface"]
    assert line["depth_views_used"] == full["depth_views_used"] == 5
    assert line["depth_views_drawn"] == full["depth_views_drawn"] and line["render_ms"] > 0
    tool.main(["--mesh", wall["pred"], "--gt-mesh", room, "--no-cull", "--samples", "50000", "--seed", "4"])
    assert "depth_l1_cm" not in json.loads(capsys.readouterr().out.strip().splitlines()[-1])
