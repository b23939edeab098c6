"""GPU suite of mesh extraction: sb_tsdf_integrate and the marching-cubes passes bit for bit against the numpy
restatement (oracle/mesh_numpy.py), batching, the empty and fully inside volumes, and mesh_record / extract_mesh.py
end to end on a synthetic run record, with its fusion loop free of host synchronisation."""
import json

import numpy as np
import pytest
import torch

from util import load, look_at
from oracle import mesh_numpy as O
from splatam_b200 import formats
from splatam_b200.mesh import RecordFusion, TSDFVolume, mesh_record

pytestmark = pytest.mark.gpu
H, W = 32, 40
K = np.array([[40.0, 0, 19.5], [0, 40.0, 15.5], [0, 0, 1]], np.float32)


def _frames(B, seed):
    """Random poses around a 1 m volume (some cameras inside it, so voxels lie behind them), depth near the volume's
    centre with holes (0), values past depth_max = 2.5 and NaN, and random colours."""
    g = np.random.default_rng(seed)
    w2c, depth = [], []
    for b in range(B):
        r = 0.3 if b % 3 == 0 else g.uniform(1.2, 1.8)
        d = g.normal(size=3)
        cam = r * d / np.linalg.norm(d)
        w2c.append(look_at(cam, g.uniform(-0.1, 0.1, 3)).astype(np.float32))
        base = r + g.uniform(-0.3, 0.3) + 0.1 * np.sin(np.arange(W) / 5.0)[None, :] + 0.05 * g.standard_normal((H, W))
        base[g.uniform(size=(H, W)) < 0.15] = 0.0
        base[g.uniform(size=(H, W)) < 0.05] = 3.0
        base[g.uniform(size=(H, W)) < 0.01] = np.nan
        depth.append(np.clip(base, 0, None) if b % 2 else base)
    depth = np.stack(depth).astype(np.float32)
    rgb = g.uniform(0, 1, (B, 3, H, W)).astype(np.float32)
    return depth, rgb, np.stack(w2c)


def _volume(dev, voxel=0.05):
    return TSDFVolume((-0.5, -0.45, -0.4, 0.45, 0.5, 0.55), voxel, device=dev)


def _host_state(vol):
    return [t.cpu().numpy() for t in (vol.tsdf, vol.weight, vol.color)]


@pytest.mark.parametrize("depth_max", [None, 2.5])
def test_integrate_is_bit_equal_to_the_oracle(cuda_device, depth_max):
    depth, rgb, w2c = _frames(9, seed=1)
    vol = _volume(cuda_device)
    vol.integrate(torch.from_numpy(depth).to(cuda_device), torch.from_numpy(rgb).to(cuda_device), K,
                  torch.from_numpy(w2c).to(cuda_device), depth_max=depth_max)
    tsdf, weight, color = _host_state(vol)
    t0 = np.ones_like(tsdf)
    w0 = np.zeros_like(weight)
    c0 = np.zeros_like(color)
    O.integrate(t0, w0, c0, vol.origin, vol.voxel_size, vol.trunc, depth, rgb, w2c, K, depth_max)
    assert weight.max() >= 2 and (weight > 0).mean() > 0.05 and (tsdf < 0).any()
    for a, b in ((tsdf, t0), (weight, w0), (color, c0)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_batch_equals_single_frames(cuda_device):
    depth, rgb, w2c = _frames(6, seed=2)
    d, c, w = (torch.from_numpy(x).to(cuda_device) for x in (depth, rgb, w2c))
    one, many = _volume(cuda_device), _volume(cuda_device)
    many.integrate(d, c, K, w, depth_max=2.5)
    for b in range(6):
        one.integrate(d[b], c[b], K, w[b], depth_max=2.5)
    for a, b in zip(_host_state(one), _host_state(many)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("min_weight", [1.0, 3.0])
def test_marching_cubes_is_bit_equal_to_the_oracle(cuda_device, min_weight):
    depth, rgb, w2c = _frames(12, seed=3)
    vol = _volume(cuda_device, voxel=0.04)
    vol.integrate(torch.from_numpy(depth).to(cuda_device), torch.from_numpy(rgb).to(cuda_device), K,
                  torch.from_numpy(w2c).to(cuda_device))
    v, c, f = vol.extract(min_weight)
    tsdf, weight, color = _host_state(vol)
    ov, oc, of = O.marching_cubes(tsdf, weight, color, vol.origin, vol.voxel_size, min_weight)
    assert len(of) > 50
    assert v.dtype == torch.float32 and f.dtype == torch.int32
    assert np.array_equal(v.cpu().numpy().view(np.uint32), ov.view(np.uint32))
    assert np.array_equal(c.cpu().numpy().view(np.uint32), oc.view(np.uint32))
    assert np.array_equal(f.cpu().numpy(), of)


def test_analytic_sphere_field_on_the_gpu(cuda_device):
    vol = TSDFVolume((0, 0, 0, 23, 23, 23), 1.0, device=cuda_device)
    g = torch.arange(24, dtype=torch.float32, device=cuda_device)
    z, y, x = torch.meshgrid(g, g, g, indexing="ij")
    vol.tsdf.copy_(torch.sqrt((x - 11.3) ** 2 + (y - 11.3) ** 2 + (z - 11.3) ** 2) - 7.2)
    vol.weight.fill_(1.0)
    v, c, f = vol.extract()
    ov, _, of = O.marching_cubes(*_host_state(vol), vol.origin, 1.0)
    assert np.array_equal(f.cpu().numpy(), of) and np.array_equal(v.cpu().numpy(), ov)
    fe = f.cpu().numpy()
    e = np.concatenate([fe[:, [0, 1]], fe[:, [1, 2]], fe[:, [2, 0]]])
    assert len(v) - len(np.unique(np.sort(e, 1), axis=0)) + len(fe) == 2


def test_empty_and_fully_inside_volumes(cuda_device):
    vol = _volume(cuda_device)
    for prepare in (lambda: None, lambda: (vol.tsdf.fill_(-1.0), vol.weight.fill_(1.0))):
        prepare()
        v, c, f = vol.extract()
        assert v.shape == (0, 3) and c.shape == (0, 3) and f.shape == (0, 3) and v.is_cuda
    flat = TSDFVolume((0, 0, 0, 1, 1, 0), 0.1, device=cuda_device)          # one sample thick: no cells
    flat.weight.fill_(1.0)
    assert flat.extract()[2].shape == (0, 3)


# ---- end to end: a wall of flat Gaussians ------------------------------------------------------------------------

WALL_Z = 2.0
REC_W, REC_H = 160, 120
REC_K = np.array([[150.0, 0, 79.5], [0, 150.0, 59.5], [0, 0, 1]], np.float32)


@pytest.fixture(scope="module")
def wall_record(tmp_path_factory):
    """A wall of flat anisotropic Gaussians on z = 2 (2 cm spacing, 1.5 cm x 1.5 cm x 1 mm, nearly opaque) covering
    every view of a short trajectory, saved with formats.save_run_record."""
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
    d = tmp_path_factory.mktemp("wall")
    return formats.save_run_record(str(d), gauss, rots, trans, np.zeros(P), REC_K, np.eye(4), REC_W, REC_H,
                                   [np.eye(4)] * T, [0])


def _check_wall(v, f, voxel):
    v = np.asarray(v, np.float64)
    assert len(f) > 1000
    assert np.abs(v[:, 2] - WALL_Z).max() < voxel
    # the observed middle of the wall is covered: every 5 cm cell of [-0.6, 0.6] x [-0.45, 0.45] holds a vertex
    cells = {(int(np.floor(x / 0.05)), int(np.floor(y / 0.05))) for x, y in v[:, :2]}
    want = {(i, j) for i in range(-12, 12) for j in range(-9, 9)}
    assert want <= cells, len(want - cells)


def test_mesh_record_meshes_the_wall(cuda_device, wall_record, tmp_path):
    voxel = 0.02
    v, c, f, info = mesh_record(wall_record, voxel, batch=4, device=cuda_device)
    assert info["frames"] == 6 and info["voxels"] == np.prod(info["dims"])
    _check_wall(v.cpu().numpy(), f.cpu().numpy(), voxel)
    assert float(c.min()) >= 0.15 and float(c.max()) <= 0.85
    one, _, f1, _ = mesh_record(wall_record, voxel, batch=1, device=cuda_device)
    assert torch.equal(one, v) and torch.equal(f1, f)                    # batching does not change the mesh
    path = formats.save_mesh_ply(str(tmp_path / "wall.ply"), v, c, f)
    lv, lc, lf = formats.load_mesh_ply(path)
    assert np.array_equal(lv, v.cpu().numpy()) and np.array_equal(lf, f.cpu().numpy())


def test_mesh_record_from_input_frames(cuda_device, wall_record):
    """--source input: the same frames given as depth/colour images (here the map's own renders, read back through
    a frame list) mesh the same wall."""
    rf = RecordFusion(wall_record, device=cuda_device)
    frames = []
    for k in range(len(rf.ids)):
        rf._frame_into(0, k)
        frames.append(dict(im=rf.rgb_b[0].clone(), depth=rf.depth_b[0][None].clone()))
    v0, _, f0, _ = mesh_record(wall_record, 0.02, device=cuda_device)
    v1, _, f1, _ = mesh_record(wall_record, 0.02, device=cuda_device, source=frames)
    assert torch.equal(v0, v1) and torch.equal(f0, f1)


def test_extract_mesh_tool(cuda_device, wall_record, tmp_path, capsys):
    tool = load("tools/extract_mesh.py")
    out = str(tmp_path / "mesh.ply")
    tool.main(["--record", wall_record, "--out", out, "--voxel", "0.02", "--every", "2", "--batch", "2"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line["frames"] == 3 and line["V"] > 0 and line["F"] > 1000
    assert {"voxels", "render_ms", "integrate_ms", "extract_ms"} <= set(line)
    v, c, f = formats.load_mesh_ply(out)
    assert len(v) == line["V"] and len(f) == line["F"]
    _check_wall(v, f, 0.02)


def test_fusion_loop_has_no_torch_synchronisation(cuda_device, wall_record):
    """Rendering and integrating never wait for the device; the only wait left per rendered frame is the
    rasterizer's instance-count read inside the library."""
    rf = RecordFusion(wall_record, batch=4, device=cuda_device)
    vol = TSDFVolume((-1, -1, 1.8, 1, 1, 2.2), 0.02, device=cuda_device)
    rf.fuse(vol)                                       # warms every shape
    torch.cuda.synchronize()
    vol2 = TSDFVolume((-1, -1, 1.8, 1, 1, 2.2), 0.02, device=cuda_device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rf.fuse(vol2)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(vol.tsdf, vol2.tsdf)
