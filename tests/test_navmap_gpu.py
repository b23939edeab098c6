"""GPU suite of navigation maps: sb_nav_labels, sb_esdf and sb_esdf_query bit for bit against the numpy restatement
(oracle/navmap_numpy.py) and the signed squared distance against scipy, NavMap free of host synchronisation, and
nav_record / tools/nav_map.py end to end on a closed box room seen from inside."""
import json
import math

import numpy as np
import pytest
import torch
from scipy import ndimage

import scenes
from util import load, look_at
from oracle import navmap_numpy as O
from splatam_b200 import formats, mapping
from splatam_b200.mesh import RecordFusion, TSDFVolume
from splatam_b200.navmap import NavMap, nav_record

pytestmark = pytest.mark.gpu

TRUNC, MIN_W, OCC = 0.2, 1.0, 0.025


def _volume(shape, dev, p_occ, seed):
    """A TSDFVolume of `shape` (nz, ny, nx) holding random samples: occupied (T = -0.5) with probability p_occ,
    T = t_eq (T * trunc == occ_dist exactly) for a few, free otherwise; W = 0 for a tenth, W == min_weight for some."""
    nz, ny, nx = shape
    o, v = np.array([0.25, -0.5, 0.75]), 0.25                 # exact in binary: the grid is exactly `shape`
    vol = TSDFVolume(np.concatenate([o, o + v * (np.array([nx, ny, nz]) - 1)]), v, TRUNC, device=dev)
    assert (vol.nz, vol.ny, vol.nx) == shape, (vol.nz, vol.ny, vol.nx)
    g = np.random.default_rng(seed)
    u = g.uniform(size=shape)
    t = np.where(u < p_occ, -0.5, g.uniform(0.2, 1.0, shape)).astype(np.float32)
    t[g.uniform(size=shape) < 0.01] = np.float32(OCC) / np.float32(TRUNC)
    w = np.where(g.uniform(size=shape) < 0.1, 0.0, np.where(g.uniform(size=shape) < 0.2, MIN_W, 3.0))
    vol.tsdf.copy_(torch.from_numpy(t))
    vol.weight.copy_(torch.from_numpy(w.astype(np.float32)))
    return vol, t, w.astype(np.float32)


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _same_floats(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(_bits(a[~np.isnan(a)]), _bits(b[~np.isnan(b)]))


CASES = [((1, 1, 1), 0.3), ((1, 1, 37), 0.05), ((37, 1, 1), 0.05), ((5, 64, 3), 0.05), ((3, 4, 1100), 0.01),
         ((300, 2, 3), 0.01), ((5, 64, 3), 0.0), ((5, 64, 3), 1.0), ((256, 256, 256), 0.3)]


@pytest.mark.parametrize("shape,p_occ", CASES)
def test_kernels_are_bit_equal_to_the_oracle(cuda_device, shape, p_occ):
    vol, t, w = _volume(shape, cuda_device, p_occ, seed=sum(shape))
    for uio in (True, False):
        nm = NavMap.from_volume(vol, MIN_W, OCC, unknown_is_obstacle=uio)
        lab = O.labels(t, w, np.float32(TRUNC), MIN_W, np.float32(OCC))
        assert np.array_equal(nm.labels.cpu().numpy(), lab)
        obst = O.obstacles(lab, uio)
        sd2 = O.signed_sq_distance(obst)
        assert np.array_equal(nm.sd2.cpu().numpy(), sd2)
        if obst.any() and not obst.all():
            out = np.round(ndimage.distance_transform_edt(~obst) ** 2)
            ins = np.round(ndimage.distance_transform_edt(obst) ** 2)
            assert np.array_equal(sd2, np.where(obst, -ins, out).astype(np.int64))
        esdf = O.esdf_from_sd2(sd2, vol.voxel_size)
        assert np.array_equal(_bits(nm.esdf.cpu().numpy()), _bits(esdf))
        if min(shape) < 2:
            continue
        g = np.random.default_rng(7)
        lo, hi = vol.origin.astype(np.float64), vol.origin + vol.voxel_size * (np.array(shape[::-1]) - 1.0)
        pts = g.uniform(lo - 0.03, hi + 0.03, (20000, 3))
        pts[:8] = [lo, hi, [lo[0], hi[1], lo[2]], lo - 1e-4, hi + 1e-4, [np.nan, 0, 0], [np.inf, 0, 0], lo + 0.1251]
        pts = pts.astype(np.float32)
        d, gr = nm.distance(torch.from_numpy(pts).to(cuda_device))
        od, og = O.query(esdf, vol.origin, vol.voxel_size, pts)
        assert _same_floats(d.cpu().numpy(), od) and _same_floats(gr.cpu().numpy(), og)
        assert not np.isnan(od[:3]).any() and np.isnan(od[3:7]).all()     # the first and last samples are inside


@pytest.mark.parametrize("tsdf,sd2,inf", [(1.0, O.INT32_MAX, np.inf), (-1.0, -O.INT32_MAX, -np.inf)])
def test_empty_and_full_obstacle_sets(cuda_device, tsdf, sd2, inf):
    vol, _, _ = _volume((3, 4, 5), cuda_device, 0.0, seed=0)
    vol.tsdf.fill_(tsdf)
    vol.weight.fill_(2.0)
    nm = NavMap.from_volume(vol)
    assert (nm.sd2 == sd2).all() and (nm.esdf == inf).all()
    d, g = nm.distance(torch.from_numpy(vol.origin + 0.3).to(cuda_device))
    assert float(d[0]) == inf and (g == 0).all()


def test_navmap_issues_no_host_synchronisation(cuda_device):
    vol, _, _ = _volume((20, 30, 40), cuda_device, 0.05, seed=3)
    pts = torch.rand(1000, 3, device=cuda_device) + torch.from_numpy(vol.origin).to(cuda_device)
    NavMap.from_volume(vol).distance(pts)                       # warms every shape
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        nm = NavMap.from_volume(vol, unknown_is_obstacle=False)
        d, g = nm.distance(pts)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert d.shape == (1000,) and g.shape == (1000, 3)


# ---- end to end: a closed box room, seen from inside -------------------------------------------------------------------

HALF = np.array([2.0, 1.2, 2.0])
CENTRE = np.array([0.0, 0.0, 0.3])
CAM = dict(w=256, h=192, fx=90.0, fy=90.0, cx=127.5, cy=95.5)     # 110 x 94 degrees: six views see every direction
VIEW_POINT = CENTRE + np.array([0.0137, 0.0213, 0.0171])          # off the 5 cm sample lattice
VOXEL = 0.05
SIL = 0.9                     # rendered depth where the silhouette passes this: no pixel of the closed room is a hole


def write_room_record(directory, P=400_000, scale=0.015, cam=None):
    """scenes.loop_room with P splats of `scale` metres, seen by six axis-aligned views from VIEW_POINT and four
    loop_trajectory frames, saved with formats.save_run_record; returns the path."""
    cam = CAM if cam is None else cam
    sc = scenes.loop_room(P=P, cam=cam, half=tuple(HALF), centre=tuple(CENTRE))
    gauss = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
                 logit_opacities=torch.logit(sc.opacities), log_scales=torch.full((P, 1), math.log(scale)))
    rots, trans = [], []
    for d in np.vstack([np.eye(3), -np.eye(3)]):
        w2c = torch.from_numpy(look_at(VIEW_POINT, VIEW_POINT + d)).float()
        rots.append(mapping.matrix_to_quaternion(w2c[:3, :3]))
        trans.append(w2c[:3, 3])
    lr, lt = scenes.loop_trajectory(9, "cpu")
    for s in (1, 3, 5, 7):
        rots.append(lr[0, :, s])
        trans.append(lt[0, :, s])
    rots = torch.stack(rots, -1)[None]
    trans = torch.stack(trans, -1)[None]
    T = rots.shape[-1]
    K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], np.float32)
    return formats.save_run_record(str(directory), gauss, rots, trans, np.zeros(P), K, np.eye(4), cam["w"], cam["h"],
                                   [np.eye(4)] * T, [0])


@pytest.fixture(scope="module")
def room_record(tmp_path_factory):
    return write_room_record(tmp_path_factory.mktemp("room"))


def _sample_coords(nm):
    g = [nm.origin[a] + nm.voxel_size * np.arange(n, dtype=np.float32)
         for a, n in enumerate((nm.nx, nm.ny, nm.nz))]
    z, y, x = np.meshgrid(g[2], g[1], g[0], indexing="ij")
    return np.stack([x, y, z], -1).astype(np.float64)


def _wall_gaps(p):
    """Distance of points [..., 3] to each of the six walls (positive inside the room): [..., 6]."""
    rel = p - CENTRE
    return np.concatenate([HALF - rel, HALF + rel], -1)


# the grid reaches 0.8 m past the walls: a frame integrates samples up to trunc behind the surface along its optical
# axis, up to trunc / cos(a) behind it along the wall's normal for a ray at angle a off the axis, so only beyond that
# band -- a at most the camera's half-diagonal field angle -- is space unknown
BOUNDS = np.concatenate([CENTRE - HALF - 0.8, CENTRE + HALF + 0.8])
HALF_DIAGONAL = math.atan(math.hypot(CAM["cx"] + 0.5, CAM["cy"] + 0.5) / CAM["fx"])


@pytest.fixture(scope="module")
def room_maps(cuda_device, room_record):
    return {uio: nav_record(room_record, VOXEL, sil_thres=SIL, batch=5, bounds=BOUNDS, unknown_is_obstacle=uio,
                            device=cuda_device)
            for uio in (True, False)}


def test_room_labels_and_obstacle_rule(room_maps):
    nm, info = room_maps[True]
    assert info["frames"] == 10 and info["voxels"] == np.prod(info["dims"])
    lab = nm.labels.cpu().numpy()
    esdf = nm.esdf.cpu().numpy()
    gaps = _wall_gaps(_sample_coords(nm))
    deep = gaps.min(-1) >= 3 * VOXEL
    assert deep.sum() > 100_000 and (lab[deep] == 1).mean() >= 0.99, np.bincount(lab[deep], minlength=3)
    outside = gaps.min(-1) < -(info["trunc"] / math.cos(HALF_DIAGONAL) + VOXEL)
    assert outside.sum() > 100_000 and (lab[outside] == 0).all()
    assert (esdf[outside] <= 0).all()
    assert (lab == 2).sum() > 10_000
    assert len(info["clearance"]) == 10 and min(info["clearance"]) > 1.0
    nm_free = room_maps[False][0]
    assert torch.equal(nm.labels, nm_free.labels)                # the obstacle rule changes no label
    assert (nm_free.esdf.cpu().numpy()[outside] > 0).all()       # unknown space is no obstacle there


def _interior_points(n=20000):
    """Points at least 3 voxels from every wall whose nearest wall is at least 2 voxels nearer than the second, with
    their six wall distances."""
    g = np.random.default_rng(0)
    p = CENTRE + g.uniform(-1, 1, (n, 3)) * (HALF - 3 * VOXEL)
    gaps = _wall_gaps(p)
    order = np.sort(gaps, -1)
    keep = (order[:, 0] >= 3 * VOXEL) & (order[:, 1] - order[:, 0] >= 2 * VOXEL)
    assert keep.sum() > 5000
    return p[keep], gaps[keep]


def _distance_and_angle(nm, p, gaps, dev):
    """|dist - distance to the nearest wall| and the angle (degrees) between the gradient and the wall's inward
    normal."""
    d, grad = nm.distance(torch.from_numpy(p.astype(np.float32)).to(dev))
    d, grad = d.cpu().numpy().astype(np.float64), grad.cpu().numpy().astype(np.float64)
    wall = gaps.argmin(-1)
    away = np.zeros_like(p)
    away[np.arange(len(p)), wall % 3] = np.where(wall < 3, -1.0, 1.0)   # from the +axis wall inwards is -axis
    cos = (grad * away).sum(-1) / np.linalg.norm(grad, axis=-1)
    return np.abs(d - gaps.min(-1)), np.degrees(np.arccos(np.clip(cos, -1, 1)))


def test_room_distance_against_the_walls(cuda_device, room_maps):
    p, gaps = _interior_points()
    err, _ = _distance_and_angle(room_maps[False][0], p, gaps, cuda_device)
    assert err.max() <= 1.5 * VOXEL, err.max()


def _box_depth(w2c, cam):
    """Depth [H,W] of the room's inside seen by a camera w2c [4,4]: the exit of each pixel's ray from the box."""
    c2w = np.linalg.inv(np.asarray(w2c, np.float64))
    u, v = np.meshgrid(np.arange(cam["w"]), np.arange(cam["h"]))
    rays = np.stack([(u - cam["cx"]) / cam["fx"], (v - cam["cy"]) / cam["fy"], np.ones(u.shape)], -1) @ c2w[:3, :3].T
    o = c2w[:3, 3]
    with np.errstate(divide="ignore"):
        exit_lo, exit_hi = (CENTRE - HALF - o) / rays, (CENTRE + HALF - o) / rays
    return np.where(rays > 0, exit_hi, exit_lo).min(-1).astype(np.float32)


def test_room_gradient_from_exact_depth(cuda_device, room_record):
    """The distance and its gradient against the walls, on depth frames of the exact box at the record's poses.  (The
    splat map's rendered depth puts the occupied layer one voxel in front of the wall in places, at grazing views; the
    distance to such a stepped layer is still within the bound above, but its gradient tilts near the steps.)"""
    rf = RecordFusion(room_record, device=cuda_device)
    frames = [dict(im=torch.zeros(3, CAM["h"], CAM["w"], device=cuda_device),
                   depth=torch.from_numpy(_box_depth(w2c, CAM))[None].to(cuda_device)) for w2c in rf.w2cs.cpu().numpy()]
    nm, _ = nav_record(room_record, VOXEL, bounds=BOUNDS, unknown_is_obstacle=False, device=cuda_device,
                       source=frames)
    p, gaps = _interior_points()
    err, ang = _distance_and_angle(nm, p, gaps, cuda_device)
    assert err.max() <= 1.5 * VOXEL, err.max()
    assert ang.max() <= 10.0, (ang.max(), p[ang.argmax()], gaps[ang.argmax()])


def test_nav_map_tool_end_to_end(cuda_device, room_record, room_maps, tmp_path, capsys):
    tool = load("tools/nav_map.py")
    out = str(tmp_path / "navmap.npz")
    tool.main(["--record", room_record, "--out", out, "--voxel", str(VOXEL), "--batch", "5", "--sil-thres", str(SIL),
               "--bounds"] +
              [str(b) for b in BOUNDS])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    for k in ("dims", "voxels", "frames", "free", "occupied", "unknown", "clearance_min", "clearance_median",
              "render_ms", "integrate_ms", "labels_ms", "esdf_ms", "wall_s"):
        assert k in line, k
    assert line["free"] + line["occupied"] + line["unknown"] == line["voxels"] and line["frames"] == 10
    assert 1.0 < line["clearance_min"] <= HALF.min() and line["clearance_median"] <= HALF.min() + VOXEL
    raw = formats.load_nav_map(out)
    nm = NavMap.load(out, cuda_device)
    assert np.array_equal(nm.labels.cpu().numpy(), raw["labels"])
    assert np.array_equal(_bits(nm.esdf.cpu().numpy()), _bits(raw["esdf"]))
    ref = room_maps[True][0]
    assert np.array_equal(raw["labels"], ref.labels.cpu().numpy())
    assert np.array_equal(_bits(raw["esdf"]), _bits(ref.esdf.cpu().numpy()))
    assert nm.unknown_is_obstacle and nm.occ_dist == np.float32(VOXEL / 2)


def test_nav_record_from_input_frames(cuda_device, room_record, room_maps):
    """--source input: the renders given back as depth/colour frames give the same labels."""
    rf = RecordFusion(room_record, sil_thres=SIL, device=cuda_device)
    frames = []
    for k in range(len(rf.ids)):
        rf._frame_into(0, k)
        frames.append(dict(im=rf.rgb_b[0].clone(), depth=rf.depth_b[0][None].clone()))
    nm, info = nav_record(room_record, VOXEL, sil_thres=SIL, batch=5, bounds=BOUNDS, device=cuda_device,
                          source=frames)
    assert torch.equal(nm.labels, room_maps[True][0].labels)
    assert math.isclose(min(info["clearance"]), min(room_maps[True][1]["clearance"]))
