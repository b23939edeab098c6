"""GPU suite of mesh evaluation: sb_points_visible and sb_nn_query bit for bit against the numpy restatement
(oracle/mesh_eval_numpy.py), the grid search on the clouds where it is easiest to get wrong, area sampling, and
evaluate_mesh / eval_mesh.py end to end on a meshed synthetic run record, with the culling loop free of host
synchronisation."""
import json

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from util import load, look_at
from oracle import mesh_eval_numpy as O
from splatam_b200 import formats
from splatam_b200 import mesh_eval as E
from splatam_b200.mesh import RecordFusion, mesh_record

pytestmark = pytest.mark.gpu
H, W = 32, 40
K = np.array([[40.0, 0, 19.5], [0, 40.0, 15.5], [0, 0, 1]], np.float32)


def _frames(B, seed):
    """Random poses around a 1 m cloud (every third camera inside it, so points lie behind it), depth near the
    points' depth with holes (0), far values and NaN, and one frame with a NaN pose."""
    g = np.random.default_rng(seed)
    w2c, depth = [], []
    for b in range(B):
        r = 0.2 if b % 3 == 0 else g.uniform(1.2, 2.0)
        d = g.normal(size=3)
        w2c.append(look_at(r * d / np.linalg.norm(d), g.uniform(-0.1, 0.1, 3)).astype(np.float32))
        base = r + g.uniform(-0.4, 0.4) + 0.2 * g.standard_normal((H, W))
        base[g.uniform(size=(H, W)) < 0.1] = 0.0
        base[g.uniform(size=(H, W)) < 0.05] = 1e6
        base[g.uniform(size=(H, W)) < 0.02] = np.nan
        base[g.uniform(size=(H, W)) < 0.02] = -1.0
        depth.append(base)
    w2c[B // 2][:] = np.nan
    return np.stack(depth).astype(np.float32), np.stack(w2c)


def _frame_dicts(depth, w2c, dev):
    return [dict(depth=torch.from_numpy(d[None]).to(dev), gt_w2c=torch.from_numpy(m).to(dev)) for d, m in zip(depth, w2c)]


def test_visibility_is_bit_equal_to_the_oracle(cuda_device):
    g = np.random.default_rng(1)
    pts = g.uniform(-0.5, 0.5, (30_000, 3)).astype(np.float32)
    depth, w2c = _frames(13, seed=2)
    frames = _frame_dicts(depth, w2c, cuda_device)
    p = torch.from_numpy(pts).to(cuda_device)
    want = O.points_visible(pts, depth, w2c, K, 0.03)
    assert 0 < want.mean() < 1
    one = [O.points_visible(pts, depth[b:b + 1], w2c[b:b + 1], K, 0.03) for b in range(13)]
    assert sum(0.2 < m.mean() < 0.8 for m in one) >= 3
    for b in range(13):                                                  # single frames, including the NaN pose
        assert np.array_equal(E.visible_mask(p, frames[b:b + 1], K, 0.03).cpu().numpy(), one[b]), b
    for batch in (1, 4, 13, 32):
        got = E.visible_mask(p, frames, K, 0.03, batch=batch)
        assert got.dtype == torch.uint8 and np.array_equal(got.cpu().numpy(), want), batch
    # the NaN pose alone marks nothing; the mask is only ever set
    nan = E.visible_mask(p, frames[13 // 2:13 // 2 + 1], K, 0.03)
    assert int(nan.sum()) == 0
    assert np.array_equal(E.visible_mask(p, frames[5:], K, 0.03, mask=E.visible_mask(p, frames[:5], K, 0.03)).cpu()
                          .numpy(), want)
    assert np.array_equal(E.visible_mask(p, frames, K, 0.0).cpu().numpy(), O.points_visible(pts, depth, w2c, K, 0.0))


def _clouds():
    g = np.random.default_rng(7)
    lattice = np.stack(np.meshgrid(*[np.arange(0, 2.01, 0.25)] * 3, indexing="ij"), -1).reshape(-1, 3)
    centres = g.uniform(-5, 5, (6, 3))
    clustered = (centres[g.integers(0, 6, 6000)] + 0.01 * g.standard_normal((6000, 3)))
    dup = g.uniform(0, 1, (500, 3))
    return {
        "random": (g.uniform(-1, 2, (8000, 3)), g.uniform(-1.5, 2.5, (4000, 3))),
        "boundaries": (lattice, np.concatenate([lattice[::3] + 0.125, lattice[::5], g.uniform(0, 2, (2000, 3))])),
        "duplicates": (np.concatenate([dup, dup, dup[:100]]), np.concatenate([dup[:300], g.uniform(0, 1, (2000, 3))])),
        "single": (np.float64([[0.3, -0.2, 0.7]]), g.uniform(-3, 3, (2000, 3))),
        "far": (g.uniform(0, 1, (3000, 3)), np.concatenate([g.uniform(-1e3, 1e3, (1000, 3)),
                                                           g.uniform(5, 6, (500, 3)) * [1, -1, 1]])),
        "clustered": (clustered, np.concatenate([g.uniform(-6, 6, (3000, 3)), clustered[::7] + 0.003])),
    }


@pytest.mark.parametrize("case", ["random", "boundaries", "duplicates", "single", "far", "clustered"])
def test_nearest_neighbour_is_bit_equal_to_brute_force(cuda_device, case):
    refs, q = (np.asarray(a, np.float32) for a in _clouds()[case])
    want = O.min_sq_dist(q, refs, chunk=128)
    r, qq = torch.from_numpy(refs).to(cuda_device), torch.from_numpy(q).to(cuda_device)
    grid = E.NearestGrid(r)
    got = [grid.query(qq).cpu().numpy()]
    for scale in (0.37, 3.0):
        got.append(E.NearestGrid(r, cell=grid.cell * scale).query(qq).cpu().numpy())
    if case == "boundaries":
        got.append(E.NearestGrid(r, cell=0.25).query(qq).cpu().numpy())     # every point on a cell boundary
    for d2 in got:
        assert d2.dtype == np.float32 and np.array_equal(d2.view(np.uint32), want.view(np.uint32))


def test_nearest_neighbour_at_a_million_points(cuda_device):
    g = np.random.default_rng(11)
    refs = g.uniform(-5, 5, (1_000_000, 3)).astype(np.float32)
    refs[:, 2] = np.sin(refs[:, 0]) + 0.01 * g.standard_normal(len(refs))          # a thin, wavy surface
    q = (refs[g.integers(0, len(refs), 200_000)] + 0.02 * g.standard_normal((200_000, 3))).astype(np.float32)
    d2 = E.NearestGrid(torch.from_numpy(refs).to(cuda_device)).query(torch.from_numpy(q).to(cuda_device)).cpu()
    ref, _ = cKDTree(refs.astype(np.float64)).query(q.astype(np.float64))
    np.testing.assert_allclose(np.sqrt(d2.numpy().astype(np.float64)), ref, rtol=1e-5, atol=1e-7)
    sub = slice(0, 512)
    assert np.array_equal(d2.numpy()[sub], O.min_sq_dist(q[sub], refs, chunk=16))


def test_empty_and_non_finite_reference_sets_are_refused(cuda_device):
    with pytest.raises(ValueError, match="at least one"):
        E.NearestGrid(torch.zeros(0, 3, device=cuda_device))
    with pytest.raises(ValueError, match="finite"):
        E.NearestGrid(torch.tensor([[0.0, float("nan"), 0.0]], device=cuda_device))


def test_area_sampling_on_the_gpu(cuda_device):
    g = np.random.default_rng(5)
    v = g.uniform(-1, 1, (30, 3)).astype(np.float32)
    f = g.integers(0, 30, (12, 3))
    f[3] = [4, 4, 5]                                                   # zero area
    n = 400_000
    p, fid = E.sample_surface(v, f, n, torch.Generator(cuda_device).manual_seed(3), cuda_device)
    p2, fid2 = E.sample_surface(v, f, n, torch.Generator(cuda_device).manual_seed(3), cuda_device)
    assert torch.equal(p, p2) and torch.equal(fid, fid2)
    p, fid = p.cpu().numpy().astype(np.float64), fid.cpu().numpy()
    vd = v.astype(np.float64)
    a, b, c = vd[f[fid, 0]], vd[f[fid, 1]], vd[f[fid, 2]]
    e1, e2, r = b - a, c - a, p - a
    # barycentrics by least squares; the residual is the distance off the face's plane
    G = np.stack([np.einsum("ij,ij->i", e1, e1), np.einsum("ij,ij->i", e1, e2), np.einsum("ij,ij->i", e2, e2)], 1)
    rhs = np.stack([np.einsum("ij,ij->i", e1, r), np.einsum("ij,ij->i", e2, r)], 1)
    det = G[:, 0] * G[:, 2] - G[:, 1] ** 2
    u = (G[:, 2] * rhs[:, 0] - G[:, 1] * rhs[:, 1]) / det
    w = (G[:, 0] * rhs[:, 1] - G[:, 1] * rhs[:, 0]) / det
    off = np.linalg.norm(r - u[:, None] * e1 - w[:, None] * e2, axis=1)
    tol = 1e-5
    assert off.max() < 1e-6 and u.min() > -tol and w.min() > -tol and (u + w).max() < 1 + tol
    area = 0.5 * np.linalg.norm(np.cross(vd[f[:, 1]] - vd[f[:, 0]], vd[f[:, 2]] - vd[f[:, 0]]), axis=1)
    prob = area / area.sum()
    counts = np.bincount(fid, minlength=len(f))
    assert counts[3] == 0
    assert np.all(np.abs(counts - n * prob) <= 6 * np.sqrt(n * prob * (1 - prob)) + 1)


# ---- end to end: the wall of Gaussians of test_mesh_gpu.py ---------------------------------------------------------

WALL_Z = 2.0
REC_W, REC_H = 160, 120
REC_K = np.array([[150.0, 0, 79.5], [0, 150.0, 59.5], [0, 0, 1]], np.float32)
VOXEL = 0.02


@pytest.fixture(scope="module")
def wall(tmp_path_factory, cuda_device):
    """A wall of flat Gaussians on z = 2 seen by six cameras (test_mesh_gpu.py's record), its mesh, the frames it was
    meshed from (rendered depth, map-frame w2c) and a ground-truth plane PLY on z = 2, 8 m x 8 m in 2,500 quads."""
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
    d = tmp_path_factory.mktemp("wall_eval")
    record = formats.save_run_record(str(d), gauss, rots, trans, np.zeros(P), REC_K, np.eye(4), REC_W, REC_H,
                                     [np.eye(4)] * T, [0])
    v, c, f, _ = mesh_record(record, VOXEL, device=cuda_device)
    pred = formats.save_mesh_ply(str(d / "mesh.ply"), v, c, f)
    rf = RecordFusion(record, device=cuda_device)
    frames = []
    for k in range(len(rf.ids)):
        rf._frame_into(0, k)
        frames.append(dict(depth=rf.depth_b[0][None].clone(), gt_w2c=rf.w2cs[k].clone()))
    n = 51
    gx, gy = np.meshgrid(np.linspace(-4, 4, n), np.linspace(-4, 4, n))
    gv = np.c_[gx.ravel(), gy.ravel(), np.full(n * n, WALL_Z)].astype(np.float32)
    q = np.arange(n - 1)
    i00 = (q[:, None] * n + q[None, :]).ravel()
    quads = np.stack([i00, i00 + 1, i00 + n + 1, i00 + n], 1)
    gt = str(d / "gt.ply")
    with open(gt, "wb") as fh:
        fh.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                  "property float z\nelement face %d\nproperty list uchar uint vertex_indices\nend_header\n"
                  % (len(gv), len(quads))).encode())
        fh.write(gv.tobytes())
        face = np.zeros(len(quads), [("n", "u1"), ("v", "<u4", (4,))])
        face["n"], face["v"] = 4, quads
        fh.write(face.tobytes())
    return dict(pred=pred, gt=gt, frames=frames, K=rf.K)


def test_wall_scores_with_and_without_culling(cuda_device, wall):
    pred, gt = formats.load_mesh_ply(wall["pred"]), formats.load_mesh_ply(wall["gt"])
    pred, gt = (pred[0], pred[2]), (gt[0], gt[2])
    culled = E.evaluate_mesh(pred, gt, wall["frames"], wall["K"], device=cuda_device)
    assert culled["accuracy"] < VOXEL and culled["completion"] < VOXEL and culled["recall"] > 0.95, culled
    assert culled["precision"] > 0.95 and culled["gt_samples"] == culled["pred_samples"] == 200_000
    assert 0 < culled["gt_samples_kept"] < 200_000 // 4
    assert min(culled["cull_ms"], culled["grid_ms"], culled["query_ms"]) > 0
    whole = E.evaluate_mesh(pred, gt, device=cuda_device)
    assert whole["recall"] < 0.5 and whole["gt_samples_kept"] == 200_000, whole
    assert whole["accuracy"] < culled["accuracy"]                      # denser ground-truth samples
    again = E.evaluate_mesh(pred, gt, wall["frames"], wall["K"], device=cuda_device)
    assert {k: again[k] for k in ("accuracy", "completion", "recall")} == \
        {k: culled[k] for k in ("accuracy", "completion", "recall")}


def test_eval_mesh_tool_prints_the_same_numbers(cuda_device, wall, capsys):
    tool = load("tools/eval_mesh.py")
    tool.main(["--mesh", wall["pred"], "--gt-mesh", wall["gt"], "--no-cull", "--samples", "50000", "--seed", "4"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    pred, gt = formats.load_mesh_ply(wall["pred"]), formats.load_mesh_ply(wall["gt"])
    want = E.evaluate_mesh((pred[0], pred[2]), (gt[0], gt[2]), samples=50_000, seed=4, device=cuda_device)
    assert line["accuracy_cm"] == 100 * want["accuracy"] and line["completion_cm"] == 100 * want["completion"]
    assert line["recall"] == want["recall"] and line["fscore"] == want["fscore"] and not line["culled"]


def test_culling_loop_has_no_host_synchronisation(cuda_device, wall):
    g = torch.Generator(cuda_device).manual_seed(0)
    pts = torch.rand(100_000, 3, device=cuda_device, generator=g) * 4 - 2
    pts[:, 2] = WALL_Z
    want = E.visible_mask(pts, wall["frames"], wall["K"], batch=4)     # warms every shape
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = E.visible_mask(pts, wall["frames"], wall["K"], batch=4)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(got, want) and 0 < int(want.sum()) < len(pts)
