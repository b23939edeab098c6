"""CPU suite of mesh extraction: the generated marching-cubes table, the numpy restatement of TSDF fusion and marching
cubes (oracle/mesh_numpy.py) on analytic surfaces, the mesh PLY format, TSDFVolume's argument checks and the new
entry points' argument checks (no GPU: every check comes before the first CUDA call)."""
import ctypes

import numpy as np
import pytest
import torch

from util import look_at
from oracle import mesh_numpy as O
from splatam_b200 import _lib, formats, mc_table
from splatam_b200.mesh import TSDFVolume

T = mc_table


def _inside(case, c):
    return bool(case >> c & 1)


def test_generated_header_is_current():
    with open(T.HEADER_PATH) as f:
        assert f.read() == T.header_text(), "csrc/mc_table.h is stale: run python splatam_b200/mc_table.py"


def test_edges_are_in_global_id_order():
    # global id 3 * (s + dx + dy nx + dz nx ny) + axis must increase with the local edge id for any grid >= 2^3
    for nx, ny in ((2, 2), (2, 5), (7, 3)):
        gid = [3 * ((c & 1) + (c >> 1 & 1) * nx + (c >> 2 & 1) * nx * ny) + a for c, a in T.EDGES]
        assert gid == sorted(gid) and len(set(gid)) == 12


def test_every_case_uses_exactly_its_crossed_edges():
    for case in range(256):
        crossed = {e for e, (p, q) in enumerate(T.EDGE_ENDS) if _inside(case, p) != _inside(case, q)}
        used = {e for tri in T.TRIANGLES[case] for e in tri}
        assert used == crossed, case
        assert all(len(set(tri)) == 3 for tri in T.TRIANGLES[case])
    assert T.TRIANGLES[0] == () and T.TRIANGLES[255] == ()


def _boundary(case):
    """Directed triangle edges of one case whose reverse is not in the case: its boundary on the cube's faces."""
    d = [(t[i], t[(i + 1) % 3]) for t in T.TRIANGLES[case] for i in range(3)]
    return {e for e in d if (e[1], e[0]) not in d}


def test_face_boundary_depends_only_on_the_face_signs():
    """For all 256 x 6 (case, face) pairs: the boundary a case leaves on a face, in the face's own edge positions, is a
    function of that face's four corner signs, and the opposite face of a neighbouring cell with the same signs has
    the same segments reversed -- so neighbouring cells agree on every shared face."""
    seen = {}
    for case in range(256):
        bnd = _boundary(case)
        on_faces = set()
        for face in T.FACES:
            fe = T.face_edges(face)
            seg = frozenset((fe.index(a), fe.index(b)) for a, b in bnd if a in fe and b in fe)
            on_faces |= {(fe[a], fe[b]) for a, b in seg}
            signs = tuple(_inside(case, c) for c in T.face_corners(face))
            seen.setdefault((face, signs), set()).add(seg)
        assert on_faces == bnd, case           # every boundary edge lies on a face
    assert len(seen) == 6 * 16
    for (face, signs), segs in seen.items():
        assert len(segs) == 1, (face, signs, segs)
    for a in range(3):
        lo, hi = T.face_edges((a, 0)), T.face_edges((a, 1))
        # edge positions correspond: the side-1 edge is the side-0 edge shifted by one step along `a`
        assert [T.EDGES[e][1] for e in lo] == [T.EDGES[e][1] for e in hi]
        for signs in range(16):
            s = tuple(bool(signs >> i & 1) for i in range(4))
            (seg0,), (seg1,) = seen[((a, 0), s)], seen[((a, 1), s)]
            assert seg1 == frozenset((q, p) for p, q in seg0), (a, s)


def _grid(n):
    g = np.arange(n, dtype=np.float32)
    return np.meshgrid(g, g, g, indexing="ij")


def _mesh(tsdf):
    return O.marching_cubes(tsdf, np.ones_like(tsdf), np.zeros(tsdf.shape + (3,), np.float32), (0, 0, 0), 1.0)


def _topology(v, f):
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    _, und = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    _, dire = np.unique(e, axis=0, return_counts=True)
    chi = len(v) - len(und) + len(f)
    vol = np.einsum("ij,ij->i", v[f[:, 0]].astype(np.float64),
                    np.cross(v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64))).sum() / 6
    return chi, und, dire, vol


def _vertex_manifold(v, f):
    """Every vertex's incident faces form one closed fan (no pinched vertices)."""
    nxt = {}
    for a, b, c in f:
        for p, q, r in ((a, b, c), (b, c, a), (c, a, b)):
            nxt.setdefault(p, {})[q] = r
    for p, m in nxt.items():
        start = next(iter(m))
        q, n = start, 0
        while True:
            q = m[q]
            n += 1
            if q == start:
                break
        if n != len(m):
            return False
    return True


def test_sphere_is_a_closed_oriented_manifold_on_the_surface():
    z, y, x = _grid(24)
    c, r = np.float32(11.3), 7.2
    tsdf = (np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) - r).astype(np.float32)
    v, col, f = _mesh(tsdf)
    chi, und, dire, vol = _topology(v, f)
    assert chi == 2 and set(und) == {2} and set(dire) == {1}
    assert _vertex_manifold(v, f)
    assert vol > 0                                      # outward: triangles face increasing T
    assert abs(vol - 4 / 3 * np.pi * r ** 3) < 0.03 * 4 / 3 * np.pi * r ** 3
    rad = np.linalg.norm(v.astype(np.float64) - 11.3, axis=1)
    assert np.abs(rad - r).max() < 0.1                  # within a tenth of a voxel of the sphere
    assert f.dtype == np.int32 and v.dtype == np.float32


def test_torus_has_euler_characteristic_zero():
    z, y, x = _grid(24)
    c = np.float32(11.3)
    tsdf = (np.sqrt((np.sqrt((x - c) ** 2 + (y - c) ** 2) - 7.0) ** 2 + (z - c) ** 2) - 2.6).astype(np.float32)
    v, _, f = _mesh(tsdf)
    chi, und, dire, vol = _topology(v, f)
    assert chi == 0 and set(und) == {2} and set(dire) == {1} and vol > 0
    assert _vertex_manifold(v, f)


@pytest.mark.parametrize("seed", range(8))
def test_random_fields_give_edge_manifold_meshes(seed):
    g = np.random.default_rng(seed)
    tsdf = g.standard_normal((9, 10, 11)).astype(np.float32) - 0.2 * (seed % 3)
    tsdf[0] = tsdf[-1] = 1
    tsdf[:, 0] = tsdf[:, -1] = 1
    tsdf[:, :, 0] = tsdf[:, :, -1] = 1
    v, _, f = _mesh(tsdf)
    assert len(f) > 0
    _, und, dire, _ = _topology(v, f)
    assert set(und) == {2} and set(dire) == {1}
    assert len(np.unique(f)) == len(v)                  # every vertex is used


def test_vertices_in_edge_order_and_interpolated():
    g = np.random.default_rng(3)
    tsdf = g.standard_normal((5, 6, 7)).astype(np.float32)
    color = g.uniform(0, 1, (5, 6, 7, 3)).astype(np.float32)
    weight = np.ones_like(tsdf)
    weight[2, 3, 4] = 0.5                               # below min_weight: its eight cells are not live
    v, c, f = O.marching_cubes(tsdf, weight, color, (0.5, -1.0, 2.0), 0.25)
    assert len(v) and len(f) and f.max() < len(v)
    # every vertex lies on a grid edge: two of its coordinates are sample coordinates
    on = [np.isin(v[:, a], 0.5 * (a == 0) - 1.0 * (a == 1) + 2.0 * (a == 2) + 0.25 * np.arange(8, dtype=np.float32))
          for a in range(3)]
    assert np.all(np.sum(on, 0) >= 2)


def _ray_depth(w2c, K, H, W, hit):
    """Camera-z depth image [H,W] of the surface `hit(origin, dirs) -> ray parameter` (dirs have camera z = 1)."""
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d_cam = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)
    R, t = w2c[:3, :3], w2c[:3, 3]
    d_world = d_cam @ R                                  # R^T d per pixel
    o = -R.T @ t
    return np.nan_to_num(hit(o, d_world), nan=0.0).astype(np.float32)


@pytest.mark.parametrize("shape", ["plane", "sphere"])
def test_oracle_tsdf_of_analytic_depth_meshes_the_surface(shape):
    H, W = 120, 160
    K = np.array([[150.0, 0, 79.5], [0, 150.0, 59.5], [0, 0, 1]])
    voxel = 0.05
    centre, r = np.array([0.0, 0.0, 2.0]), 0.6
    if shape == "plane":
        hit = lambda o, d: np.where(np.abs(d[..., 2]) > 1e-9, (2.0 - o[2]) / d[..., 2], np.nan)
        cams = [np.array(p) for p in ((0.0, 0.0, 0.0), (0.3, -0.2, 0.1), (-0.4, 0.1, 0.3), (0.1, 0.3, -0.2))]
        target = lambda cam: np.array([cam[0] * 0.5, cam[1] * 0.5, 2.0])
        lo, hi = np.array([-0.6, -0.45, 1.6]), np.array([0.6, 0.45, 2.4])
    else:
        def hit(o, d):
            oc = o - centre
            a = np.sum(d * d, -1)
            b = 2 * np.sum(d * oc, -1)
            cc = oc @ oc - r * r
            disc = b * b - 4 * a * cc
            return np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.nan)
        cams = [centre + 1.8 * np.array(p) / np.linalg.norm(p)
                for p in ((0, 0, -1), (1, 0.2, -1), (-1, -0.3, -0.8), (0.2, 1, -0.6), (0.3, -1, -0.4), (1, 0.1, 0.2),
                          (-1, 0.2, 0.3), (0.1, 0.2, 1), (0.2, 1, 0.7), (-0.3, -1, 0.5))]
        target = lambda cam: centre
        lo, hi = centre - 0.8, centre + 0.8
    origin = (np.floor(lo / voxel) * voxel).astype(np.float32)
    dims = (np.floor((hi - origin) / voxel) + 1).astype(int)
    tsdf = np.ones(dims[::-1], np.float32)
    weight = np.zeros_like(tsdf)
    color = np.zeros(tuple(dims[::-1]) + (3,), np.float32)
    for cam in cams:
        w2c = look_at(cam, target(cam))
        depth = _ray_depth(w2c, K, H, W, hit)
        rgb = np.full((3, H, W), 0.5, np.float32)
        O.integrate(tsdf, weight, color, origin, voxel, 4 * voxel, depth, rgb, w2c, K)
    v, c, f = O.marching_cubes(tsdf, weight, color, origin, voxel)
    assert len(f) > 100
    p = v.astype(np.float64)
    err = np.abs(p[:, 2] - 2.0) if shape == "plane" else np.abs(np.linalg.norm(p - centre, axis=1) - r)
    # the projective distance along a ray is not the distance to a curved surface, so where views seen at grazing
    # angles are averaged in the zero crossing drifts; nine vertices in ten are within half a voxel
    assert np.median(err) < 0.15 * voxel and np.percentile(err, 90) < 0.5 * voxel and err.max() < 1.1 * voxel, \
        (np.median(err), np.percentile(err, 90), err.max())
    assert np.allclose(c, 0.5)


def test_mesh_ply_header_and_round_trip(tmp_path):
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    c = np.array([[0, 0.5, 1], [-1, 2, np.nan], [0.2, 0.4, 0.6], [1 / 510, 3 / 510, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    path = formats.save_mesh_ply(str(tmp_path / "m.ply"), v, c, f)
    blob = open(path, "rb").read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float x\nproperty float y\n"
              b"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nelement face 4\n"
              b"property list uchar int vertex_indices\nend_header\n")
    assert blob.startswith(header)
    assert len(blob) == len(header) + 4 * 15 + 4 * 13
    assert blob[len(header) + 4 * 15:len(header) + 4 * 15 + 13] == b"\x03" + np.array([0, 2, 1], "<i4").tobytes()
    v2, c2, f2 = formats.load_mesh_ply(path)
    assert np.array_equal(v2, v) and np.array_equal(f2, f)
    expect = np.rint(np.clip(np.nan_to_num(c.astype(np.float64)), 0, 1) * 255).astype(np.uint8)
    assert np.array_equal(c2, expect)
    assert c2[1].tolist() == [0, 255, 0] and c2[0].tolist() == [0, 128, 255]   # rint: 127.5 -> 128
    e = formats.save_mesh_ply(str(tmp_path / "e.ply"), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3), int))
    v3, c3, f3 = formats.load_mesh_ply(e)
    assert v3.shape == (0, 3) and c3.shape == (0, 3) and f3.shape == (0, 3)
    with pytest.raises(ValueError, match="face indices"):
        formats.save_mesh_ply(str(tmp_path / "b.ply"), v, c, f + 1)


def test_tsdf_volume_argument_errors():
    with pytest.raises(ValueError, match=r"needs 1030301 voxels .* voxel size of"):
        TSDFVolume((0, 0, 0, 1, 1, 1), 0.01, device="cpu", max_voxels=1_000_000)
    try:
        TSDFVolume((0, 0, 0, 1, 1, 1), 0.01, device="cpu", max_voxels=1_000_000)
    except ValueError as e:
        fit = float(str(e).split("voxel size of ")[1].split()[0])
        v = TSDFVolume((0, 0, 0, 1, 1, 1), fit, device="cpu", max_voxels=1_000_000)
        assert v.num_voxels <= 1_000_000
    with pytest.raises(ValueError, match="bounds"):
        TSDFVolume((0, 0, 0, 1, 1), 0.1, device="cpu")
    with pytest.raises(ValueError, match="bounds"):
        TSDFVolume((0, 0, 0, 1, -1, 1), 0.1, device="cpu")
    with pytest.raises(ValueError, match="voxel_size"):
        TSDFVolume((0, 0, 0, 1, 1, 1), 0.0, device="cpu")
    with pytest.raises(ValueError, match="trunc"):
        TSDFVolume((0, 0, 0, 1, 1, 1), 0.1, trunc=-1, device="cpu")
    v = TSDFVolume((-0.33, 0.05, 1.0, 0.4, 0.5, 1.2), 0.1, device="cpu")
    assert np.allclose(v.origin, [-0.4, 0.0, 1.0]) and (v.nx, v.ny, v.nz) == (9, 6, 3)
    assert v.trunc == np.float32(0.4)
    assert float(v.tsdf.min()) == 1.0 and float(v.weight.max()) == 0.0 and tuple(v.color.shape) == (3, 6, 9, 3)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        v.integrate(torch.zeros(4, 4), torch.zeros(3, 4, 4), np.eye(3), torch.eye(4))


def test_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.load()
    inf = float("inf")
    ok = dict(nx=4, ny=4, nz=4, o=(0.0, 0.0, 0.0), v=0.1, tr=0.4, B=1, H=8, W=8, k=(10.0, 10.0, 4.0, 4.0), dmax=inf)

    def integ(**kw):
        a = dict(ok, **kw)
        return lib.sb_tsdf_integrate(a["nx"], a["ny"], a["nz"], *a["o"], a["v"], a["tr"], a["B"], a["H"], a["W"],
                                     a.get("depth", 1), a.get("rgb", 1), a.get("w2c", 1), *a["k"], a["dmax"],
                                     a.get("tsdf", 1), a.get("weight", 1), a.get("color", 1), None)

    assert integ(nx=0) == 1 and integ(ny=-1) == 1 and integ(nx=2048, ny=2048, nz=512) == 1
    assert integ(v=0.0) == 1 and integ(v=float("nan")) == 1 and integ(tr=0.0) == 1 and integ(tr=inf) == 1
    assert integ(o=(0.0, float("nan"), 0.0)) == 1 and integ(B=-1) == 1 and integ(H=0) == 1
    assert integ(k=(inf, 10.0, 4.0, 4.0)) == 1 and integ(dmax=0.0) == 1 and integ(dmax=float("nan")) == 1
    assert integ(depth=None) == 1 and integ(rgb=None) == 1 and integ(w2c=None) == 1 and integ(tsdf=None) == 1
    assert integ(weight=None) == 1 and integ(color=None) == 1
    assert integ(B=0, depth=None, rgb=None, w2c=None) == 0           # no frames: nothing to do
    n = ctypes.c_size_t(0)
    assert lib.sb_mc_workspace_bytes(4, 5, 6, ctypes.byref(n)) == 0 and n.value >= 8 * 121 + 120
    assert lib.sb_mc_workspace_bytes(0, 5, 6, ctypes.byref(n)) == 1
    assert lib.sb_mc_workspace_bytes(1200, 1200, 1200, ctypes.byref(n)) == 1
    assert lib.sb_mc_workspace_bytes(4, 5, 6, None) == 1
    lib.sb_mc_workspace_bytes(4, 4, 4, ctypes.byref(n))
    need = n.value
    assert lib.sb_mc_count(4, 4, 4, None, 1, 1.0, 1, need, 1, None) == 1
    assert lib.sb_mc_count(4, 4, 4, 1, 1, float("nan"), 1, need, 1, None) == 1
    assert lib.sb_mc_count(4, 4, 4, 1, 1, 1.0, 1, need, None, None) == 1
    assert lib.sb_mc_count(4, 4, 4, 1, 1, 1.0, 1, need - 1, 1, None) == 2         # SB_ERR_WORKSPACE
    assert lib.sb_mc_emit(4, 4, 4, 0.0, 0.0, 0.0, 0.0, 1, 1, 1, need, 1, 1, 1, None) == 1
    assert lib.sb_mc_emit(4, 4, 4, 0.0, 0.0, 0.0, 0.1, 1, None, 1, need, 1, 1, 1, None) == 1
    assert lib.sb_mc_emit(4, 4, 4, 0.0, 0.0, 0.0, 0.1, 1, 1, 1, need - 1, 1, 1, 1, None) == 2
