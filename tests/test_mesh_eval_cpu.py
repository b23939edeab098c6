"""CPU suite of mesh evaluation (splatam_b200/mesh_eval.py): the brute-force restatement of the nearest-neighbour
kernel against scipy's KD-tree, the metric definitions on hand-built cases, load_mesh_ply on the PLY layouts of
ground-truth meshes, world_to_map on the synthetic sequences of every reader, eval_mesh.py's argument checks and the
library's refusal to run without a GPU."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from util import GOLDEN, load
from oracle import mesh_eval_numpy as O
from splatam_b200 import _lib, datasets as D, formats, mesh_eval as E


# ---- the brute-force restatement and the metric ------------------------------------------------------------------

def test_brute_force_matches_a_kd_tree():
    g = np.random.default_rng(0)
    refs = g.uniform(-2, 3, (20_000, 3)).astype(np.float32)
    refs[1000:1500] = refs[:500]                                    # duplicates
    q = np.concatenate([g.uniform(-3, 4, (3000, 3)), refs[:200], refs[200:400] + 1e-4]).astype(np.float32)
    d2 = O.min_sq_dist(q, refs, chunk=512)
    ref, _ = cKDTree(refs.astype(np.float64)).query(q.astype(np.float64))
    assert d2.dtype == np.float32
    assert np.all(d2[3000:3200] == 0)
    np.testing.assert_allclose(np.sqrt(d2.astype(np.float64)), ref, rtol=1e-6, atol=1e-7)


def _plane(n, seed, lo=(0.0, 0.0), hi=(1.0, 1.0)):
    v = np.array([[lo[0], lo[1], 0], [hi[0], lo[1], 0], [hi[0], hi[1], 0], [lo[0], hi[1], 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    p, _ = E.sample_surface(v, f, n, torch.Generator().manual_seed(seed), device="cpu")
    return p.numpy()


def test_parallel_planes_three_centimetres_apart():
    gt = _plane(3000, 1)
    pred = gt + np.float32([0, 0, 0.03])
    acc, comp = O.min_sq_dist(pred, gt), O.min_sq_dist(gt, pred)
    s = E.scores(acc, comp, threshold=0.05)
    assert abs(s["accuracy"] - 0.03) < 1e-6 and abs(s["completion"] - 0.03) < 1e-6
    assert s["precision"] == s["recall"] == s["fscore"] == 1.0
    s = E.scores(acc, comp, threshold=0.02)
    assert s["precision"] == s["recall"] == s["fscore"] == 0.0


def test_half_coverage_gives_half_recall_and_full_precision():
    gt = _plane(4000, 2)
    pred = gt[gt[:, 0] < 0.5]
    s = E.scores(O.min_sq_dist(pred, gt), O.min_sq_dist(gt, pred), threshold=0.01)
    assert s["precision"] == 1.0 and s["accuracy"] == 0.0
    assert abs(s["recall"] - 0.51) < 0.03
    assert abs(s["fscore"] - 2 * s["recall"] / (1 + s["recall"])) < 1e-12


def test_threshold_is_strict():
    s = E.scores(np.float32([0.25, 0.0]), np.float32([0.25]), threshold=0.5)    # distance exactly 0.5
    assert s["precision"] == 0.5 and s["recall"] == 0.0 and s["fscore"] == 0.0
    s = E.scores(np.float32([0.25, 0.0]), np.float32([0.25]), threshold=np.nextafter(0.5, 1))
    assert s["precision"] == s["recall"] == s["fscore"] == 1.0
    with pytest.raises(ValueError):
        E.scores(np.float32([]), np.float32([1.0]))


def test_area_sampling_on_the_host():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [5, 5, 5]], np.float32)
    f = np.array([[0, 1, 2], [3, 4, 3]])                             # the second face has zero area
    p, fid = E.sample_surface(v, f, 1000, torch.Generator().manual_seed(0), device="cpu")
    assert p.dtype == torch.float32 and torch.all(fid == 0)
    assert torch.all(p[:, 2] == 0) and torch.all(p[:, :2] >= 0) and torch.all(p[:, :2].sum(1) <= 1 + 1e-6)
    for bad in ((v, f[1:]), (v[:0], f[:0]), (v, np.zeros((0, 3), int))):
        with pytest.raises(ValueError):
            E.sample_surface(*bad, 10, device="cpu")


def test_grid_geometry_caps_the_cell_count():
    o, cell, dims = E._grid_geometry([0, 0, 0], [10, 10, 3], 1_000_000)
    assert o.dtype == np.float32 and np.all(dims * cell > [10, 10, 3])
    assert np.prod(dims) <= 4_000_064
    _, cell2, dims2 = E._grid_geometry([0, 0, 0], [10, 10, 3], 1_000_000, cell=1e-4)    # grows until it fits
    assert cell2 > 1e-4 and np.prod(dims2) <= 4_000_064
    _, cell3, dims3 = E._grid_geometry([1, 1, 1], [1, 1, 1], 5)                          # one point, repeated
    assert cell3 == 1.0 and list(dims3) == [1, 1, 1]
    with pytest.raises(ValueError):
        E._grid_geometry([0, 0, 0], [1, 1, 1], 10, cell=-1.0)


# ---- load_mesh_ply ---------------------------------------------------------------------------------------------------

QUADS = np.array([[0, 1, 2, 3], [4, 5, 6, 7]])
VERTS = np.arange(24, dtype=np.float32).reshape(8, 3) / 4
COLS = (np.arange(24).reshape(8, 3) * 10).astype(np.uint8)
FANNED = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])


def _header(fmt, nv, nf, count="uchar", index="uint", name="vertex_index", colours=True):
    lines = ["ply", "format %s 1.0" % fmt, "comment extra properties before and after", "element vertex %d" % nv,
             "property float x", "property float y", "property float z", "property float nx", "property float ny",
             "property float nz"]
    if colours:
        lines += ["property uchar red", "property uchar green", "property uchar blue", "property uchar alpha"]
    lines += ["property double quality", "element face %d" % nf, "property list %s %s %s" % (count, index, name),
              "property int flags", "end_header", ""]
    return "\n".join(lines).encode("ascii")


def _binary(path, polys, count="uchar", index="uint", name="vertex_index", colours=True, fmt="binary_little_endian"):
    e = ">" if fmt == "binary_big_endian" else "<"
    vd = [("x", e + "f4"), ("y", e + "f4"), ("z", e + "f4"), ("nx", e + "f4"), ("ny", e + "f4"), ("nz", e + "f4")]
    if colours:
        vd += [("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1")]
    vert = np.zeros(8, vd + [("quality", e + "f8")])
    for k, a in enumerate("xyz"):
        vert[a] = VERTS[:, k]
    if colours:
        for k, a in enumerate(("red", "green", "blue")):
            vert[a] = COLS[:, k]
    ct = {"uchar": "u1", "int": e + "i4"}[count]
    it = {"uint": e + "u4", "int": e + "i4"}[index]
    body = b""
    for p in polys:
        body += np.array([len(p)], ct).tobytes() + np.array(p, it).tobytes() + np.array([7], e + "i4").tobytes()
    with open(path, "wb") as f:
        f.write(_header(fmt, 8, len(polys), count, index, name, colours) + vert.tobytes() + body)
    return str(path)


def _ascii(path, polys, vertex_rows=None):
    rows = vertex_rows or ["%r %r %r 0 0 1 %d %d %d 255 0.5" % (*map(float, VERTS[i]), *COLS[i]) for i in range(8)]
    faces = ["%d %s 7" % (len(p), " ".join(str(int(x)) for x in p)) for p in polys]
    with open(path, "wb") as f:
        f.write(_header("ascii", 8, len(polys), "uchar", "int", "vertex_indices") + "\n".join(rows + faces).encode()
                + b"\n")
    return str(path)


@pytest.mark.parametrize("count, index, name", [("uchar", "uint", "vertex_index"), ("int", "int", "vertex_indices")])
def test_binary_quads_with_extra_properties(tmp_path, count, index, name):
    v, c, f = formats.load_mesh_ply(_binary(tmp_path / "m.ply", QUADS, count, index, name))
    assert v.dtype == np.float32 and c.dtype == np.uint8 and f.dtype == np.int32
    assert np.array_equal(v, VERTS) and np.array_equal(c, COLS) and np.array_equal(f, FANNED)


def test_ascii_quads_and_missing_colours(tmp_path):
    v, c, f = formats.load_mesh_ply(_ascii(tmp_path / "a.ply", QUADS))
    assert np.array_equal(v, VERTS) and np.array_equal(c, COLS) and np.array_equal(f, FANNED)
    v, c, f = formats.load_mesh_ply(_binary(tmp_path / "n.ply", [[0, 1, 2], [5, 6, 7]], colours=False))
    assert np.array_equal(c, np.zeros((8, 3), np.uint8)) and np.array_equal(f, [[0, 1, 2], [5, 6, 7]])


def test_own_files_read_back_unchanged(tmp_path):
    g = np.random.default_rng(3)
    v = g.normal(size=(50, 3)).astype(np.float32)
    c = g.uniform(0, 1, (50, 3))
    f = g.integers(0, 50, (80, 3))
    lv, lc, lf = formats.load_mesh_ply(formats.save_mesh_ply(str(tmp_path / "own.ply"), v, c, f))
    assert np.array_equal(lv, v) and np.array_equal(lf, f) and np.array_equal(lc, np.rint(c * 255).astype(np.uint8))
    ev, ec, ef = formats.load_mesh_ply(formats.save_mesh_ply(str(tmp_path / "e.ply"), v[:0], c[:0], f[:0]))
    assert ev.shape == (0, 3) and ef.shape == (0, 3)


def test_bad_files_are_rejected_with_their_path(tmp_path):
    mixed = [[0, 1, 2], [4, 5, 6, 7]]
    cases = [(_binary(tmp_path / "mixed.ply", mixed), "mix|truncated"),
             (_binary(tmp_path / "mixed2.ply", mixed[::-1]), "mix|truncated"),
             (_ascii(tmp_path / "mixed.txt.ply", mixed), "mix"),
             (_binary(tmp_path / "big.ply", QUADS, fmt="binary_big_endian"), "big-endian"),
             (_binary(tmp_path / "range.ply", [[0, 1, 8]]), "outside"),
             (_ascii(tmp_path / "neg.ply", [[0, -1, 2]]), "outside")]
    rows = ["%r %r %r 0 0 1 1 2 3 255 0.5" % tuple(map(float, VERTS[i])) for i in range(8)]
    rows[2] = "nan 0 0 0 0 1 1 2 3 255 0.5"
    cases.append((_ascii(tmp_path / "nan.ply", [[0, 1, 2]], rows), "non-finite"))
    for path, what in cases:
        with pytest.raises(ValueError, match="(?s)%s.*(%s)" % (os.path.basename(path), what)):
            formats.load_mesh_ply(path)
    v, _, f = formats.load_mesh_ply(_ascii(tmp_path / "unused_nan.ply", [[0, 1, 3]], rows))     # vertex 2 is unused
    assert np.isnan(v[2, 0]) and np.array_equal(f, [[0, 1, 3]])


# ---- world_to_map --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = load("tests/golden/datasets/make_golden_datasets.py")
    nvs = load("tests/golden/datasets/make_golden_nvs_datasets.py")
    d = str(tmp_path_factory.mktemp("w2m"))
    base.write_sequences(d, dict(np.load(os.path.join(GOLDEN, "datasets", "ref_datasets.npz"))))
    nvs.write_sequences(d, dict(np.load(os.path.join(GOLDEN, "datasets", "ref_nvs_datasets.npz"))))
    cap = dict(np.load(os.path.join(GOLDEN, "capture", "ref_capture.npz")))
    for k, v in cap.items():
        if k.startswith("demo/"):
            p = os.path.join(d, "nerfcapture", k)
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(v.tobytes())
    seqs = dict(base.SEQUENCES, **nvs.SEQUENCES, nerfcapture="demo")
    configs = {k: base.config(k) for k in base.SEQUENCES}
    configs["replicav2"] = nvs.REPLICAV2_CONFIG
    return d, seqs, configs


def _native_c2w(sf, dataset):
    """The dataset's own c2w of every retained frame, read from its files (no reader axis change)."""
    root = sf.root
    names = [os.path.basename(p) for p in sf.color_paths]
    if dataset == "replica":
        rows = open(os.path.join(root, "traj.txt")).read().split("\n")
        return [np.array(rows[int(i)].split(), float).reshape(4, 4) for i in sf.retained_inds]
    if dataset == "replicav2":
        rows = open(os.path.join(root, "imap", "00", "traj_w_c.txt")).read().split("\n")
        return [np.array(rows[int(i)].split(), float).reshape(4, 4) for i in sf.retained_inds]
    if dataset == "scannet":
        return [np.loadtxt(os.path.join(root, "pose", n.replace(".jpg", ".txt"))) for n in names]
    if dataset == "tum":
        poses = D._tum_files(root)[2]
        return [poses[int(i)].double().numpy() for i in sf.retained_inds]
    if dataset == "scannetpp":
        meta = json.load(open(os.path.join(root, "dslr", "nerfstudio", "transforms_undistorted.json")))
        by = {fr["file_path"]: fr for fr in meta["frames"]}
        return [np.array(by[n]["transform_matrix"]) for n in names]
    meta = json.load(open(os.path.join(root, "transforms.json")))
    by = {fr["file_path"]: fr for fr in meta["frames"]}
    return [np.array(by["rgb/" + n]["transform_matrix"]) for n in names]


@pytest.mark.parametrize("dataset, start, stride", [
    ("replica", 0, 1), ("replica", 3, 2), ("tum", 1, 2), ("scannet", 2, 3), ("scannetpp", 0, 1), ("scannetpp", 2, 1),
    ("replicav2", 4, 3), ("nerfcapture", 0, 1), ("nerfcapture", 1, 1)])
def test_world_to_map_takes_native_cameras_to_the_map(roots, dataset, start, stride):
    d, seqs, configs = roots
    sf = D.SequenceFiles(dataset, os.path.join(d, dataset), seqs[dataset], configs.get(dataset), start=start,
                         stride=stride)
    M = sf.world_to_map
    assert M.dtype == np.float64 and M.shape == (4, 4)
    native = _native_c2w(sf, dataset)
    assert np.abs(M @ native[0][:, 3] - [0, 0, 0, 1]).max() < 1e-5       # the first camera is the map's origin
    for k, c2w in enumerate(native):                                      # every camera lands on its map-frame pose
        if np.all(np.isfinite(c2w)):
            assert np.abs((M @ c2w[:, 3])[:3] - sf.poses[k][:3, 3].double().numpy()).max() < 1e-4
    A = np.diag([1.0, -1, -1, 1]) if dataset in ("scannetpp", "nerfcapture") else np.eye(4)
    x = np.array([0.3, -1.2, 2.5, 1.0])
    assert np.allclose(sf._raw_pose0 @ (M @ x), A @ x, atol=1e-9)        # back through raw_pose_0
    other = D.SequenceFiles(dataset, os.path.join(d, dataset), seqs[dataset], configs.get(dataset), start=start,
                            stride=stride + 1)
    assert np.array_equal(other.world_to_map, M)                          # stride does not move the map's frame


def test_world_to_map_refuses_a_non_finite_first_pose(roots):
    d, seqs, configs = roots
    sf = D.SequenceFiles("scannet", os.path.join(d, "scannet"), seqs["scannet"], configs["scannet"], start=5)
    assert sf.poses.shape[0] == 6                                         # the rest of the reader is unchanged
    with pytest.raises(ValueError, match="not finite"):
        sf.world_to_map


# ---- the tool and the library without a GPU -----------------------------------------------------------------------

def test_eval_mesh_argument_errors(tmp_path):
    tool = load("tools/eval_mesh.py")
    mesh = formats.save_mesh_ply(str(tmp_path / "m.ply"), VERTS, np.zeros((8, 3)), FANNED)
    ok = ["--mesh", mesh, "--gt-mesh", mesh]
    data = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0"]
    assert tool.parse_args(ok + ["--no-cull"]).no_cull
    assert tool.parse_args(ok + data).every == 1
    for bad in (["--mesh", mesh, "--gt-mesh", str(tmp_path / "missing.ply"), "--no-cull"],
                ok,                                                       # culling needs the sequence
                ok + ["--no-cull", "--stride", "2"],                      # a selection without a sequence
                ok + ["--dataset", "replica", "--no-cull"],               # partial dataset flags
                ok + data + ["--every", "0"], ok + data + ["--samples", "0"], ok + data + ["--threshold", "0"],
                ok + data + ["--occlusion-eps", "-0.1"], ok + data + ["--threshold", "nan"]):
        with pytest.raises(SystemExit):
            tool.parse_args(bad)


def test_to_map_applies_the_transform_in_float64():
    tool = load("tools/eval_mesh.py")
    M = np.eye(4)
    M[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    M[:3, 3] = [1, 2, 3]
    out = tool.to_map(np.float32([[1, 0, 0], [0, 0, 0]]), M)
    assert out.dtype == np.float32 and np.array_equal(out, [[1, 3, 3], [1, 2, 3]])


def test_no_cpu_fallback():
    p = torch.zeros(4, 3)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.NearestGrid(p)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.visible_mask(p, [], np.eye(3))
    v = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        E.evaluate_mesh((v, [[0, 1, 2]]), (v, [[0, 1, 2]]), device="cpu")


def test_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_nn_grid_workspace_bytes(1000, 10, 10, 10, ctypes.byref(n)) == 0 and n.value >= 4 * 1001 + 16 * 1000
    assert lib.sb_nn_grid_workspace_bytes(0, 10, 10, 10, ctypes.byref(n)) == 1            # no reference points
    assert lib.sb_nn_grid_workspace_bytes(10, 1 << 10, 1 << 10, 1 << 9, ctypes.byref(n)) == 1   # 2^29 cells
    assert lib.sb_nn_grid_workspace_bytes(10, 0, 1, 1, ctypes.byref(n)) == 1
    assert lib.sb_nn_grid_build(0, 1, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, 1, 1 << 20, None) == 1    # empty reference set
    assert lib.sb_nn_grid_build(4, 1, 0.0, 0.0, 0.0, 0.0, 1, 1, 1, 1, 1 << 20, None) == 1    # cell 0
    assert lib.sb_nn_grid_build(4, 1, float("nan"), 0.0, 0.0, 1.0, 1, 1, 1, 1, 1 << 20, None) == 1
    assert lib.sb_nn_grid_build(4, 1, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, 1, 16, None) == 2        # short workspace
    assert lib.sb_nn_query(4, None, 4, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, 1, 1 << 20, 1, None) == 1
    assert lib.sb_nn_query(-1, 1, 4, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, 1, 1 << 20, 1, None) == 1
    assert lib.sb_nn_query(0, None, 4, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, 1, 1 << 20, None, None) == 0   # nothing to do
    assert lib.sb_points_visible(4, 1, 1, 8, 8, None, 1, 1.0, 1.0, 4.0, 4.0, 0.03, 1, None) == 1   # no depth
    assert lib.sb_points_visible(4, 1, 1, 8, 8, 1, 1, 1.0, 1.0, 4.0, 4.0, -0.1, 1, None) == 1      # negative eps
    assert lib.sb_points_visible(4, 1, 1, 0, 8, 1, 1, 1.0, 1.0, 4.0, 4.0, 0.03, 1, None) == 1
    assert lib.sb_points_visible(4, 1, 0, 8, 8, None, None, 1.0, 1.0, 4.0, 4.0, 0.03, 1, None) == 0  # no frames
