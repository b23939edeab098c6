"""CPU suite of navigation maps: the numpy restatement (oracle/navmap_numpy.py) against scipy's exact Euclidean
distance transform and against hand-checked labels and queries, the navigation-map npz reader, the argument checks
of the CUDA entry points (no device needed: they reject before any launch) and tools/nav_map.py's flags."""
import ctypes

import numpy as np
import pytest
from scipy import ndimage

from util import load
from oracle import navmap_numpy as O
from splatam_b200 import _lib, formats

SHAPES = [(1, 1, 1), (1, 1, 37), (37, 1, 1), (5, 64, 3), (3, 4, 1100)]


def _scipy_sd2(obstacle):
    out = np.round(ndimage.distance_transform_edt(~obstacle) ** 2).astype(np.int64)
    inside = np.round(ndimage.distance_transform_edt(obstacle) ** 2).astype(np.int64)
    return np.where(obstacle, -inside, out)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("density", [0.001, 0.05, 0.5, 0.95])
def test_oracle_sd2_equals_scipy(shape, density):
    g = np.random.default_rng(int(density * 1000) + sum(shape))
    m = g.uniform(size=shape) < density
    sd2 = O.signed_sq_distance(m)
    assert sd2.dtype == np.int32 and sd2.shape == shape
    if m.any() and not m.all():
        assert np.array_equal(sd2, _scipy_sd2(m))
        assert (sd2[m] < 0).all() and (sd2[~m] > 0).all()
    elif not m.any():
        assert (sd2 == O.INT32_MAX).all()
    else:
        assert (sd2 == -O.INT32_MAX).all()


def test_single_obstacle_gives_the_analytic_distances():
    m = np.zeros((7, 9, 11), bool)
    m[2, 5, 3] = True
    k, j, i = np.meshgrid(np.arange(7), np.arange(9), np.arange(11), indexing="ij")
    want = (k - 2) ** 2 + (j - 5) ** 2 + (i - 3) ** 2
    want[2, 5, 3] = -1                                          # its nearest free sample is one step away
    assert np.array_equal(O.signed_sq_distance(m), want)
    e = O.esdf_from_sd2(O.signed_sq_distance(m), 0.05)
    assert e[2, 5, 4] == np.float32(0.05) and e[2, 5, 3] == -np.float32(0.05)


def test_empty_and_full_obstacle_sets_give_the_sentinels():
    e = np.zeros((3, 4, 5), bool)
    assert (O.signed_sq_distance(e) == O.INT32_MAX).all()
    assert (O.signed_sq_distance(~e) == -O.INT32_MAX).all()
    assert (O.esdf_from_sd2(O.signed_sq_distance(e), 0.1) == np.inf).all()
    assert (O.esdf_from_sd2(O.signed_sq_distance(~e), 0.1) == -np.inf).all()


def test_labels_at_the_boundary_values():
    trunc, occ = np.float32(0.2), np.float32(0.025)
    t_eq = occ / trunc                                         # T * trunc == occ_dist, if it rounds back exactly
    assert np.float32(t_eq) * trunc == occ
    tsdf = np.array([t_eq, np.nextafter(t_eq, np.float32(1)), -1.0, 1.0, 0.5, t_eq], np.float32)
    weight = np.array([1.0, 1.0, 1.0, 1.0, np.nextafter(np.float32(1), np.float32(0)), 0.0], np.float32)
    lab = O.labels(tsdf.reshape(1, 1, -1), weight.reshape(1, 1, -1), trunc, 1.0, occ).reshape(-1)
    assert lab.tolist() == [2, 1, 2, 1, 0, 0]
    assert O.labels(tsdf[:1].reshape(1, 1, 1), np.float32([[[1.0]]]), trunc, 1.0, occ)[0, 0, 0] == 2   # W == min_weight


def test_obstacle_rule():
    lab = np.array([0, 1, 2], np.uint8)
    assert O.obstacles(lab, True).tolist() == [True, False, True]
    assert O.obstacles(lab, False).tolist() == [False, False, True]


def _smooth_esdf():
    g = np.arange(6, dtype=np.float64)
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    return (0.3 * x * x - 0.2 * y * z + 0.5 * z + 0.1 * x * y * z).astype(np.float32)


def test_query_gradient_matches_central_differences():
    esdf, origin, vox = _smooth_esdf(), np.float32([0.1, -0.2, 0.3]), np.float32(0.05)
    g = np.random.default_rng(0)
    cell = g.integers(0, 5, (200, 3))
    frac = g.uniform(0.2, 0.8, (200, 3))                        # away from the cell faces
    p = (origin + vox * (cell + frac)).astype(np.float32)
    d, grad = O.query(esdf, origin, vox, p)
    h = 1e-3 * vox
    for a in range(3):
        e = np.zeros(3)
        e[a] = h
        dp, _ = O.query(esdf, origin, vox, (p.astype(np.float64) + e).astype(np.float32))
        dm, _ = O.query(esdf, origin, vox, (p.astype(np.float64) - e).astype(np.float32))
        step = ((p.astype(np.float64) + e).astype(np.float32) - (p.astype(np.float64) - e).astype(np.float32))[:, a]
        fd = (dp.astype(np.float64) - dm) / step
        np.testing.assert_allclose(grad[:, a], fd, rtol=2e-2, atol=2e-2 * np.abs(grad).max())


def test_query_bounds_nan_and_infinite_corners():
    esdf, origin, vox = _smooth_esdf(), np.float32([0.0, 0.0, 0.0]), np.float32(0.5)
    last = vox * np.float32(5)
    d, g = O.query(esdf, origin, vox, np.float32([[0, 0, 0], [last, last, last]]))
    assert d[0] == esdf[0, 0, 0] and d[1] == esdf[5, 5, 5] and np.isfinite(g).all()
    below = np.nextafter(np.float32(0), np.float32(-1))
    above = np.nextafter(last, np.float32(10))
    bad = np.float32([[below, 1, 1], [1, above, 1], [1, 1, np.nan], [np.inf, 1, 1], [1, -np.inf, 1]])
    d, g = O.query(esdf, origin, vox, bad)
    assert np.isnan(d).all() and np.isnan(g).all()
    e = esdf.copy()
    e[1, 1, 1] = np.inf
    e[1, 1, 2] = -np.inf
    d, g = O.query(e, origin, vox, np.float32([[0.7, 0.7, 0.7], [1.7, 1.7, 1.7], [1.2, 0.7, 0.7]]))
    assert d[0] == np.inf and d[2] == -np.inf and (g[[0, 2]] == 0).all()     # the first infinite corner, zero gradient
    assert np.isfinite(d[1]) and np.isfinite(g[1]).all()
    with pytest.raises(ValueError, match="dimension >= 2"):
        O.query(np.zeros((1, 4, 4), np.float32), origin, vox, np.zeros((1, 3), np.float32))


# ---- formats ---------------------------------------------------------------------------------------------------------

def _map():
    g = np.random.default_rng(1)
    lab = g.integers(0, 3, (4, 5, 6)).astype(np.uint8)
    esdf = g.normal(size=(4, 5, 6)).astype(np.float32)
    esdf[0, 0, 0] = np.inf
    return dict(labels=lab, esdf=esdf, origin=np.float32([0.1, 0.2, -0.3]), voxel_size=0.05, trunc=0.2,
                min_weight=1.0, occ_dist=0.025, unknown_is_obstacle=False)


def test_nav_map_round_trip(tmp_path):
    m = _map()
    path = formats.save_nav_map(str(tmp_path / "sub" / "nav.npz"), **m)
    d = formats.load_nav_map(path)
    assert np.array_equal(d["labels"], m["labels"]) and d["labels"].dtype == np.uint8
    assert np.array_equal(d["esdf"].view(np.uint32), m["esdf"].view(np.uint32))
    assert np.array_equal(d["origin"], m["origin"]) and d["voxel_size"] == np.float32(0.05)
    assert d["trunc"] == np.float32(0.2) and d["min_weight"] == 1 and d["occ_dist"] == np.float32(0.025)
    assert d["unknown_is_obstacle"] == False  # noqa: E712


def _write(path, **over):
    m = _map()
    formats.save_nav_map(path, **m)
    with np.load(path) as z:
        d = {k: z[k] for k in z.files}
    for k, v in over.items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    np.savez(path, **d)
    return path


@pytest.mark.parametrize("key,value", [
    ("labels", None), ("esdf", None), ("origin", None), ("voxel_size", None), ("trunc", None), ("min_weight", None),
    ("occ_dist", None), ("unknown_is_obstacle", None),
    ("labels", np.zeros((4, 5, 6), np.int32)), ("labels", np.zeros((4, 30), np.uint8)),
    ("labels", np.full((4, 5, 6), 3, np.uint8)),
    ("esdf", np.zeros((4, 5, 6), np.float64)), ("esdf", np.zeros((4, 5, 7), np.float32)),
    ("origin", np.float32([0, np.nan, 0])), ("origin", np.float32([0, 0])), ("origin", np.float64([0, 0, 0])),
    ("voxel_size", np.float32(0)), ("voxel_size", np.float32(-0.1)), ("voxel_size", np.float32(np.inf)),
    ("voxel_size", np.float32([0.05])), ("trunc", np.float32(0)), ("min_weight", np.float32(np.nan)),
    ("occ_dist", np.float32(np.inf)), ("unknown_is_obstacle", np.int64(1)),
])
def test_nav_map_reader_rejects(tmp_path, key, value):
    path = _write(str(tmp_path / "nav.npz"), **{key: value})
    with pytest.raises(ValueError, match=key):
        formats.load_nav_map(path)


# ---- ABI argument checks ---------------------------------------------------------------------------------------------

P = 1          # a non-null dummy pointer: every call below returns before it could be dereferenced
BAD = 1        # SB_ERR_BAD_ARG
inf, nan = float("inf"), float("nan")


def test_nav_labels_rejects_bad_arguments():
    lib = _lib.load()
    f = lib.sb_nav_labels
    ok = [4, 4, 4, P, P, 0.2, 1.0, 0.025, P, None]
    for i, v in [(0, 0), (1, -1), (2, 8193), (3, None), (4, None), (8, None), (5, 0.0), (5, -1.0), (5, inf), (5, nan),
                 (6, nan), (6, inf), (7, nan), (7, -inf)]:
        a = list(ok)
        a[i] = v
        assert f(*a) == BAD, (i, v)
    assert f(2048, 1024, 1024, P, P, 0.2, 1.0, 0.025, P, None) == BAD      # 2^31 samples


def test_esdf_rejects_bad_arguments():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_esdf_workspace_bytes(4, 5, 6, ctypes.byref(n)) == 0 and n.value >= 24 * 120
    assert lib.sb_esdf_workspace_bytes(8192, 8192, 31, ctypes.byref(n)) == 0     # just under 2^31 samples
    assert lib.sb_esdf_workspace_bytes(8192, 8192, 32, ctypes.byref(n)) == BAD
    assert lib.sb_esdf_workspace_bytes(8193, 1, 1, ctypes.byref(n)) == BAD
    assert lib.sb_esdf_workspace_bytes(0, 1, 1, ctypes.byref(n)) == BAD
    assert lib.sb_esdf_workspace_bytes(4, 4, 4, None) == BAD
    assert lib.sb_esdf_workspace_bytes(4, 5, 6, ctypes.byref(n)) == 0
    need = n.value
    f = lib.sb_esdf
    ok = [4, 5, 6, P, 0.05, 1, P, need, P, P, None]
    for i, v in [(0, 0), (1, -2), (2, 8193), (3, None), (6, None), (8, None), (9, None), (4, 0.0), (4, -0.05),
                 (4, inf), (4, nan), (5, 2), (5, -1)]:
        a = list(ok)
        a[i] = v
        assert f(*a) == BAD, (i, v)
    assert f(4, 5, 6, P, 0.05, 1, P, need - 1, P, P, None) == 2             # SB_ERR_WORKSPACE


def test_esdf_query_rejects_bad_arguments():
    lib = _lib.load()
    f = lib.sb_esdf_query
    ok = [4, 4, 4, 0.0, 0.0, 0.0, 0.05, P, 10, P, P, P, None]
    for i, v in [(0, 1), (1, 0), (2, 8193), (3, nan), (4, inf), (5, -inf), (6, 0.0), (6, -1.0), (6, nan), (6, inf),
                 (7, None), (8, -1), (9, None), (10, None), (11, None)]:
        a = list(ok)
        a[i] = v
        assert f(*a) == BAD, (i, v)
    assert f(2048, 1024, 1024, 0.0, 0.0, 0.0, 0.05, P, 10, P, P, P, None) == BAD
    assert f(4, 4, 4, 0.0, 0.0, 0.0, 0.05, P, 0, None, None, None, None) == 0   # nothing to query: no launch


# ---- tools/nav_map.py ------------------------------------------------------------------------------------------------

def test_nav_map_tool_rejects_bad_flags(tmp_path):
    tool = load("tools/nav_map.py")
    rec = tmp_path / "params.npz"
    rec.write_bytes(b"")
    base = ["--record", str(rec), "--out", str(tmp_path / "nav.npz")]
    a = tool.parse_args(base + ["--voxel", "0.05", "--unknown", "free", "--occ-dist", "0.01"])
    assert a.unknown == "free" and a.occ_dist == 0.01 and a.voxel == 0.05 and a.source == "render"
    assert tool.parse_args(base).unknown == "obstacle"
    for extra in (["--unknown", "maybe"], ["--occ-dist", "nan"], ["--occ-dist", "inf"], ["--every", "0"],
                  ["--batch", "0"], ["--source", "input"], ["--stride", "2"], ["--bogus"], ["--unk", "free"]):
        with pytest.raises(SystemExit):
            tool.parse_args(base + extra)
    with pytest.raises(SystemExit):
        tool.parse_args(["--record", str(tmp_path / "missing.npz"), "--out", "x.npz"])
