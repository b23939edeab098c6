"""CPU: splatam_b200/viewer.py against the reference's unmodified viewers, through tests/golden/viewer/ref_viewer.npz
(make_golden_viewer.py runs final_recon's and online_recon's `visualize` on two seeded records, one with a
non-monotone timestep).  Loading, cameras, per-frame selection and camera-line colours are compared exactly; the
picture rules are checked against rgbd2pcd's back-projected points and its depth-mode mask."""
import os

import numpy as np
import pytest
import torch

from splatam_b200 import viewer as V

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "viewer", "ref_viewer.npz")
RUNS = {  # name: (online, record, viz overrides), as make_golden_viewer.RUNS
    "final_color": (False, "mono", dict()),
    "final_depth_nooffset": (False, "mono", dict(render_mode="depth", offset_first_viz_cam=False)),
    "online_color": (True, "mono", dict()),
    "online_depth": (True, "mono", dict(render_mode="depth")),
    "online_centers_shuffled": (True, "shuffled", dict(render_mode="centers")),
    "online_color_shuffled": (True, "shuffled", dict()),
}
VIZ = dict(viz_w=48, viz_h=32, viz_near=0.01, viz_far=100.0, view_scale=2, viz_fps=1)


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLD) as z:
        return {k: z[k] for k in z.files}


def _load(gold, record, tmp_path):
    pre = "record_%s_" % record
    path = str(tmp_path / (record + ".npz"))
    np.savez(path, **{k[len(pre):]: v for k, v in gold.items() if k.startswith(pre)})
    return V.load_record(path, "cpu")


def _run(gold, name):
    return {k[len(name) + 1:]: v for k, v in gold.items() if k.startswith(name + "_")}


@pytest.mark.parametrize("name", list(RUNS))
def test_loading_cameras_and_selection_match_the_reference(gold, tmp_path, name):
    online, record, over = RUNS[name]
    ref = _run(gold, name)
    rec = _load(gold, record, tmp_path)
    cfg = V.ViewerConfig.from_viz(dict(VIZ, **over))
    assert rec.monotone == (record == "mono")
    assert np.array_equal(rec.k(cfg), ref["k"])
    assert np.array_equal(rec.all_w2cs, ref["all_w2cs"])
    assert np.array_equal(V.view_w2cs(rec, cfg, online), ref["view_w2c"])
    mine = dict(sel_means3D=rec.means3D, sel_colors_precomp=rec.colors, sel_rotations=rec.rotations,
                sel_opacities=rec.opacities, sel_scales=rec.scales)
    counts = ref["frame_counts"]
    starts = np.concatenate([[0], np.cumsum(counts)])
    for f in range(len(counts)):
        sel = V.select_mask(rec, f) if online else torch.ones(rec.P, dtype=torch.bool)
        for k, v in mine.items():
            assert np.array_equal(v[sel].numpy(), ref[k][starts[f]:starts[f + 1]]), (k, f)
        if online and rec.monotone:
            assert rec.counts[f] == counts[f] and bool(sel[:counts[f]].all())


@pytest.mark.parametrize("name", list(RUNS))
def test_frustums_and_trajectory_match_the_reference(gold, tmp_path, name):
    online, record, over = RUNS[name]
    ref = _run(gold, name)
    rec = _load(gold, record, tmp_path)
    cfg = V.ViewerConfig.from_viz(dict(VIZ, **over))
    fr, fc, tr, tc = V.camera_lines(rec, cfg)
    T = rec.T
    # create_camera_visualization(w, h, k, all_w2cs[t], 0.045) for every frame t, painted cool(x_t)
    assert np.array_equal(ref["frustum_w2c"], rec.all_w2cs)
    assert all(np.array_equal(k, rec.k(cfg)) for k in ref["frustum_k"])
    assert (ref["frustum_whs"] == [cfg.viz_w, cfg.viz_h, V.FRUSTUM_SIZE]).all()
    cool_u8 = lambda xs: V.to_u8(np.stack([V.COOL_LUT[V.cmap_index(x)] for x in xs]))
    assert np.array_equal(fc[::8], cool_u8(ref["frustum_cmap_x"]))
    # the trajectory: lines (i, i - 1) through the camera centres, segment i painted cool(x_i)
    pts, lines = ref["traj_points"], ref["traj_lines"]
    assert np.array_equal(lines, np.stack([np.arange(1, T), np.arange(T - 1)], 1))
    assert np.array_equal(tr, np.concatenate([pts[:-1], pts[1:]], 1).astype(tr.dtype))
    assert np.array_equal(tc, cool_u8(ref["traj_cmap_x"]))
    if online:
        # frame t (t >= 1) draws the first t segments, coloured as in the final view
        assert ref["traj_counts_per_frame"].tolist() == list(range(1, T))
        xs = ref["traj_cmap_x_per_frame"]
        o = 0
        for t in range(1, T):
            assert np.array_equal(cool_u8(xs[o:o + t]), tc[:t])
            o += t


@pytest.mark.parametrize("name", [n for n in RUNS if "centers" not in n])
def test_picture_rules_against_rgbd2pcd(gold, tmp_path, name):
    """rgbd2pcd's point of render pixel (x, y), seen from the same camera at k * view_scale, lands on (s x, s y) at
    camera depth d -- the compose rule; in depth mode its colour mask is d < 15 and Normalize's vmax is the largest
    masked depth."""
    online, record, over = RUNS[name]
    ref = _run(gold, name)
    cfg = V.ViewerConfig.from_viz(dict(VIZ, **over))
    s = cfg.view_scale
    for depth, pts, cols, w2c, k, vmax in zip(ref["pcd_depth"], ref["pcd_points"], ref["pcd_cols"], ref["pcd_w2c"],
                                              ref["pcd_k"], ref["pcd_vmax"]):
        h, w = depth.shape
        cam = (w2c @ np.c_[pts, np.ones(len(pts))].T).T[:, :3]
        d = depth.reshape(-1).astype(float)
        fg = d > 0
        assert fg.mean() > 0.3
        assert np.allclose(cam[:, 2], d, rtol=1e-5, atol=1e-6)
        view_k = k * s
        view_k[2, 2] = 1                                     # the display intrinsics, as the viewers set them
        uv = cam[fg] @ view_k.T
        uv = uv[:, :2] / uv[:, 2:]
        yy, xx = np.divmod(np.arange(h * w), w)
        assert np.abs(uv - s * np.c_[xx, yy][fg]).max() < 1e-3
        assert np.allclose(cam[~fg], 0, atol=1e-6)           # depth 0: on the camera centre, not drawn
        if cfg.render_mode == "depth":
            mask = d < V.DEPTH_FAR
            assert np.array_equal(cols[:, 0], 1.0 - mask) and (~mask).any()
            assert vmax == np.float32(depth[depth < V.DEPTH_FAR].max())


def test_jet_table_in_matplotlibs_operation_order():
    """JET_U8 from a second restatement of colors._create_lookup_table (x and the sample positions scaled by N - 1
    before the interpolation), and the entries whose green lands on a .5 tie at 255 scale."""
    N = 256
    xind = (N - 1) * np.linspace(0, 1, N)
    table = []
    for ch in ("red", "green", "blue"):
        a = np.array(V.JET_DATA[ch], float)
        x = a[:, 0] * (N - 1)
        ind = np.searchsorted(x, xind)[1:-1]
        dist = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        table.append(np.clip(np.r_[a[0, 2], dist * (a[ind, 1] - a[ind - 1, 2]) + a[ind - 1, 2], a[-1, 1]], 0, 1))
    table = np.stack(table, -1)
    assert np.array_equal(V.JET_LUT, table)
    assert np.array_equal(V.JET_U8, np.rint(table * 255).astype(np.uint8))
    assert V.JET_U8[35, 1] == 12 and V.JET_U8[94, 1] == 248
