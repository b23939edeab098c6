"""CPU: the viewer's colour tables, settings, record loading and camera geometry (splatam_b200/viewer.py) and the
numpy restatement of its kernels (oracle/viewer_numpy.py)."""
import numpy as np
import pytest
import torch

from oracle import viewer_numpy as O
from splatam_b200 import formats
from splatam_b200 import viewer as V


def test_jet_and_cool_follow_the_segment_data():
    # the table's entries at the segment breakpoints' neighbourhood, from the published (x, y0, y1) rows
    x = np.linspace(0, 1, 256)
    for lut, data in ((V.JET_LUT, V.JET_DATA), (V.COOL_LUT, V.COOL_DATA)):
        for c, ch in enumerate(("red", "green", "blue")):
            rows = np.array(data[ch], float)
            assert np.allclose(lut[:, c], np.interp(x, rows[:, 0], rows[:, 1]), atol=1e-12)
    assert V.JET_U8[0].tolist() == [0, 0, 128] and V.JET_U8[255].tolist() == [128, 0, 0]
    assert np.allclose(V.COOL_LUT[:, 0], x) and np.allclose(V.COOL_LUT[:, 1], 1 - x) and (V.COOL_LUT[:, 2] == 1).all()


def test_luts_match_matplotlib():
    mpl = pytest.importorskip("matplotlib")
    for name, lut in (("jet", V.JET_LUT), ("cool", V.COOL_LUT)):
        cm = mpl.colormaps[name]
        assert np.array_equal(cm(np.arange(256))[:, :3], lut)
        for x in (0.0, 0.1, 0.25, 0.5, 0.5 + 1e-12, 0.999, 1.0):
            assert np.array_equal(np.array(cm(x)[:3]), V.COOL_LUT[V.cmap_index(x)] if name == "cool" else
                                  V.JET_LUT[V.cmap_index(x)])


def test_cmap_index_rule():
    assert [V.cmap_index(x) for x in (0.0, 1 / 256, 0.5, 255.5 / 256, 1.0, -0.1, 1.1)] == [0, 1, 128, 255, 255, 0, 255]


@pytest.mark.parametrize("s", [0, -1, 2.5, True, "2", None])
def test_view_scale_must_be_a_positive_integer(s):
    with pytest.raises(ValueError, match="view_scale"):
        V.ViewerConfig(view_scale=s)


def test_config_checks():
    assert V.ViewerConfig(view_scale=3.0).view_scale == 3
    with pytest.raises(ValueError, match="render_mode"):
        V.ViewerConfig(render_mode="normals")
    with pytest.raises(ValueError, match="unknown viz keys: viz_ww"):
        V.ViewerConfig.from_viz(dict(viz_ww=3))
    with pytest.raises(ValueError, match="viz_near"):
        V.ViewerConfig(viz_near=0.0)
    cfg = V.ViewerConfig.from_viz(dict(render_mode="depth", offset_first_viz_cam=True, show_sil=False,
                                       visualize_cams=True, viz_w=600, viz_h=340, viz_near=0.01, viz_far=100.0,
                                       view_scale=2, viz_fps=5, enter_interactive_post_online=True))
    assert cfg.render_mode == "depth"


def _record(tmp_path, T=4, P=50, seed=0, timestep=True, **drop):
    g = torch.Generator().manual_seed(seed)
    gauss = dict(means3D=torch.randn(P, 3, generator=g), rgb_colors=torch.rand(P, 3, generator=g),
                 unnorm_rotations=torch.randn(P, 4, generator=g), logit_opacities=torch.randn(P, 1, generator=g),
                 log_scales=torch.randn(P, 1, generator=g))
    rots = torch.randn(1, 4, T, generator=g)
    trans = torch.randn(1, 3, T, generator=g)
    K = np.array([[300.0, 0, 319.5], [0, 300.0, 239.5], [0, 0, 1]], np.float32)
    ts = torch.sort(torch.randint(0, T, (P,), generator=g).float()).values
    path = formats.save_run_record(str(tmp_path), gauss, rots, trans, ts, K, np.eye(4), 640, 480,
                                   [np.eye(4)] * T, list(range(T)))
    if not timestep or drop:
        raw = dict(np.load(path))
        if not timestep:
            raw.pop("timestep")
        raw.update(drop)
        np.savez(path, **raw)
    return path


def test_load_record_on_the_host(tmp_path):
    path = _record(tmp_path)
    rec = V.load_record(path, "cpu")
    raw = dict(np.load(path))
    assert rec.T == 4 and rec.P == 50 and rec.monotone
    assert rec.counts.tolist() == [int((raw["timestep"] <= t).sum()) for t in range(4)]
    assert rec.scales.shape == (50, 3) and torch.equal(rec.scales[:, 0], rec.scales[:, 2])
    k = rec.k(V.ViewerConfig())
    assert np.allclose(k, raw["intrinsics"] * np.array([[600 / 640], [340 / 480], [1.0]]), rtol=1e-6)
    for t in range(4):
        q = torch.nn.functional.normalize(torch.from_numpy(raw["cam_unnorm_rots"][..., t]))
        assert np.allclose(rec.all_w2cs[t][:3, :3], formats_rot(q), atol=1e-6)
        assert np.array_equal(rec.all_w2cs[t][:3, 3], raw["cam_trans"][0, :, t])
    final = V.view_w2cs(rec, V.ViewerConfig(), online=False)
    assert final.shape == (1, 4, 4) and final[0, 2, 3] == np.float32(0.5)
    assert V.view_w2cs(rec, V.ViewerConfig(offset_first_viz_cam=False), online=False)[0, 2, 3] == 0
    online = V.view_w2cs(rec, V.ViewerConfig(offset_first_viz_cam=False), online=True)
    first = np.eye(4, dtype=np.float32)
    first[2, 3] = 0.5
    assert np.array_equal(online, np.stack([first @ w for w in rec.all_w2cs]))


def formats_rot(q):
    from splatam_b200 import mapping as M
    return M.build_rotation(q).numpy()[0]


def test_load_record_argument_checks(tmp_path):
    with pytest.raises(ValueError, match="intrinsics.*camera="):
        path = str(tmp_path / "ckpt")
        formats.save_checkpoint(path, 3, dict(np.load(_record(tmp_path / "a"))), [0])
        V.load_record(str(tmp_path / "ckpt" / "params3.npz"), "cpu")
    rec = V.load_record(str(tmp_path / "ckpt" / "params3.npz"), "cpu",
                        camera=dict(intrinsics=np.eye(3), w2c=np.eye(4), org_width=640, org_height=480))
    assert rec.timestep is None and rec.T == 4
    with pytest.raises(ValueError, match="timestep"):
        next(V.online_frames(rec, V.ViewerConfig()))
    with pytest.raises(ValueError, match="camera count"):
        V.load_record(_record(tmp_path / "b", cam_trans=np.zeros((1, 3, 3), np.float32)), "cpu")
    with pytest.raises(ValueError, match="rgb_colors has 7 rows"):
        V.load_record(_record(tmp_path / "c", rgb_colors=np.zeros((7, 3), np.float32)), "cpu")
    with pytest.raises(ValueError, match="lacks means3D"):
        raw = dict(np.load(_record(tmp_path / "d")))
        raw.pop("means3D")
        np.savez(str(tmp_path / "d" / "params.npz"), **raw)
        V.load_record(str(tmp_path / "d" / "params.npz"), "cpu")
    # the offline drivers' 13-key record (no keyframe_time_indices) loads
    raw = dict(np.load(_record(tmp_path / "e")))
    raw.pop("keyframe_time_indices")
    np.savez(str(tmp_path / "e" / "params.npz"), **raw)
    assert V.load_record(str(tmp_path / "e" / "params.npz"), "cpu").P == 50


def test_camera_lines(tmp_path):
    rec = V.load_record(_record(tmp_path, T=3), "cpu")
    cfg = V.ViewerConfig()
    fr, fc, tr, tc = V.camera_lines(rec, cfg)
    assert fr.shape == (24, 6) and fc.shape == (24, 3) and tr.shape == (2, 6) and tc.shape == (2, 3)
    assert fc[0].tolist() == [0, 255, 255] and fc[8].tolist() == V.to_u8(V.cool(0.5 / 3)).tolist()
    assert tc[0].tolist() == V.to_u8(V.cool(0.5)).tolist() and tc[1].tolist() == V.to_u8(V.cool(0.75)).tolist()
    # frustum 0: the centre inv(w2c)[:3, 3] and four corners at camera depth 0.045 through k
    c2w = np.linalg.inv(rec.all_w2cs[0].astype(float))
    assert np.allclose(fr[0, :3], c2w[:3, 3])
    k = rec.k(cfg).astype(float)
    corners = fr[:4, 3:]
    cam = (np.linalg.inv(c2w) @ np.c_[corners, np.ones(4)].T).T[:, :3]
    assert np.allclose(cam[:, 2], 0.045)
    px = (k @ cam.T).T
    assert np.allclose(px[:, :2] / px[:, 2:], [[0, 0], [600, 0], [600, 340], [0, 340]], atol=1e-6)
    assert np.allclose(tr[0], np.r_[c2w[:3, 3], np.linalg.inv(rec.all_w2cs[1].astype(float))[:3, 3]], atol=1e-5)
    one = V.load_record(_record(tmp_path / "one", T=1), "cpu")            # one frame: no trajectory, no division
    assert V.camera_lines(one, cfg)[2].shape == (0, 6)


def test_oracle_rules():
    # compose: depth 0 / NaN / >= 15 white, vmax over 0 < d < 15, upsampled blocks
    color = np.full((3, 1, 4), 0.5, np.float32)
    depth = np.array([[0.0, np.nan, 15.0, 3.0]], np.float32)
    out, z = O.compose(color, depth, None, 1, 2, V.JET_U8)
    assert out.shape == (2, 8, 3) and (out[:, :6] == 255).all() and (out[:, 6:] == V.JET_U8[255]).all()
    assert np.isinf(z[0, :4]).all() and z[0, 4] == 15 and z[1, 7] == 3
    out, _ = O.compose(color, depth, None, 0, 1, V.JET_U8)
    assert out[0, 3].tolist() == [128, 128, 128]                      # 0.5 * 255 = 127.5 rounds half to even
    # points: equal depths at one pixel -> lower index
    w2c = np.eye(4, dtype=np.float32)
    means = np.array([[0, 0, 1], [0, 0, 1], [0, 0, 0.5]], np.float32)
    colors = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    out, z = O.points(means[:2], colors[:2], None, 0, w2c, (10, 10, 4.5, 4.5), 10, 10, 1, 0.01, 100)
    assert out[5, 5].tolist() == [255, 0, 0] and z[5, 5] == 1
    out, _ = O.points(means, colors, np.array([0, 0, 2], np.float32), 1, w2c, (10, 10, 4.5, 4.5), 10, 10, 1, 0.01, 100)
    assert out[5, 5].tolist() == [255, 0, 0]                          # the nearer point is filtered by its timestep
    # lines: a horizontal segment covers the pixel centres of its span on one row
    base = np.zeros((10, 10, 3), np.uint8)
    seg = np.array([[-0.25, 0.05, 1, 0.25, 0.05, 1]], np.float32)
    out = O.lines(seg, np.array([[9, 8, 7]], np.uint8), w2c, (10, 10, 4.5, 4.5), 10, 10, 0.01,
                  np.full((10, 10), np.inf, np.float32), base)
    assert (out[5, 2:7] == [9, 8, 7]).all() and out.sum() == 24 * 5
