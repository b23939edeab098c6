"""GPU: the headless viewer kernels (csrc/viewer.cu) bit-equal to oracle/viewer_numpy.py on seeded inputs with their
edge cases, and the viewer end to end on a record from a short SLAM run: every frame equals the oracle applied to the
same device renders, the prefix and compaction selections agree, the PNGs decode to the device frames, and the frame
loop enqueues no host synchronisation of its own."""
import os

import numpy as np
import pytest
import torch

from oracle import viewer_numpy as O

pytestmark = pytest.mark.gpu


def _w2c(rx=0.1, ry=-0.2, t=(0.1, -0.05, 0.3)):
    cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
    R = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    m = np.eye(4)
    m[:3, :3], m[:3, 3] = R, t
    return m.astype(np.float32)


def _compose_inputs(g, h, w):
    color = g.uniform(-0.2, 1.2, (3, h, w)).astype(np.float32)
    color[0, 0, :4] = [np.nan, 0.5 / 255, 1.5 / 255, 2.5 / 255]
    depth = g.uniform(0.5, 20.0, (h, w)).astype(np.float32)
    depth.reshape(-1)[:6] = [0.0, np.nan, 15.0, np.nextafter(np.float32(15), np.float32(0)), -1.0, 14.0]
    sil = g.uniform(-0.1, 1.1, (h, w)).astype(np.float32)
    sil[1, 0] = np.nan
    return color, depth, sil


@pytest.mark.parametrize("s", [1, 2, 3])
def test_compose_matches_oracle(cuda_device, s):
    from splatam_b200 import viewer as V
    dev = cuda_device
    g = np.random.default_rng(s)
    h, w = 37, 53
    color, depth, sil = _compose_inputs(g, h, w)
    lut = torch.from_numpy(V.JET_U8.copy()).to(dev)
    cases = [(0, depth), (1, depth), (2, depth),
             (1, np.where(depth < 15, 0, depth).astype(np.float32)),          # vmax == 0: every pixel white
             (1, np.full((h, w), np.nan, np.float32))]
    for mode, d in cases:
        out = torch.empty(h * s, w * s, 3, dtype=torch.uint8, device=dev)
        zbuf = torch.empty(h * s, w * s, dtype=torch.float32, device=dev)
        vmax = torch.empty(1, dtype=torch.int32, device=dev)
        T = lambda a: torch.from_numpy(a).to(dev)
        V.compose(T(color), T(d), T(sil), mode, s, lut, out, zbuf, vmax)
        ro, rz = O.compose(color, d, sil, mode, s, V.JET_U8)
        assert np.array_equal(out.cpu().numpy(), ro), (mode, s)
        assert np.array_equal(zbuf.cpu().numpy(), rz, equal_nan=True), (mode, s)


def test_points_match_oracle(cuda_device):
    from splatam_b200 import viewer as V
    dev = cuda_device
    g = np.random.default_rng(5)
    P, W, H, s = 20000, 160, 96, 2
    w2c = _w2c()
    k = (np.float32(90.0), np.float32(88.0), np.float32(79.5), np.float32(47.5))
    means = np.concatenate([g.uniform(-1.5, 1.5, (P, 2)), g.uniform(-0.5, 4.0, (P, 1))], 1).astype(np.float32)
    colors = g.uniform(-0.1, 1.1, (P, 3)).astype(np.float32)
    ts = g.integers(0, 10, P).astype(np.float32)
    near, far = 0.01, 3.0
    # a point exactly on the near plane and one on the far plane, in front of the camera
    inv = np.linalg.inv(w2c.astype(np.float64))
    means[0] = (inv @ np.array([0.0, 0.0, near, 1.0]))[:3]
    means[1] = (inv @ np.array([0.0, 0.0, far, 1.0]))[:3]
    means[2] = (inv @ np.array([500.0, 0.0, 1.0, 1.0]))[:3]                # far off screen
    means[10:20] = means[30]                                               # equal depths at one pixel
    Td = lambda a: torch.from_numpy(a).to(dev)
    for timestep, t_max in ((None, 0.0), (ts, 4.0)):
        out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev)
        zbuf = torch.empty(H, W, dtype=torch.float32, device=dev)
        keys = torch.empty(H * W, dtype=torch.int64, device=dev)
        V.draw_points(Td(means), Td(colors), None if timestep is None else Td(timestep), t_max, Td(w2c), k, W, H, s,
                      near, far, keys, out, zbuf)
        ro, rz = O.points(means, colors, timestep, t_max, w2c, k, W, H, s, near, far)
        assert np.array_equal(out.cpu().numpy(), ro)
        assert np.array_equal(zbuf.cpu().numpy(), rz)
        assert (rz < np.inf).mean() > 0.2


def test_lines_match_oracle(cuda_device):
    from splatam_b200 import viewer as V
    dev = cuda_device
    g = np.random.default_rng(7)
    W, H = 200, 120
    w2c = _w2c(0.05, 0.1, (0.0, 0.0, 0.5))
    inv = np.linalg.inv(w2c.astype(np.float64))
    k = (np.float32(120.0), np.float32(118.0), np.float32(99.5), np.float32(59.5))
    cam = lambda x, y, z: (inv @ np.array([x, y, z, 1.0]))[:3]
    segs = [np.concatenate([g.uniform(-1, 1, 2).tolist() + [g.uniform(0.2, 3)],
                            g.uniform(-1, 1, 2).tolist() + [g.uniform(0.2, 3)]]) for _ in range(300)]
    segs = [np.concatenate([cam(*s[:3]), cam(*s[3:])]) for s in segs]
    segs += [np.concatenate([cam(-0.3, 0.1, 1.0), cam(0.2, -0.1, -1.0)]),      # crosses the near plane
             np.concatenate([cam(0.1, -0.4, -0.5), cam(0.1, 0.4, -0.2)]),      # wholly behind the camera
             np.concatenate([cam(0.0, -0.4, 1.0), cam(0.0, 0.4, 1.0)]),        # vertical
             np.concatenate([cam(-0.6, 0.1, 1.5), cam(0.6, 0.1, 1.5)]),        # horizontal
             np.concatenate([cam(-0.6, 0.1, 1.5), cam(0.6, 0.1, 1.5)]),        # the same, a later index
             np.concatenate([cam(-0.5, -0.2, 9.0), cam(0.5, 0.2, 9.0)])]       # behind the picture's depth
    segs = np.array(segs, np.float32)
    cols = g.integers(0, 256, (len(segs), 3)).astype(np.uint8)
    zbuf = np.full((H, W), np.inf, np.float32)
    zbuf[:, : W // 2] = g.uniform(0.5, 5.0, (H, W // 2)).astype(np.float32)
    zbuf[10:20, :] = 8.0
    base = g.integers(0, 256, (H, W, 3)).astype(np.uint8)
    out = torch.from_numpy(base.copy()).to(dev)
    keys = torch.empty(H * W, dtype=torch.int64, device=dev)
    V.draw_lines(torch.from_numpy(segs).to(dev), torch.from_numpy(cols).to(dev), torch.from_numpy(w2c).to(dev), k, W,
                 H, 0.01, torch.from_numpy(zbuf).to(dev), keys, out)
    ref = O.lines(segs, cols, w2c, k, W, H, 0.01, zbuf, base)
    got = out.cpu().numpy()
    assert np.array_equal(got, ref)
    assert (got != base).any(axis=-1).sum() > 500


@pytest.fixture(scope="module")
def record_path(tmp_path_factory):
    import splatam_b200 as S
    from splatam_b200 import formats, slam
    from test_checkpoint_gpu import K
    from test_slam_gpu import _opaque_sequence
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    dev = torch.device("cuda:0")
    cam, frames, _, _ = _opaque_sequence(dev, S.GaussianRasterizationSettings, T=5)
    init, radius = slam.initialize_map(frames[0], K)
    torch.manual_seed(3); np.random.seed(3)
    out = slam.run_slam(init, frames, cam, fused=True, intrinsics=K, add_new_gaussians=True, sil_thres=0.5,
                        scene_radius=radius, window=4, mapping_iters=4, first_frame_iters=10, tracking_iters=10,
                        map_every=1)
    d = str(tmp_path_factory.mktemp("viewer_record"))
    H, W = frames[0]["im"].shape[-2:]
    return formats.save_run_record(d, out["gauss"], out["rots"], out["trans"], out["timestep"], K, torch.eye(4), W, H,
                                   [torch.eye(4)] * len(frames), out["keyframe_time_indices"])


def _expected(record, cfg, views, v, t, compact=False):
    """The oracle's frame from the viewer's own device renders."""
    from splatam_b200 import viewer as V
    s = cfg.view_scale
    if cfg.render_mode == "centers":
        sel = np.ones(record.P, bool) if t is None else record.timestep_host <= t
        out, z = O.points(record.means3D.cpu().numpy()[sel], record.colors.cpu().numpy()[sel], None, 0.0,
                          views.w2c[v].cpu().numpy(), views.k_out, views.W, views.H, s, cfg.viz_near, cfg.viz_far)
    else:
        im, depth, sil = V.render_view(record, views, v, t, compact)
        mode = 1 if cfg.render_mode == "depth" else 2 if sil is not None else 0
        out, z = O.compose(im.cpu().numpy(), depth[0].cpu().numpy(), None if sil is None else sil[0].cpu().numpy(),
                           mode, s, V.JET_U8)
    if cfg.visualize_cams:
        segs, cols = views.lines(t if views.online else 0)
        out = O.lines(segs.cpu().numpy(), cols.cpu().numpy(), views.w2c[v].cpu().numpy(), views.k_out, views.W,
                      views.H, cfg.viz_near, z, out)
    return out


CFGS = [dict(), dict(render_mode="depth"), dict(render_mode="centers"), dict(show_sil=True),
        dict(visualize_cams=False, offset_first_viz_cam=False, view_scale=1)]


@pytest.mark.parametrize("viz", CFGS, ids=["color", "depth", "centers", "sil", "plain_s1"])
def test_views_equal_oracle(cuda_device, record_path, viz):
    from splatam_b200 import viewer as V
    rec = V.load_record(record_path, cuda_device)
    assert rec.monotone and rec.T == 5
    cfg = V.ViewerConfig.from_viz(dict(viz_w=160, viz_h=96, **viz))
    frame = V.final_view(rec, cfg)
    assert frame.shape == (96 * cfg.view_scale, 160 * cfg.view_scale, 3)
    assert np.array_equal(frame.cpu().numpy(), _expected(rec, cfg, V._Views(rec, cfg, False), 0, None))
    views = V._Views(rec, cfg, True)
    prefix = list(V.online_frames(rec, cfg))
    gathered = list(V.online_frames(rec, cfg, compact=True))
    assert [t for t, _ in prefix] == list(range(rec.T))
    for (t, a), (_, b) in zip(prefix, gathered):
        assert torch.equal(a, b), t
        assert np.array_equal(a.cpu().numpy(), _expected(rec, cfg, views, t, t)), t
    assert not torch.equal(prefix[0][1], prefix[-1][1])


def test_selection_prefix_and_compaction(cuda_device, record_path, tmp_path):
    from splatam_b200 import viewer as V
    rec = V.load_record(record_path, cuda_device)
    for t in range(rec.T):
        sel = rec.timestep <= t
        want = [x[sel] for x in (rec.means3D, rec.colors, rec.rotations, rec.opacities, rec.scales)]
        for compact in (False, True):
            got = V._subset(rec, t, compact)
            assert all(torch.equal(a, b) for a, b in zip(got, want)), (t, compact)
    # a record whose timestep is not monotone (as offline densification leaves it) takes the compaction path
    raw = dict(np.load(record_path))
    perm = np.random.default_rng(0).permutation(raw["means3D"].shape[0])
    for k in ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales", "timestep"):
        raw[k] = raw[k][perm]
    path = str(tmp_path / "params.npz")
    np.savez(path, **raw)
    shuffled = V.load_record(path, cuda_device)
    assert not shuffled.monotone
    cfg = V.ViewerConfig(viz_w=160, viz_h=96, render_mode="centers")
    views = V._Views(shuffled, cfg, True)
    for t, f in V.online_frames(shuffled, cfg, every=2):
        assert np.array_equal(f.cpu().numpy(), _expected(shuffled, cfg, views, t, t)), t
        sel = shuffled.timestep <= t
        got = V._subset(shuffled, t, False)
        assert torch.equal(got[0], shuffled.means3D[sel])


def test_render_record_writes_frames(cuda_device, record_path, tmp_path):
    from PIL import Image
    from splatam_b200 import viewer as V
    rec = V.load_record(record_path, cuda_device)
    cfg = V.ViewerConfig(viz_w=160, viz_h=96)
    raw = str(tmp_path / "frames.rgb")
    paths = V.render_record(rec, cfg, str(tmp_path), "online", every=2, raw=raw)
    assert paths == [str(tmp_path / "online" / ("%06d.png" % t)) for t in (0, 2, 4)]
    frames = {t: f.cpu().numpy() for t, f in V.online_frames(rec, cfg, every=2)}
    stream = np.fromfile(raw, np.uint8).reshape(3, 192, 320, 3)
    for i, (t, f) in enumerate(sorted(frames.items())):
        assert np.array_equal(np.asarray(Image.open(paths[i])), f)
        assert np.array_equal(stream[i], f)
    (final,) = V.render_record(rec, cfg, str(tmp_path), "final")
    assert final == str(tmp_path / "final.png")
    assert np.array_equal(np.asarray(Image.open(final)), V.final_view(rec, cfg).cpu().numpy())


@pytest.mark.parametrize("mode", ["color", "centers"])
def test_frame_loop_has_no_torch_synchronisation(cuda_device, record_path, mode):
    """The frames' own work (selection, cameras, kernels) never waits for the device; the only wait left per rendered
    frame is the rasterizer's instance-count read inside the library."""
    from splatam_b200 import viewer as V
    rec = V.load_record(record_path, cuda_device)
    cfg = V.ViewerConfig(viz_w=160, viz_h=96, render_mode=mode)
    gen = V.online_frames(rec, cfg)
    next(gen)                                          # builds the cameras (one upload) and warms every shape
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        frames = [f for _, f in gen]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(frames) == rec.T - 1


def test_reference_loaders_and_render(cuda_device, record_path):
    """load_record / cameras / selection against the reference's unmodified load_camera, load_scene_data,
    get_rendervars and render (from the install in oracle/_ref, with this project's drop-in rasterizer)."""
    from test_checkpoint_cpu import _final_recon
    from splatam_b200 import viewer as V
    ref = _final_recon()
    cfg = V.ViewerConfig(viz_w=160, viz_h=96)
    viz = dict(viz_w=160, viz_h=96, viz_near=0.01, viz_far=100.0)
    w2c, k = ref.load_camera(viz, record_path)
    rec = V.load_record(record_path, cuda_device)
    assert np.array_equal(rec.k(cfg), k) and np.array_equal(rec.first_w2c, w2c)
    rv, _, all_w2cs = ref.load_scene_data(record_path, w2c, k)
    # the reference builds all_w2cs with CUDA kernels, load_record on the host: F.normalize's norm is a reduction whose
    # order differs between the two devices, so agreement is to float32 round-off here.  Run on the host, the
    # reference gives load_record's matrices bit for bit (tests/test_viewer_golden_cpu.py).
    assert np.allclose(np.stack(all_w2cs), rec.all_w2cs, rtol=0, atol=1e-6)
    for a, b in ((rv["means3D"], rec.means3D), (rv["colors_precomp"], rec.colors), (rv["rotations"], rec.rotations),
                 (rv["opacities"], rec.opacities), (rv["scales"], rec.scales)):
        assert torch.equal(a, b)
    view = V.view_w2cs(rec, cfg, online=False)[0]
    im, depth, _ = ref.render(view, k, rv, dict(rv, colors_precomp=torch.zeros_like(rv["means3D"])), viz)
    mine = V.render_view(rec, V._Views(rec, cfg, False), 0, None)
    assert torch.equal(im, mine[0]) and torch.equal(depth, mine[1])
