"""RGB-D ICP and the photometric health check on the GPU (csrc/icp.cu, csrc/reloc.cu through splatam_b200/icp.py
and reloc.py): grey pyramids, gradients and photometric codes equal the numpy restatement bit for bit, the joint
normal equations and the pose agree to double rounding, weight 0 is sb_icp_align bit for bit, a captured call replays
bit for bit, a textured plane and the corridor are aligned, the NCC health record matches the oracle, and the
photometric options inside run_slam and relocalisation."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import icp_scene as S
from oracle import icp_numpy as G
from oracle import rgbd_icp_numpy as O
from util import bits_equal, load

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def _inputs(H, W, seed):
    icp_gpu = load("tests/test_icp_gpu.py")
    K, ds, data, prev, guess, cur = icp_gpu._inputs(H, W, seed)
    cpu = load("tests/test_rgbd_icp_cpu.py")
    mrgb = cpu._texture(prev.astype(np.float64), K, np.where(ds[1] > 0.99, ds[0] / np.maximum(ds[1], 1e-6), 0))
    drgb = cpu._texture(cur, K, np.nan_to_num(data, nan=0.0, posinf=0.0))
    mrgb[:, 5, 7] = np.nan                                          # a NaN colour sample in each
    drgb[:, H // 2, W // 2] = np.inf
    return K, ds, mrgb, data, drgb, prev, guess


@pytest.mark.parametrize("H,W", [(45, 97), (680, 1200)])
def test_grey_maps_codes_and_pose_match_the_oracle(cuda_device, H, W):
    from splatam_b200 import icp
    dev = cuda_device
    K, ds, mrgb, data, drgb, prev, guess = _inputs(H, W, seed=H)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    levels = O.pyramid(ds, mrgb, data, drgb, K)
    T0 = (G._h(prev.astype(np.float64)[:3]) @ G._h(G.rigid_inverse(guess)))[:3]
    lam = icp.DEFAULT_WEIGHT
    lam2 = float(np.float32(lam)) ** 2
    for l in range(G.LEVELS):
        iters = [0, 0, 0]
        iters[l] = 1
        _, st = icp.align_rgbd(t(ds), t(mrgb), t(data), t(drgb), K, t(prev), t(guess), iters, lam)
        maps = {k: v.cpu().numpy() for k, v in icp.export_level_rgbd(H, W, l, dev).items()}
        ref = levels[l]
        for k in ("model_grey", "data_grey", "model_grad", "model_depth", "model_normal"):
            assert bits_equal(maps[k], ref[k]), (l, k)
        assoc, photo, terms, ph = O.associate(ref, T0, l)
        assert bits_equal(maps["assoc"], assoc) and bits_equal(maps["photo"], photo), l
        assert (photo == 2).sum() > 0.3 * (photo > 0).sum(), l
        s = st.cpu().numpy()
        joint = terms[:27] + lam2 * ph[:27]
        assert s[3] == terms[28] and s[4] == terms[29] and s[36] == ph[28], l
        assert _rel(s[8:35], joint) <= 1e-9 and _rel(s[38:59], ph[:21]) <= 1e-9 and _rel(s[59:65], ph[21:27]) <= 1e-9
        assert _rel(s[65], ph[27]) <= 1e-9 and _rel(s[35], terms[27]) <= 1e-9, l
    w2c, st = icp.align_rgbd(t(ds), t(mrgb), t(data), t(drgb), K, t(prev), t(guess), weight=lam)
    ref_w2c, ref_st, _ = O.align(ds, mrgb, data, drgb, K, prev, guess, weight=lam)
    s = st.cpu().numpy()
    assert s[0] == ref_st[0] == 1.0, (s[:8], ref_st[:8])
    assert np.abs(w2c.cpu().numpy() - ref_w2c).max() <= 1e-6


def test_weight_zero_is_the_geometric_alignment_bit_for_bit(cuda_device):
    from splatam_b200 import icp
    dev = cuda_device
    for H, W, seed in ((45, 97, 3), (680, 1200, 4)):
        K, ds, mrgb, data, drgb, prev, guess = _inputs(H, W, seed)
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        a_w, a_s = icp.align(t(ds), t(data), K, t(prev), t(guess))
        b_w, b_s = icp.align_rgbd(t(ds), t(mrgb), t(data), t(drgb), K, t(prev), t(guess), weight=0.0)
        assert torch.equal(a_w, b_w) and torch.equal(a_s, b_s[:36])
        assert bool(b_s[36] > 0) and bool(torch.isfinite(b_s).all())


def test_graph_replay_is_bit_identical(cuda_device):
    from splatam_b200 import icp
    dev = cuda_device
    K, ds, mrgb, data, drgb, prev, guess = _inputs(120, 160, 7)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    args = (t(ds), t(mrgb), t(data), t(drgb), K, t(prev), t(guess))
    a_w, a_s = icp.align_rgbd(*args)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            g_w, g_s = icp.align_rgbd(*args)
    torch.cuda.current_stream(dev).wait_stream(side)
    g_w.zero_(); g_s.zero_()
    g.replay()
    torch.cuda.synchronize(dev)
    assert bool(a_s[0] == 1.0)
    assert torch.equal(a_w, g_w) and torch.equal(a_s, g_s)


def _two_views(dev, gt, cam, axis, deg, tvec):
    rots = torch.zeros(1, 4, 2, device=dev)
    rots[0, 0] = 1.0
    axis = torch.tensor(axis, dtype=torch.float32)
    axis = axis / axis.norm()
    a = math.radians(deg) / 2
    rots[0, :, 1] = torch.cat([torch.tensor([math.cos(a)]), math.sin(a) * axis]).to(dev)
    trans = torch.zeros(1, 3, 2, device=dev)
    trans[0, :, 1] = torch.tensor(tvec)
    return dict(gt, cam_unnorm_rots=rots, cam_trans=trans), dict(cam=cam, w2c=torch.eye(4, device=dev))


def _err(w2c, params):
    from splatam_b200 import mapping as M
    truth = M.camera_w2c(params["cam_unnorm_rots"][..., 1], params["cam_trans"][..., 1])[0]
    e = (w2c.double() @ torch.linalg.inv(truth.double())).cpu().numpy()
    return float(np.linalg.norm(e[:3, 3])), float(np.degrees(Rotation.from_matrix(e[:3, :3]).magnitude()))


def _align_views(params, frame, K, weight=None):
    from splatam_b200 import icp
    im0, ds0 = icp.model_render(params, 0, frame)
    im1, ds1 = icp.model_render(params, 1, frame)
    data = torch.where(ds1[1] > 0.99, ds1[0] / ds1[1], torch.zeros_like(ds1[0]))
    eye = torch.eye(4, device=data.device)
    if weight is None:
        return icp.align(ds0, data, K, eye, eye)
    return icp.align_rgbd(ds0, im0, data, im1, K, eye, eye, weight=weight)


def test_textured_plane_rendered_by_the_rasterizer(cuda_device):
    """One textured wall of small opaque splats at one depth: the geometric alignment rejects it, the RGB-D one accepts
    it and recovers a 5.8 cm / 3 deg motion to within 2.5 cm, 0.4 of the guess's error, and 0.1 deg.  Measured on an
    H100: 16.9 mm and 0.007 deg.  The residual is converged (the same with three times the iterations and with ten
    times the weight) and shrinks with the splats (24.2, 20.1 and 16.9 mm for 12, 6 and 4 mm splats): where opaque
    splats overlap, each pixel shows the splat nearest the camera, so after a turn the rendered texture is displaced
    by a fraction of a splat toward the nearer side.  Depth jitter that fixes the order also gives depth alone enough
    relief to be accepted, so the test keeps one depth."""
    import scenes
    import splatam_b200 as SB
    from splatam_b200 import icp
    dev = cuda_device
    g = torch.Generator().manual_seed(5)
    n = 480_000
    xy = (torch.rand(n, 2, generator=g) - 0.5) * torch.tensor([5.0, 3.5])
    means = torch.cat([xy, torch.full((n, 1), 2.5)], 1)
    grey = (0.5 + 0.25 * torch.sin(7 * xy[:, :1]) * torch.cos(5 * xy[:, 1:])
            + 0.1 * torch.sin(3 * xy[:, :1] + 4 * xy[:, 1:]))
    gt = dict(means3D=means, rgb_colors=grey.repeat(1, 3), unnorm_rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1),
              logit_opacities=torch.full((n, 1), 6.0), log_scales=torch.full((n, 1), math.log(0.004)))
    gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
    camd = dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5)
    sc = scenes.room(seed=1, P=10, cam=camd)
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    K = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])
    params, frame = _two_views(dev, gt, cam, (0.2, 1.0, 0.3), 3.0, (0.04, -0.03, 0.03))
    _, gs = _align_views(params, frame, K)
    w2c, st = _align_views(params, frame, K, icp.DEFAULT_WEIGHT)
    dt, dr = _err(w2c, params)
    d0, _ = _err(torch.eye(4, device=dev), params)                 # the guess: the first view's pose
    print("textured plane: geometric", icp.read_stats(gs), "rgbd", icp.read_stats(st), "error %.3f mm %.4f deg"
          % (1e3 * dt, dr), "guess %.3f mm" % (1e3 * d0))
    assert not icp.read_stats(gs)["accepted"]
    assert icp.read_stats(st)["accepted"] and dt <= 2.5e-2 and dt <= 0.4 * d0 and dr <= 0.1, (dt, d0, dr)


def test_corridor_views(cuda_device):
    """test_icp_gpu's two corridor views (8.1 cm and 4 deg apart), aligned with depth and colour: within 1 cm and 0.2
    deg (the geometric alignment: 8.26 mm on an H100).  The error is printed."""
    import splatam_b200 as SB
    from splatam_b200 import icp
    icp_gpu = load("tests/test_icp_gpu.py")
    dev = cuda_device
    sc, gt = icp_gpu._opaque_room(dev)
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    params, frame = _two_views(dev, gt, cam, (0.3, 1.0, -0.2), 4.0, (0.05, -0.03, 0.055))
    res = {}
    for lam in (None, icp.DEFAULT_WEIGHT):
        w2c, st = _align_views(params, frame, icp_gpu.K_ROOM, lam)
        res[lam] = (_err(w2c, params), icp.read_stats(st))
        print("corridor weight", lam, "error %.3f mm %.4f deg" % (1e3 * res[lam][0][0], res[lam][0][1]), res[lam][1])
    (dt, dr), s = res[icp.DEFAULT_WEIGHT]
    assert s["accepted"] and dt <= 1e-2 and dr <= 0.2, (dt, dr)


def test_health_rgb_matches_the_oracle(cuda_device):
    from splatam_b200 import reloc
    dev = cuda_device
    rel = load("tests/test_reloc_gpu.py")
    for H, W, seed in ((45, 97, 1), (680, 1200, 2)):
        rgb, depth, sil = rel._images(2, H, W, seed, dev)
        frame = depth[0]
        g = torch.Generator().manual_seed(seed)
        dmap = torch.nan_to_num(frame.cpu(), nan=2.0, posinf=2.0) + torch.randn(H, W, generator=g) * 0.04
        ds = torch.stack([dmap.to(dev) * sil[0], sil[0]])
        m_rgb = (0.7 * rgb[1] + 0.3 * rgb[0]).contiguous()          # correlated with the frame's colour
        cfg = reloc.config(dict(photometric=True))
        st = reloc._health_rgb_of(ds, m_rgb, frame, rgb[0], cfg).cpu().numpy()
        geo = reloc._health_of(ds, frame, cfg).cpu().numpy()
        ref = O.health_ncc(ds.cpu().numpy(), frame.cpu().numpy(), m_rgb.cpu().numpy(), rgb[0].cpu().numpy(),
                           cfg["tau_abs"], cfg["tau_rel"], cfg["min_coverage"], cfg["min_inliers"], cfg["min_ncc"])
        assert bits_equal(st[:4], geo[:4])
        assert bits_equal(st[[0, 1, 2, 4, 5]], ref[[0, 1, 2, 4, 5]]) and abs(st[6] - ref[6]) <= 1e-9
        assert 0 < st[5] <= st[2] and 0.1 < st[6] < 0.99


def test_fast_motion_with_rgbd_icp_start(cuda_device):
    """test_icp_gpu's fast-motion sequence with pose_init="rgbd_icp": within that test's ATE bound."""
    import splatam_b200 as SB
    from splatam_b200 import slam
    icp_gpu = load("tests/test_icp_gpu.py")
    dev = cuda_device
    cam, frames, rots_gt, trans_gt = icp_gpu._fast_sequence(dev, SB.GaussianRasterizationSettings, 4.0)
    travelled = float(trans_gt[0, :, -1].norm())
    timing = {}
    out = icp_gpu._full_loop(frames, cam, mapping_iters=12, first_frame_iters=60, tracking_iters=40,
                             pose_init="rgbd_icp", timing=timing)
    ate = slam.ate_rmse(out["rots"], out["trans"], rots_gt, trans_gt)
    print("rgbd_icp ATE %.4f m of %.3f m travelled" % (ate, travelled), "timing", timing, "icp", out["icp"])
    assert len(out["icp"]) == 8 and all("photo_rms" in s for s in out["icp"])
    assert sum(s["accepted"] for s in out["icp"]) >= 6
    assert ate < 0.05 * travelled, (ate, travelled)


def test_loop_room_retrieval_with_photometric_verification(cuda_device):
    """test_reloc_gpu's loop-room queries with relocalise photometric: recall is unchanged (the descriptors are), every
    pose within 5 cm and 2 deg and at least 10 of 11 within 5 mm and 0.3 deg.  Frame 38's error is printed."""
    import scenes
    import splatam_b200 as SB
    from splatam_b200 import mapping as M, reloc
    rel = load("tests/test_reloc_gpu.py")
    dev = cuda_device
    sc = scenes.loop_room()
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    gt = {k: v.contiguous() for k, v in sc.splatam_params(dev).items()}
    rots, trans = scenes.loop_trajectory(81, dev)
    cols = list(range(0, 81, 5))
    db = reloc.Database.from_record(dict(gt, cam_unnorm_rots=rots, cam_trans=trans), cols, cam)
    cfg = reloc.config(dict(photometric=True))
    bad, close, hitsk = [], 0, 0
    queries = [2, 8, 13, 22, 31, 38, 47, 53, 62, 69, 77]
    for t in queries:
        p = rel._query_params(gt, rots, trans, t)
        f = rel._frame(gt, rots, trans, t, cam)
        rec = reloc.relocalise(p, f, t, db, rel.K_LOOP, cfg, tracking=dict(num_iters=40))
        near = cols[int(np.argmin([abs(c - t) for c in cols]))]
        alt = [c for c in cols if abs(c - t) == abs(near - t)]
        hitsk += any(c in alt for c in rec["columns"])
        est = M.camera_w2c(p["cam_unnorm_rots"][..., t], p["cam_trans"][..., t])[0]
        e = rel._pose_err(est, M.camera_w2c(rots[..., t], trans[..., t])[0])
        print("query %d: candidates %s accepted %s health %s error %.2f mm %.3f deg" % (
            t, rec["columns"], rec["accepted"], rec["health"], 1e3 * e[0], e[1]))
        close += e[0] < 0.005 and e[1] < 0.3
        if not (rec["accepted"] and e[0] < 0.05 and e[1] < 2.0):
            bad.append((t, rec["columns"], rec["accepted"], e))
    print("recall@k %d/%d, within 5 mm and 0.3 deg %d" % (hitsk, len(queries), close))
    assert hitsk == len(queries) and not bad and close >= 10, (bad, close)


@pytest.fixture(scope="module")
def kidnapped(cuda_device, tmp_path_factory):
    rel = load("tests/test_reloc_gpu.py")
    root = tmp_path_factory.mktemp("kidnap_rgb")
    return (rel._room_sequence(cuda_device, root, "kidnap"),
            rel._room_sequence(cuda_device, root, "unmapped", unmapped=True))


def test_kidnapped_sequences_with_photometric_relocalisation(cuda_device, kidnapped):
    """Mapped jump: frame 41 is relocalised and the ATE bound of test_kidnapped_sequence_is_relocalised holds.  Jump
    into unmapped space: the jump frame is flagged lost, no frame after 41 is relocalised more than 5 cm or 2 deg from
    the truth, and lost frames add no Gaussians.  With the depth-only check the same sequence relocalises frame 45 at a
    wrong pose (test_reloc_gpu's test_jump_into_unmapped_space_is_flagged_lost), so this fails without the colour NCC.
    The NCC of every final health check is printed."""
    from splatam_b200 import mapping as M
    rel = load("tests/test_reloc_gpu.py")
    (cam, frames, gt_w2c), (cam_u, frames_u, gt_u) = kidnapped
    on = rel._run(frames, cam, relocalise=dict(photometric=True))
    ref = rel._run(frames[:41], cam)
    a_on, a_ref = rel._ate(on, gt_w2c), rel._ate(ref, gt_w2c[:41])
    print("kidnapped photometric: ATE %.4f m, frames 0..40 %.4f m; reloc %s" % (a_on, a_ref, on["reloc"]))
    assert any(r["frame"] == 41 and r["relocalised"] for r in on["reloc"]), on["reloc"]
    assert a_on <= 2 * a_ref + 0.005, (a_on, a_ref)
    out = rel._run(frames_u, cam_u, relocalise=dict(photometric=True))
    lost = out["reloc_lost"]
    errs = {}
    for r in out["reloc"]:
        if r["relocalised"]:
            t = r["frame"]
            est = M.camera_w2c(out["rots"][..., t], out["trans"][..., t])[0].double().cpu()
            errs[t] = rel._pose_err(est, gt_u[t].double())
    print("unmapped photometric: lost %s, relocalised %s, reloc %s" % (lost, errs, out["reloc"]))
    print("unmapped photometric: (frame, ncc of the checked candidate)",
          [(r["frame"], r.get("ncc")) for r in out["reloc"] if r.get("ncc") is not None])
    assert lost and lost[0] == 41, lost
    assert all(e[0] < 0.05 and e[1] < 2.0 for t, e in errs.items() if t > 41), errs
    assert not torch.isin(out["timestep"].cpu(), torch.tensor(lost, dtype=out["timestep"].dtype)).any()


def test_photometric_opt_in_without_lost_frames_changes_nothing(cuda_device, tmp_path, monkeypatch):
    """test_reloc_gpu's opt-in check with relocalise photometric: on the loop sequence and the 40-frame corridor, no
    frame is flagged and the run equals relocalise=None bit for bit."""
    import scenes
    import splatam_b200 as SB
    from splatam_b200 import mapping as M
    dev = cuda_device
    icp_gpu, rel = load("tests/test_icp_gpu.py"), load("tests/test_reloc_gpu.py")
    cam_c, frames_c, rots_c, trans_c = icp_gpu._fast_sequence(dev, SB.GaussianRasterizationSettings, 1.0, T=40)
    cam_l, frames_l, _ = rel._room_sequence(dev, tmp_path, "loop", T=31)
    rots_l, trans_l = scenes.loop_trajectory(31, dev)
    for name, frames, cam, rots_gt, trans_gt, run in (
            ("corridor", frames_c, cam_c, rots_c, trans_c, icp_gpu._full_loop),
            ("loop", frames_l, cam_l, rots_l, trans_l, rel._run)):
        def stand_in(params, frame, **k):
            t = frame["id"]
            with torch.no_grad():
                params["cam_unnorm_rots"][..., t] = rots_gt[..., t]
                params["cam_trans"][..., t] = trans_gt[..., t]
            return [0.0]
        monkeypatch.setattr(M, "track_frame", stand_in)
        kw = dict(mapping_iters=0, tracking_iters=10) if name == "corridor" else dict(mapping_iters=0,
                                                                                       first_frame_iters=0)
        a = run(frames, cam, **kw)
        b = run(frames, cam, relocalise=dict(photometric=True), **kw)
        print(name, "reloc", b["reloc"])
        nccs = []
        for t in range(1, len(frames)):                 # the photometric health of every frame at its true pose
            from splatam_b200 import reloc
            p = dict(b["gauss"], cam_unnorm_rots=b["rots"], cam_trans=b["trans"])
            nccs.append(reloc.read_health(reloc.health(p, frames[t], t, reloc.config(dict(photometric=True))))["ncc"])
        print(name, "ncc of healthy frames: min %.4f median %.4f max %.4f" % (min(nccs), float(np.median(nccs)),
                                                                             max(nccs)))
        assert b["reloc"] == [] and b["reloc_lost"] == []
        assert torch.equal(a["rots"], b["rots"]) and torch.equal(a["trans"], b["trans"]), name
        for k in a["gauss"]:
            assert torch.equal(a["gauss"][k], b["gauss"][k]), (name, k)


def test_default_options_never_reach_the_new_entry_points(cuda_device, monkeypatch):
    """A short GPU run with the defaults, and one with pose_init="icp" and relocalise={} (the depth-only options), call
    neither sb_rgbd_icp_* nor sb_track_health_rgb; with pose_init="rgbd_icp" and relocalise photometric both are
    called (so the spy sees them)."""
    import splatam_b200 as SB
    from splatam_b200 import _lib
    icp_gpu = load("tests/test_icp_gpu.py")
    cam, frames, _, _ = icp_gpu._fast_sequence(cuda_device, SB.GaussianRasterizationSettings, 1.0, T=4)
    called = []
    real = _lib.call

    def spy(name, *a, **k):
        called.append(name)
        return real(name, *a, **k)
    monkeypatch.setattr(_lib, "call", spy)
    new = lambda: sorted({n for n in called if n.startswith("sb_rgbd_icp") or n == "sb_track_health_rgb"})
    for kw in ({}, dict(pose_init="icp", relocalise={})):
        called.clear()
        icp_gpu._full_loop(frames, cam, mapping_iters=2, tracking_iters=4, **kw)
        assert new() == [], (kw, new())
        assert ("sb_icp_align" in called) == ("pose_init" in kw)
    called.clear()
    icp_gpu._full_loop(frames, cam, mapping_iters=2, tracking_iters=4, pose_init="rgbd_icp",
                       relocalise=dict(photometric=True))
    assert new() == ["sb_rgbd_icp_align", "sb_track_health_rgb"], new()
