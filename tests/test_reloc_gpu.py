"""Relocalisation on the GPU (csrc/reloc.cu through splatam_b200/reloc.py): descriptors, scores, top-k and health
records against the numpy restatement; retrieval and recovery in the loop room; no false accept; an opt-in run with
no lost frame equals the default run; the kidnapped sequence inside run_slam; localisation of a new sequence in a
saved map; and a resume that rebuilds the database."""
import math

import numpy as np
import pytest
import torch

import scenes
from oracle import reloc_numpy as O
from util import bits_equal, load

pytestmark = pytest.mark.gpu

K_LOOP = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])


def _images(B, H, W, seed, dev):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(B, 3, H, W, generator=g)
    depth = torch.rand(B, H, W, generator=g) * 4 + 0.3
    sil = torch.rand(B, H, W, generator=g) * 0.1 + 0.93          # some at or below 0.99
    holes = torch.rand(B, H, W, generator=g)
    depth[holes < 0.05] = 0.0
    depth[(holes >= 0.05) & (holes < 0.07)] = float("nan")
    depth[(holes >= 0.07) & (holes < 0.09)] = float("inf")
    depth[(holes >= 0.09) & (holes < 0.11)] = -1.0
    depth[:, : H // 3, : W // 4] = 0.0                           # a large hole: invalid descriptor pixels
    rgb[0, :, 1, 1] = float("nan")
    return rgb.to(dev), depth.to(dev), sil.to(dev)


@pytest.mark.parametrize("H,W", [(45, 97), (480, 640), (680, 1200)])
def test_thumbnails_are_bit_equal_to_the_oracle(cuda_device, H, W):
    from splatam_b200 import reloc
    rgb, depth, sil = _images(2, H, W, H, cuda_device)
    for s in (None, sil):
        d = depth if s is None else depth * s
        ours = reloc.thumbnails(rgb, d, s).cpu().numpy()
        ref = O.thumbnails(rgb.cpu().numpy(), d.cpu().numpy(), None if s is None else s.cpu().numpy())
        assert ours.shape == (2, 2) + O.thumbnail_size(H, W)[:2]
        assert bits_equal(ours, ref), (H, W, s is None)
        assert np.isnan(ours).any() and not np.isnan(ours).all()


@pytest.mark.parametrize("N", [1, 7, 2000, 10_000])
def test_scores_and_topk_match_the_oracle(cuda_device, N):
    from splatam_b200 import reloc
    dev = cuda_device
    g = torch.Generator().manual_seed(N)
    base = torch.rand(2, 48, 85, generator=g)
    db = base[None] + 0.5 * torch.rand(N, 2, 48, 85, generator=g)
    db[torch.rand(N, 2, 48, 85, generator=g) < 0.1] = float("nan")
    if N > 3:
        db[3] = db[1]                                            # a tie: the lower index first
    db[N - 1, :, :30] = float("nan")                             # too little overlap: -2
    q = base.clone()
    q[:, :5] = float("nan")
    s = reloc.score(q.to(dev), db.to(dev)).cpu().numpy()
    ref = O.score(q.numpy(), db.numpy())
    assert np.abs(s - ref).max() <= 1e-12 * np.abs(ref).max()
    assert (s == -2.0).sum() >= 1 and bits_equal(s[ref == -2.0], ref[ref == -2.0])
    k = min(8, N)
    idx, top = reloc.topk(torch.from_numpy(s).to(dev), k)
    ridx, rtop = O.topk(s, k)
    assert idx.cpu().numpy().tolist() == ridx.tolist() and bits_equal(top.cpu().numpy(), rtop)


def test_health_records_match_the_oracle(cuda_device):
    from splatam_b200 import reloc
    dev = cuda_device
    for H, W, seed in ((45, 97, 1), (680, 1200, 2)):
        _, depth, sil = _images(1, H, W, seed, dev)
        frame = depth[0]
        g = torch.Generator().manual_seed(seed)
        dmap = torch.nan_to_num(frame.cpu(), nan=2.0, posinf=2.0) + torch.randn(H, W, generator=g) * 0.04
        ds = torch.stack([dmap.to(dev) * sil[0], sil[0]])
        cfg = reloc.config({})
        st = reloc._health_of(ds, frame, cfg).cpu().numpy()
        ref = O.health(ds.cpu().numpy(), frame.cpu().numpy(), cfg["tau_abs"], cfg["tau_rel"], cfg["min_coverage"],
                       cfg["min_inliers"])
        assert bits_equal(st[[0, 1, 2, 4]], ref[[0, 1, 2, 4]]) and abs(st[3] - ref[3]) <= 1e-9 * ref[3]
        assert 0 < st[2] < st[1] < st[0]


# ---- the loop room --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def room(cuda_device):
    import splatam_b200 as SB
    sc = scenes.loop_room()
    cam = sc.settings(SB.GaussianRasterizationSettings, cuda_device)
    gt = {k: v.contiguous() for k, v in sc.splatam_params(cuda_device).items()}
    rots, trans = scenes.loop_trajectory(81, cuda_device)
    return cam, gt, rots, trans


def _frame(gt, rots, trans, t, cam, sensor=True):
    from splatam_b200 import slam
    f = slam.render_frame(gt, rots, trans, t, cam)
    if sensor:                          # a sensor's depth and no silhouette
        f["depth"] = torch.where(f["sil"] > 0.9, f["depth"] / f["sil"].clamp(min=1e-6), torch.zeros_like(f["depth"]))
        del f["sil"]
    return f


def _pose_err(a, b):
    R = a[:3, :3].T @ b[:3, :3]
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (float(R.trace()) - 1) / 2))))
    c = lambda m: -(m[:3, :3].T @ m[:3, 3])
    return float((c(a) - c(b)).norm()), ang


def _query_params(gt, rots, trans, t):
    """The map and its cameras, with column t (the query) reset to the identity: no prior."""
    r, tr = rots.clone(), trans.clone()
    r[..., t] = torch.tensor([1.0, 0, 0, 0], device=r.device)
    tr[..., t] = 0.0
    return dict(gt, cam_unnorm_rots=r, cam_trans=tr)


def test_retrieval_and_recovery_in_the_loop_room(cuda_device, room):
    """Database: renders of the map at every 5th frame of loop_trajectory(81).  Queries: in-between frames, no prior.
    The nearest database pose is among the k candidates for every query; relocalise recovers every pose within 5 cm and
    2 deg, and at least 9 of the 11 within 5 mm and 0.3 deg (the measured errors are printed).  Measured on an H100:
    10 of 11 within 3.6 mm and 0.09 deg; frame 38 ended 37.6 mm and 1.41 deg off, a pose the depth-only health check
    cannot tell from the true one in this room of planes.  The candidate is the first accepted one in score order:
    picking the one with the most ICP inliers took a candidate on the far side of the circle for frame 38 (549 mm
    off)."""
    from splatam_b200 import mapping as M, reloc
    cam, gt, rots, trans = room
    cols = list(range(0, 81, 5))
    db = reloc.Database.from_record(dict(gt, cam_unnorm_rots=rots, cam_trans=trans), cols, cam)
    hits1 = hitsk = 0
    bad, close = [], 0
    queries = [2, 8, 13, 22, 31, 38, 47, 53, 62, 69, 77]
    for t in queries:
        p = _query_params(gt, rots, trans, t)
        f = _frame(gt, rots, trans, t, cam)
        rec = reloc.relocalise(p, f, t, db, K_LOOP, tracking=dict(num_iters=40))
        near = cols[int(np.argmin([abs(c - t) for c in cols]))]
        alt = [c for c in cols if abs(c - t) == abs(near - t)]
        hits1 += bool(rec["columns"]) and rec["columns"][0] in alt
        hitsk += any(c in alt for c in rec["columns"])
        est = M.camera_w2c(p["cam_unnorm_rots"][..., t], p["cam_trans"][..., t])[0]
        gtw = M.camera_w2c(rots[..., t], trans[..., t])[0]
        e = _pose_err(est, gtw)
        print("query %d: candidates %s scores %s accepted %s error %.2f mm %.3f deg" % (
            t, rec["columns"], ["%.3f" % s for s in rec["scores"]], rec["accepted"], 1e3 * e[0], e[1]))
        close += e[0] < 0.005 and e[1] < 0.3
        if not (any(c in alt for c in rec["columns"]) and rec["accepted"] and e[0] < 0.05 and e[1] < 2.0):
            bad.append((t, rec["columns"], rec["accepted"], e))
    print("recall@1 %d/%d, recall@k %d/%d, within 5 mm and 0.3 deg %d" % (hits1, len(queries), hitsk, len(queries),
                                                                           close))
    assert not bad and close >= 9, (bad, close)


def test_no_false_accept(cuda_device, room):
    """A frame of another scene, an all-zero depth frame and a view from outside the room's walls are rejected, and
    column t is left bit for bit as it was."""
    import splatam_b200 as SB
    from splatam_b200 import reloc
    cam, gt, rots, trans = room
    cols = list(range(0, 81, 5))
    db = reloc.Database.from_record(dict(gt, cam_unnorm_rots=rots, cam_trans=trans), cols, cam)
    t = 13
    other = scenes.room(P=50_000, cam=scenes.LOOP_CAM)
    og = {k: v.contiguous() for k, v in other.splatam_params(cuda_device).items()}
    f_other = _frame(og, rots, trans, t, other.settings(SB.GaussianRasterizationSettings, cuda_device))
    f_zero = _frame(gt, rots, trans, t, cam)
    f_zero["depth"] = torch.zeros_like(f_zero["depth"])
    r_out, t_out = rots.clone(), trans.clone()
    t_out[0, 2, t] = -3.0                                # 3 m back along the view axis: behind the wall at z = -1.7
    f_outside = _frame(gt, r_out, t_out, t, cam)
    for name, f in (("other scene", f_other), ("zero depth", f_zero), ("outside", f_outside)):
        p = _query_params(gt, rots, trans, t)
        p["cam_unnorm_rots"][..., t] = torch.tensor([0.9, 0.1, -0.2, 0.3], device=cuda_device)
        p["cam_trans"][..., t] = torch.tensor([0.05, -0.1, 0.2], device=cuda_device)
        before = (p["cam_unnorm_rots"].clone(), p["cam_trans"].clone())
        rec = reloc.relocalise(p, f, t, db, K_LOOP, tracking=dict(num_iters=20))
        print(name, rec["columns"], rec["scores"], rec["icp"], rec["health"])
        assert not rec["accepted"], name
        assert bits_equal(p["cam_unnorm_rots"].detach().cpu().numpy(), before[0].cpu().numpy())
        assert bits_equal(p["cam_trans"].detach().cpu().numpy(), before[1].cpu().numpy())


# ---- run_slam ------------------------------------------------------------------------------------------------------

def _room_sequence(dev, root, name, **kw):
    from splatam_b200 import datasets
    if name == "loop":
        gt_w2c = scenes.write_loop_sequence(str(root / name), kw.pop("T"), dev)
    else:
        gt_w2c = scenes.write_kidnapped_sequence(str(root / name), dev, **kw)
    with datasets.RGBDSequence("replica", str(root), name, scenes.loop_data_config(), desired_height=192,
                               desired_width=320, device=dev, prefetch=2) as seq:
        frames = [seq[t] for t in range(len(seq))]
        cam = seq.cam
    return cam, frames, gt_w2c


def _run(frames, cam, **kw):
    from splatam_b200 import slam
    init, radius = slam.initialize_map(frames[0], K_LOOP)
    prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=4, removal_opacity_threshold=0.005,
                 final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
    torch.manual_seed(3); np.random.seed(3)
    kw = dict(dict(fused=True, mapping_iters=12, first_frame_iters=60, tracking_iters=40), **kw)
    return slam.run_slam(init if "resume" not in kw else None, frames, cam, intrinsics=K_LOOP, add_new_gaussians=True,
                         sil_thres=0.5, prune_dict=prune, scene_radius=radius, select_keyframes=True, window=4,
                         keyframe_every=5, **kw)


def _ate(out, gt_w2c):
    from splatam_b200 import mapping as M
    c = lambda m: -(m[:3, :3].T @ m[:3, 3])
    d = [c(M.camera_w2c(out["rots"][..., t], out["trans"][..., t])[0].double().cpu()) - c(gt_w2c[t])
         for t in range(len(gt_w2c))]
    return float(torch.stack(d).pow(2).sum(1).mean().sqrt())


def test_opt_in_without_lost_frames_changes_nothing(cuda_device, tmp_path, monkeypatch):
    """With relocalise on and no frame lost, the run equals relocalise=None bit for bit, on the loop sequence and on
    test_icp_gpu's 40-frame corridor.  Tracking is replaced by a deterministic stand-in that moves each column to the
    true pose (the product's tracking sums gradients with float atomics, so two runs of it differ in the last bits)."""
    import splatam_b200 as SB
    from splatam_b200 import mapping as M
    dev = cuda_device
    icp_tests = load("tests/test_icp_gpu.py")
    cam_c, frames_c, rots_c, trans_c = icp_tests._fast_sequence(dev, SB.GaussianRasterizationSettings, 1.0, T=40)
    cam_l, frames_l, gt_l = _room_sequence(dev, tmp_path, "loop", T=31)
    rots_l, trans_l = scenes.loop_trajectory(31, dev)          # the loop sequence's ground truth
    for name, frames, cam, rots_gt, trans_gt, run in (
            ("corridor", frames_c, cam_c, rots_c, trans_c, icp_tests._full_loop),
            ("loop", frames_l, cam_l, rots_l, trans_l, _run)):
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
        timing = {}
        b = run(frames, cam, relocalise={}, timing=timing, **kw)
        print(name, "reloc", b["reloc"], "health_s %.3f over %d frames" % (timing["health_s"], len(frames) - 1))
        assert b["reloc"] == [] and b["reloc_lost"] == [] and "reloc" not in a
        assert torch.equal(a["rots"], b["rots"]) and torch.equal(a["trans"], b["trans"]), name
        for k in a["gauss"]:
            assert torch.equal(a["gauss"][k], b["gauss"][k]), (name, k)
        assert a["counts"] == b["counts"] and a["keyframe_time_indices"] == b["keyframe_time_indices"]


@pytest.fixture(scope="module")
def kidnapped(cuda_device, tmp_path_factory):
    root = tmp_path_factory.mktemp("kidnap")
    return _room_sequence(cuda_device, root, "kidnap"), _room_sequence(cuda_device, root, "unmapped", unmapped=True)


def test_kidnapped_sequence_is_relocalised(cuda_device, kidnapped, tmp_path):
    """The jump at frame 41 (back to loop frame 12) is flagged lost and relocalised; the ATE stays within 2x that of
    the same frames without the jump (frames 0..40) plus 5 mm; without relocalisation the ATE is large.  A checkpoint
    taken after the jump restores the relocalised ids, and a resume rebuilds the database bit for bit."""
    from splatam_b200 import formats
    (cam, frames, gt_w2c), _ = kidnapped
    timing = {}
    on = _run(frames, cam, relocalise={}, timing=timing, checkpoint_dir=str(tmp_path / "ck"), checkpoint_every=59)
    off = _run(frames, cam)
    ref = _run(frames[:41], cam)
    a_on, a_off, a_ref = _ate(on, gt_w2c), _ate(off, gt_w2c), _ate(ref, gt_w2c[:41])
    print("kidnapped: ATE with relocalisation %.4f m, without %.4f m, unspliced frames 0..40 %.4f m; reloc %s; timing %s"
          % (a_on, a_off, a_ref, on["reloc"], timing))
    assert any(r["frame"] == 41 and r["relocalised"] for r in on["reloc"]), on["reloc"]
    assert on["reloc_lost"] == []
    assert a_on <= 2 * a_ref + 0.005, (a_on, a_ref)
    assert a_off > 0.1 and a_off > 5 * a_on, (a_off, a_on)
    ck = formats.load_checkpoint(str(tmp_path / "ck"), 59, cuda_device)
    assert 41 in ck["state"]["reloc_relocalised"].tolist()
    res = _run(frames, cam, relocalise={}, resume=ck)
    d0, d1 = on["reloc_database"], res["reloc_database"]
    assert d0.columns == d1.columns
    assert bits_equal(d0.descriptors.cpu().numpy(), d1.descriptors.cpu().numpy())


def test_jump_into_unmapped_space_is_flagged_lost(cuda_device, kidnapped):
    """After a jump to a view of a wall the map never saw, the jump frame is flagged lost and the lost frames add no
    Gaussians and join no keyframe list.  Measured on an H100: frames 41 to 44 stayed lost; frame 45 was relocalised
    (a false accept: a candidate pose whose rendered depth passes the health check against the back wall -- the room's
    walls are planes, which a depth-only check cannot tell apart), so the run does not end lost."""
    _, (cam, frames, gt_w2c) = kidnapped
    out = _run(frames, cam, relocalise={})
    lost = out["reloc_lost"]
    print("unmapped: lost %s, counts %s, reloc %s" % (lost, out["counts"], out["reloc"]))
    assert lost and lost[0] == 41
    assert all(not r["relocalised"] for r in out["reloc"] if r["frame"] in lost)
    assert all(k < 41 or k not in lost for k in out["keyframe_time_indices"])
    assert not torch.isin(out["timestep"].cpu(), torch.tensor(lost, dtype=out["timestep"].dtype)).any()


def test_localise_sequence_in_a_saved_map(cuda_device, room, tmp_path, monkeypatch, capsys):
    """A record of the loop room (formats.save_run_record) and a query with another radius and phase and one kidnap:
    frame 0 is found with no prior, so is the kidnap frame, every frame is within 3 cm and 1 deg, and the tool writes
    localised.npz and prints an absolute ATE below 1 cm.  Measured on an H100: 0.2 mm at frame 0, 24.6 mm at frame 1
    (tracked from zero velocity), at most 5.7 mm after it; absolute ATE 4.0 mm."""
    from splatam_b200 import formats, mapping as M
    import yaml
    dev = cuda_device
    cam, gt, rots, trans = room
    rec = formats.save_run_record(str(tmp_path / "run"), gt, rots, trans, torch.zeros(gt["means3D"].shape[0]), K_LOOP,
                                  torch.eye(4), 320, 192, [torch.eye(4)] * 81, list(range(0, 81, 5)))
    scenes.write_loop_sequence(str(tmp_path / "data" / "map"), 3, dev)          # its first pose defines the map frame
    r, t = scenes.loop_trajectory(81, dev, radius=0.22)
    idx = list(range(7, 37)) + list(range(55, 65))                              # phase 7, and a kidnap at frame 30
    scenes._write_room_sequence(str(tmp_path / "data" / "query"), (r[..., idx], t[..., idx]), dev, 21,
                                scenes.LOOP_CAM, 6553.5, 95)
    cfg = tmp_path / "loop.yaml"
    cfg.write_text(yaml.safe_dump(dict(dataset_name="replica", **scenes.loop_data_config())))
    argv = ["--record", rec, "--dataset", "replica", "--basedir", str(tmp_path / "data"), "--sequence", "query",
            "--config", str(cfg), "--map-dataset", "replica", "--map-basedir", str(tmp_path / "data"),
            "--map-sequence", "map", "--map-config", str(cfg), "--out", str(tmp_path / "loc")]
    tool = load("tools/localise_sequence.py")
    line = tool.main(argv)
    print(capsys.readouterr().out)
    z = np.load(tmp_path / "loc" / "localised.npz")
    assert z["cam_unnorm_rots"].shape == (1, 4, len(idx)) and z["health"].shape == (len(idx), 5)
    assert bool(z["relocalised"][0]) and bool(z["relocalised"][30]) and not z["lost"].any()
    errs = []
    for s, k in enumerate(idx):
        est = M.camera_w2c(torch.from_numpy(z["cam_unnorm_rots"][..., s]), torch.from_numpy(z["cam_trans"][..., s]))[0]
        gtw = M.camera_w2c(r[..., k].cpu(), t[..., k].cpu())[0]
        errs.append(_pose_err(est, gtw))
    e = np.array(errs)
    print("localise: max error %.2f mm %.3f deg; line %s" % (1e3 * e[:, 0].max(), e[:, 1].max(), line))
    assert e[:, 0].max() < 0.03 and e[:, 1].max() < 1.0
    assert line["ate_abs_m"] < 0.01 and "ate_horn_m" in line
