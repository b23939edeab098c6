"""Loop closure on the GPU (csrc/loop.cu through splatam_b200/loop.py): the deformation equals the numpy restatement
bit for bit and leaves a render unchanged when the camera moves with the map, the pose graph agrees with the oracle,
close_loop repairs a drifted map of a room the camera goes around, changes nothing when no loop closes, the captured
mapping step and the cached tracking graph read the moved map, and run_slam closes the loop of the loop sequence."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import scenes
from oracle import loop_numpy as O
from util import bits_equal

pytestmark = pytest.mark.gpu

K_LOOP = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])


def _map(P, aniso, seed, dev):
    g = torch.Generator().manual_seed(seed)
    means = torch.randn(P, 3, generator=g) * 2
    rots = torch.randn(P, 4, generator=g) * (1.0 if aniso else 0.0)
    if not aniso:
        rots[:, 0] = 1.0 + torch.rand(P, generator=g)            # unnormalised, as the mapper keeps them
    return means.to(dev), rots.to(dev)


@pytest.mark.parametrize("P,aniso", [(1, False), (1000, True), (100_003, False), (1_000_000, True)])
def test_deformation_is_bit_equal_to_the_oracle(cuda_device, P, aniso):
    from splatam_b200 import loop
    dev = cuda_device
    T = 37
    means, rots = _map(P, aniso, P, dev)
    g = torch.Generator().manual_seed(7)
    ts = torch.randint(0, T + 2, (P,), generator=g).float() - 1.0          # -1 and T: outside [0, T), unchanged
    table = np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32), (T, 1))
    rng = np.random.default_rng(P)
    for s in range(1, T, 2):                                                  # odd frames move, even ones do not
        table[s] = O.rigid(rng.normal(size=3), rng.uniform(-20, 20), rng.normal(size=3) * 0.2)[:3].reshape(12)
    m0, r0 = means.cpu().numpy(), rots.cpu().numpy()
    for flag in (0, 1):
        m, r = means.clone(), rots.clone()
        loop.deform_gaussians(m, r, ts.to(dev), torch.from_numpy(table).to(dev),
                              torch.tensor([flag], dtype=torch.int32, device=dev))
        om, orr = O.deform(m0, r0, ts.numpy(), table, flag)
        assert bits_equal(m.cpu().numpy(), om) and bits_equal(r.cpu().numpy(), orr), flag
        still = ~np.isin(ts.numpy(), np.arange(1, T, 2)) if flag else np.ones(P, bool)
        assert bits_equal(m.cpu().numpy()[still], m0[still]) and bits_equal(r.cpu().numpy()[still], r0[still])
        if flag and P > 1000:
            assert not np.array_equal(m.cpu().numpy(), m0)


def test_moving_map_and_camera_together_renders_the_same(cuda_device):
    """The whole map moved by C and the camera by C^-1 renders the same image, depth and silhouette to 1e-5 (relative
    where a value exceeds 1), except where float rounding of the camera-frame positions shows: the image and the
    silhouette may differ at up to 0.5 % of their values, where a rounded position flips one of the rasterizer's
    discrete decisions (a pixel radius, a tile, the 1/255 opacity cut-off), and the depth, which sums metres of
    camera-frame z, at up to 5 %; every difference stays below 1e-2.  Measured on an H100: 0.17 % of the image's values
    above 1e-5 (largest 3.3e-3); 3.0 % of the depth's above 1e-5 absolute (largest 5.6e-4 m)."""
    import splatam_b200 as SB
    from splatam_b200 import loop, mapping as M, slam
    dev = cuda_device
    sc = scenes.loop_room(P=100_000)
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    gt = {k: v.contiguous() for k, v in sc.splatam_params(dev).items()}
    gt["unnorm_rotations"] = F.normalize(torch.randn_like(gt["unnorm_rotations"]), dim=1) * 1.7
    gt["log_scales"] = gt["log_scales"].repeat(1, 3) + torch.randn(gt["log_scales"].shape[0], 3, device=dev) * 0.3
    rots, trans = scenes.loop_trajectory(9, dev)
    a = slam.render_frame(gt, rots, trans, 3, cam)
    C = O.rigid((0.3, 1.0, -0.2), 12.0, (0.2, -0.05, 0.1))
    table = torch.from_numpy(C[:3].reshape(1, 12).astype(np.float32)).to(dev)
    moved = {k: v.clone() for k, v in gt.items()}
    loop.deform_gaussians(moved["means3D"], moved["unnorm_rotations"], torch.zeros(moved["means3D"].shape[0],
                          device=dev), table, torch.ones(1, dtype=torch.int32, device=dev))
    r2, t2 = rots.clone(), trans.clone()
    loop.correct_cameras(r2, t2, table.repeat(9, 1), 8)
    w = M.camera_w2c(rots[..., 3], trans[..., 3])[0].double().cpu().numpy()
    w2 = M.camera_w2c(r2[..., 3], t2[..., 3])[0].double().cpu().numpy()
    assert np.abs(w2 - w @ O.inv(C)).max() < 1e-5
    b = slam.render_frame(moved, r2, t2, 3, cam)
    for k, frac in (("im", 5e-3), ("depth", 5e-2), ("sil", 5e-3)):
        d = (a[k] - b[k]).abs() / a[k].abs().clamp(min=1.0)
        print(k, "max %.3g, fraction above 1e-5: %.2e" % (float(d.max()), float((d > 1e-5).float().mean())))
        assert float((d > 1e-5).float().mean()) <= frac and float(d.max()) <= 1e-2, k


def test_pose_graph_matches_the_oracle(cuda_device):
    """Normal equations to 1e-9 relative (twice the same bits), solved poses to 1e-6, the acceptance and the
    correction table."""
    from splatam_b200 import loop
    dev = cuda_device
    est, edges, Z = O.random_graph(40, 4, 3)
    N, E = len(est), len(edges)
    W = [(2.0, 1.0) if k < N - 1 else (1.0, 3.0) for k in range(E)]
    H_o, b_o, r_o = O.normal_equations(est, edges, Z, W)
    poses = torch.tensor(np.stack([p[:3].reshape(12) for p in est]), dtype=torch.float64, device=dev)
    e_t = torch.tensor(edges, dtype=torch.int32, device=dev)
    Z_t = torch.tensor(np.stack([z[:3].reshape(12) for z in Z]), dtype=torch.float64, device=dev)
    W_t = torch.tensor(W, dtype=torch.float64, device=dev)
    outs = []
    for _ in range(2):
        n = 6 * (N - 1)
        H, b = torch.empty(n, n, dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.float64, device=dev)
        res, jac = torch.empty(E, 6, dtype=torch.float64, device=dev), torch.empty(E, 72, dtype=torch.float64,
                                                                                   device=dev)
        from splatam_b200 import _lib
        _lib.call("sb_pose_graph_normal_equations", N, E, poses, e_t, Z_t, W_t, res, jac, H, b, device=dev)
        outs.append((H.cpu().numpy(), b.cpu().numpy(), res.cpu().numpy()))
    (H, b, res), (H2, b2, res2) = outs
    assert bits_equal(H, H2) and bits_equal(b, b2)
    assert np.abs(H - H_o).max() <= 1e-9 * np.abs(H_o).max()
    assert np.abs(b - b_o).max() <= 1e-9 * np.abs(b_o).max()
    assert np.abs(res - r_o).max() <= 1e-9 * np.abs(r_o).max()
    g = loop.PoseGraph(0)
    for (i, j), z in zip(edges[:N - 1], Z[:N - 1]):
        g.add_odometry(i, j, torch.from_numpy(z))
    for (i, j), z in zip(edges[N - 1:], Z[N - 1:]):
        g.add_loop(i, j, torch.from_numpy(z))
    cfg = loop.config(dict(odometry_weights=(2.0, 1.0), loop_weights=(1.0, 3.0)))
    T = N + 3
    sol = g.solve(torch.from_numpy(np.stack(est)).to(dev), T, N - 1, cfg)
    new_o, steps_o = O.solve(est, edges, Z, W, iters=cfg["iters"])
    assert sol["steps"] == steps_o >= 1
    assert np.abs(sol["poses"].cpu().numpy() - new_o).max() <= 1e-6
    assert bool(int(sol["flag"])) == O.accept(new_o, edges, Z, 0.05, math.radians(3.0))
    table_o = O.correction_table(np.stack(est), new_o, g.frame_nodes(T, N - 1))
    assert np.abs(sol["correction_table"].cpu().numpy() - table_o).max() <= 1e-5


# ---- the mechanism: a drifted state built from a ground-truth loop ----------------------------------------------

def _setup(st, t, **cfg_kw):
    from splatam_b200 import loop
    return scenes.drifted_loop_at(st, t) + (loop.config(cfg_kw),)


def _kf_psnr(params, rots, trans, st, ids):
    from splatam_b200 import slam
    return float(np.mean([slam.psnr(slam.render_frame(params, rots, trans, k, st["cam"])["im"].clamp(0, 1),
                                    st["frames"][k]["im"].clamp(0, 1)) for k in ids]))


@pytest.fixture(scope="module")
def drifted(cuda_device):
    return scenes.drifted_loop(cuda_device)


def test_close_loop_repairs_a_drifted_room(cuda_device, drifted):
    """close_loop at the last keyframe accepts a loop to an early keyframe, lowers the ATE at least 4x and raises the
    keyframes' re-rendered PSNR against the ground-truth frames."""
    from splatam_b200 import loop, slam
    st = drifted
    t = st["T"] - 1
    mapper, kfs, graph, rots, trans, cfg = _setup(st, t)
    n = t + 1
    ate0 = slam.ate_rmse(rots[..., :n], trans[..., :n], st["rots_gt"][..., :n], st["trans_gt"][..., :n])
    p0 = _kf_psnr({k: v.detach() for k, v in mapper.g.params.items()}, rots, trans, st, st["kf_ids"])
    recs, j = loop.close_loop(t, st["frames"][t], kfs, rots, trans, graph, K_LOOP, cfg, mapper=mapper)
    print("records", recs)
    assert j is not None and recs[-1]["accepted"] and kfs[j]["id"] <= t - cfg["min_gap"]
    assert len([e for e in graph.edges if e[3] == loop.LOOP]) == 1
    ate1 = slam.ate_rmse(rots[..., :n], trans[..., :n], st["rots_gt"][..., :n], st["trans_gt"][..., :n])
    p1 = _kf_psnr({k: v.detach() for k, v in mapper.g.params.items()}, rots, trans, st, st["kf_ids"])
    print("ATE %.4f -> %.4f m, keyframe PSNR %.2f -> %.2f dB" % (ate0, ate1, p0, p1))
    assert ate1 * 4 <= ate0, (ate0, ate1)
    assert p1 > p0, (p0, p1)
    for kf in kfs:
        from splatam_b200 import mapping as M
        assert torch.allclose(kf["est_w2c"], M.camera_w2c(rots[..., kf["id"]], trans[..., kf["id"]])[0], atol=1e-5)


def _snapshot(mapper, kfs, rots, trans):
    return [mapper.g.flat.clone(), rots.clone(), trans.clone()] + [kf["est_w2c"].clone() for kf in kfs]


def test_no_closure_changes_nothing(cuda_device, drifted):
    """A trajectory that has not come back: half-way round, the camera faces the way it did at the start but is at
    least 0.55 m from every keyframe 30 or more frames old, so with max_dist 0.3 m there is no candidate and nothing
    moves.  A single plane seen twice is a candidate whose ICP is rejected: nothing moves either."""
    import splatam_b200 as SB
    from splatam_b200 import loop, mapping as M, slam
    st = drifted
    mapper, kfs, graph, rots, trans, cfg = _setup(st, 40, min_gap=30, max_dist=0.3)
    before = _snapshot(mapper, kfs, rots, trans)
    recs, j = loop.close_loop(40, st["frames"][40], kfs, rots, trans, graph, K_LOOP, cfg, mapper=mapper)
    assert recs == [] and j is None
    assert all(torch.equal(a, b) for a, b in zip(before, _snapshot(mapper, kfs, rots, trans)))
    # a wall of splats at z = 2 m filling the view, seen from frame 0 and (2 cm away) from frame 2
    dev = cuda_device
    P = 120_000
    g = torch.Generator().manual_seed(4)
    pts = torch.stack([(torch.rand(P, generator=g) - 0.5) * 6, (torch.rand(P, generator=g) - 0.5) * 4,
                       torch.full((P,), 2.0)], 1)
    sc = scenes.Scene("plane", 320, 192, 160.0, 160.0, 159.5, 95.5, pts, 0.5 + 0.4 * torch.sin(pts * 9.0),
                      torch.full((P,), 0.95), torch.full((P, 3), 0.012), torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1))
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    gt = sc.splatam_params(dev)
    r = torch.zeros(1, 4, 3, device=dev); r[:, 0] = 1.0
    tr = torch.zeros(1, 3, 3, device=dev); tr[0, :, 2] = torch.tensor([0.02, 0.0, 0.0])
    fr = [slam.render_frame(gt, r, tr, s, cam) for s in range(3)]
    for f in fr:
        f["depth"] = torch.where(f["sil"] > 0.9, f["depth"] / f["sil"].clamp(min=1e-6), torch.zeros_like(f["depth"]))
    mapper = M.ShardedMapper(gt, r, tr)
    kfs = [dict(fr[0], est_w2c=torch.eye(4, device=dev))]
    graph = loop.PoseGraph.chain([0, 2], r, tr)
    before = _snapshot(mapper, kfs, r, tr)
    recs, j = loop.close_loop(2, fr[2], kfs, r, tr, graph, K_LOOP, loop.config(dict(min_gap=1)), mapper=mapper)
    print("plane records", recs)
    assert len(recs) == 1 and not recs[0]["accepted"] and j is None
    assert all(torch.equal(a, b) for a, b in zip(before, _snapshot(mapper, kfs, r, tr)))


def test_captured_and_cached_graphs_read_the_moved_map(cuda_device, drifted):
    """After a deformation the next captured mapping step equals an eager step of the moved map (the tolerances of
    test_mapping_gpu's graph-mode test), and the cached tracking graph's first loss is the eager loss on the moved
    map, not on the old one."""
    from splatam_b200 import loop, mapping as M
    st = drifted
    dev = cuda_device
    t = st["T"] - 1
    rots, trans = st["rots"].clone(), st["trans"].clone()
    win = [dict(st["frames"][k], w2c=torch.eye(4, device=dev)) for k in (0, 5, 75, 80)]
    graph_m = M.ShardedMapper(st["drifted"], rots, trans, seed=9, timestep=st["timestep"])
    graph_m.enable_graph(win)
    graph_m.step(win)
    C = torch.from_numpy(np.tile(O.rigid((0, 1, 0), 3.0, (0.05, 0.0, -0.02))[:3].reshape(1, 12), (st["T"], 1))
                         .astype(np.float32)).to(dev)
    C[0] = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=torch.float32)
    one = torch.ones(1, dtype=torch.int32, device=dev)
    moved = {k: v.detach().clone() for k, v in graph_m.g.params.items()}
    loop.deform_gaussians(moved["means3D"], moved["unnorm_rotations"], graph_m.timestep, C, one)
    graph_m.deform(C, one)
    assert torch.equal(graph_m.g.params["means3D"], moved["means3D"])
    eager = M.ShardedMapper(moved, rots, trans, seed=9, timestep=st["timestep"])
    eager.schedule(len(win))                            # the schedule position of graph_m
    le, _, pe = eager.step(win)
    lg, _, pg = graph_m.step(win)
    assert pe == pg
    assert abs(le - float(lg)) < 1e-5 * max(1.0, abs(le)), (le, float(lg))
    ge, gg = eager.g.flat_grad, graph_m.g.flat_grad
    assert float((ge - gg).norm() / ge.norm()) < 1e-4
    # tracking: a graph cached on this map, then the map moves under it
    mapper = M.ShardedMapper(st["drifted"], rots, trans, timestep=st["timestep"])
    frame = dict(st["frames"][t], w2c=torch.eye(4, device=dev))

    def first_loss(graph):
        p = dict({k: v.detach() for k, v in mapper.g.params.items()}, cam_unnorm_rots=rots.clone(),
                 cam_trans=trans.clone())
        return M.track_frame(p, frame, num_iters=3, graph=graph)[0]
    old = first_loss(True)                              # builds and caches the tracking graph
    mapper.deform(C, one)
    cached = first_loss(None)                           # re-uses the cached graph (its key did not change)
    eager_loss = first_loss(False)
    print("tracking first loss: before %.6f, cached graph %.6f, eager %.6f" % (old, cached, eager_loss))
    assert abs(cached - eager_loss) <= 1e-4 * abs(eager_loss)
    assert abs(cached - old) > 1e-3 * abs(old)


# ---- end to end ---------------------------------------------------------------------------------------------------

def _loop_sequence(dev, T, root):
    """scenes.write_loop_sequence's frames, written under `root` and read back by datasets.RGBDSequence, and the
    ground-truth poses."""
    from splatam_b200 import datasets
    gt_w2c = scenes.write_loop_sequence(str(root / "loop"), T, dev)
    with datasets.RGBDSequence("replica", str(root), "loop", scenes.loop_data_config(), desired_height=192,
                               desired_width=320, device=dev, prefetch=2) as seq:
        assert torch.allclose(seq.intrinsics.cpu().float(), K_LOOP) and len(seq) == T
        frames = [seq[t] for t in range(T)]
        cam = seq.cam
    rots, trans = scenes.loop_trajectory(T, dev)
    from splatam_b200 import mapping as M
    assert torch.allclose(torch.stack([M.camera_w2c(rots[..., t], trans[..., t])[0].double().cpu()
                                       for t in range(T)]), gt_w2c, atol=1e-6)
    return cam, frames, rots, trans


def _run(frames, cam, **kw):
    from splatam_b200 import slam
    init, radius = slam.initialize_map(frames[0], K_LOOP)
    prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=4, removal_opacity_threshold=0.005,
                 final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
    torch.manual_seed(3); np.random.seed(3)
    kw = dict(dict(fused=True, mapping_iters=12, first_frame_iters=60, tracking_iters=40), **kw)
    return slam.run_slam(init if "resume" not in kw else None, frames, cam, intrinsics=K_LOOP, add_new_gaussians=True,
                         sil_thres=0.5, prune_dict=prune, scene_radius=radius, select_keyframes=True, window=4,
                         keyframe_every=5, pose_init="icp", **kw)


@pytest.fixture(scope="module")
def loop_seq(cuda_device, tmp_path_factory):
    return _loop_sequence(cuda_device, 81, tmp_path_factory.mktemp("loop_seq"))


def test_run_slam_closes_the_loop_sequence(cuda_device, tmp_path, loop_seq):
    """run_slam with loop closure on the loop sequence, written to disk and read back (tracking starts from ICP),
    records an accepted closure, and its ATE is within test_slam_gpu's bound and no worse than without it; a run
    resumed from a checkpoint taken after the closure ends within that bound too."""
    from splatam_b200 import formats, slam
    dev = cuda_device
    cam, frames, rots_gt, trans_gt = loop_seq
    travelled = 2 * math.pi * 0.3
    off = _run(frames, cam)
    timing = {}
    on = _run(frames, cam, loop_closure={}, timing=timing, checkpoint_dir=str(tmp_path / "ckpt"),
              checkpoint_every=78)
    ate_off = slam.ate_rmse(off["rots"], off["trans"], rots_gt, trans_gt)
    ate_on = slam.ate_rmse(on["rots"], on["trans"], rots_gt, trans_gt)
    print("loop sequence: ATE off %.4f on %.4f m, PSNR off %.2f on %.2f, loops %s, timing %s"
          % (ate_off, ate_on, off["psnr"], on["psnr"], on["loops"], timing))
    assert any(r["accepted"] for r in on["loops"] if r["frame"] <= 78)
    assert "loop_closure_s" in timing and "loops" not in off
    assert ate_on < 0.05 * travelled and ate_on <= ate_off + 0.005 * travelled, (ate_on, ate_off)
    ck = formats.load_checkpoint(str(tmp_path / "ckpt"), 78, dev)
    assert "loop_graph_edges" in ck["state"] and "keyframe_est_w2c" in ck["state"]
    res = _run(frames, cam, loop_closure={}, resume=ck)
    ate_res = slam.ate_rmse(res["rots"], res["trans"], rots_gt, trans_gt)
    print("resumed at 78: ATE %.4f m, loops %s" % (ate_res, res["loops"]))
    assert ate_res < 0.05 * travelled


@pytest.mark.parametrize("fused", [True, False])
def test_loop_closure_keeps_eager_mapping(cuda_device, loop_seq, monkeypatch, fused):
    """run_slam(loop_closure={}) with graph=False (the default) maps eagerly, fused or not: the pose graph never
    stands in for the `graph` flag of captured mapping."""
    from splatam_b200 import mapping as M
    cam, frames, _, _ = loop_seq

    def no_capture(*a, **k):
        raise AssertionError("a mapping phase was captured")
    monkeypatch.setattr(M.ShardedMapper, "enable_graph", no_capture)
    out = _run(frames[:11], cam, loop_closure={}, fused=fused, mapping_iters=2, first_frame_iters=2,
               tracking_iters=5)
    assert out["loops"] == [] and out["keyframe_time_indices"] == [0, 5, 10]


def _nccl_worker(rank, world, port, q):
    import torch.distributed as dist
    from splatam_b200 import loop, mapping as M
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    st = scenes.drifted_loop(torch.device("cuda", rank), P=100_000)
    t = st["T"] - 1
    mapper, kfs, graph, rots, trans, cfg = _setup(st, t)
    mapper.cam = dict(cam_unnorm_rots=rots, cam_trans=trans)
    recs, j = loop.close_loop(t, st["frames"][t], kfs, rots, trans, graph, K_LOOP, cfg, mapper=mapper)
    q.put((rank, j, mapper.g.flat.cpu().numpy(), mapper.cam["cam_unnorm_rots"].cpu().numpy(),
           mapper.cam["cam_trans"].cpu().numpy(), torch.stack([kf["est_w2c"] for kf in kfs]).cpu().numpy()))
    dist.destroy_process_group()


def test_replicas_stay_bit_identical_across_a_closure_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=900) for _ in range(2)], key=lambda x: x[0])
    [p.join(120) for p in procs]
    a, b = res
    assert a[1] is not None and a[1] == b[1]
    for x, y in zip(a[2:], b[2:]):
        assert bits_equal(x, y)
