"""Loop closure without a GPU: the numpy restatement of the pose graph (oracle/loop_numpy.py) has the Jacobians of its
residuals, leaves a consistent graph exactly where it is and spreads a loop's drift over a circle of keyframes; the
frame-to-node rule, the checkpoint arrays of the graph, the C-ABI argument checks, the refusal of CPU tensors and of
bad `loop_closure` settings, and a default run that never reaches the loop module."""
import ctypes
import io
import math
import sys

import numpy as np
import pytest
import torch

import scenes
from oracle import loop_numpy as O
from util import bits_equal, cpu_render
from splatam_b200 import _lib, loop, slam


def _rand_pose(rng, rot=0.5, trans=1.0):
    return O.exp_se3(np.concatenate([rng.normal(size=3) * rot, rng.normal(size=3) * trans]))


def test_jacobians_match_finite_differences():
    """d r / d xi_i and d r / d xi_j of r = log(Z T_i T_j^-1) against central differences of the perturbed poses
    exp(d) T, for residuals of up to a few degrees and centimetres (the series of Jl^-1 stops at the second order)."""
    rng = np.random.default_rng(5)
    for _ in range(20):
        Ti, Tj = _rand_pose(rng), _rand_pose(rng)
        Z = O.exp_se3(rng.normal(size=6) * 0.03) @ Tj @ O.inv(Ti)
        r, Ai, Aj = O.edge_terms(Ti, Tj, Z)
        assert np.linalg.norm(r) > 1e-3
        for which, A in ((0, Ai), (1, Aj)):
            fd = np.zeros((6, 6))
            for k in range(6):
                d = np.zeros(6)
                d[k] = 1e-6
                a = [Ti, Tj]
                b = [Ti, Tj]
                a[which] = O.exp_se3(d) @ a[which]
                b[which] = O.exp_se3(-d) @ b[which]
                fd[:, k] = (O.edge_terms(*a, Z)[0] - O.edge_terms(*b, Z)[0]) / 2e-6
            assert np.abs(fd - A).max() <= 1e-5, (which, np.abs(fd - A).max())


def _chain(poses, loops=()):
    """Odometry edges between consecutive poses measured exactly, plus loop edges (i, j, Z)."""
    edges = [(k - 1, k) for k in range(1, len(poses))]
    Z = [poses[k] @ O.inv(poses[k - 1]) for k in range(1, len(poses))]
    for i, j, z in loops:
        edges.append((i, j))
        Z.append(z)
    return edges, Z


def test_consistent_graph_is_a_fixed_point():
    """Measurements that the poses satisfy: no step is applied, every correction is the identity bit for bit and node
    0 never moves."""
    rng = np.random.default_rng(2)
    poses = [np.eye(4)] + [_rand_pose(rng) for _ in range(7)]
    edges, Z = _chain(poses, [(1, 7, poses[7] @ O.inv(poses[1]))])
    new, steps = O.solve(poses, edges, Z, [(1.0, 1.0)] * len(edges))
    assert steps == 0
    assert bits_equal(new, np.stack(poses))
    table = O.correction_table(np.stack(poses), new, list(range(8)) + [-1, -1])
    assert bits_equal(table, np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32), (10, 1)))
    assert O.accept(new, edges, Z, 1e-9, 1e-6)          # an angle from arccos resolves ~1e-8 rad near 0


def _circle(K, radius=2.0):
    """w2c of K cameras on a circle, each looking at its centre."""
    out = []
    for k in range(K):
        a = 2 * math.pi * k / K
        c = np.array([radius * math.sin(a), 0.0, radius * (1 - math.cos(a))])
        fwd = np.array([0.0, 0.0, radius]) - c
        fwd /= np.linalg.norm(fwd)
        right = np.cross(fwd, [0.0, 1.0, 0.0])
        right /= np.linalg.norm(right)
        R = np.stack([right, np.cross(fwd, right), fwd])
        w2c = np.eye(4)
        w2c[:3, :3], w2c[:3, 3] = R, -R @ c
        out.append(w2c)
    return out


def test_uniform_drift_is_spread_over_the_loop():
    """A circle of 24 keyframes whose estimate drifts uniformly -- the world moves by the same small rigid motion
    (0.1 degree about the vertical and 9 mm) at every keyframe, so the odometry carries it -- and one exact loop edge
    from the last keyframe back to the first: the solve cuts the worst camera-centre error at least 4x and every edge
    then passes the residual test."""
    gt = _circle(24)
    drift = O.exp_se3(np.array([0.0005, 0.001, 0.0, 0.008, -0.002, 0.004]))
    est = [gt[k] @ np.linalg.matrix_power(drift, k) for k in range(24)]
    edges, Z = _chain(est, [(0, 23, gt[23] @ O.inv(gt[0]))])
    centre = lambda p: -p[:3, :3].T @ p[:3, 3]
    worst = lambda ps: max(np.linalg.norm(centre(p) - centre(g)) for p, g in zip(ps, gt))
    new, steps = O.solve(est, edges, Z, [(1.0, 1.0)] * len(edges))
    before, after = worst(est), worst(new)
    assert steps >= 1 and np.array_equal(new[0], est[0])
    assert after * 4 <= before, (before, after)
    assert O.accept(new, edges, Z, 0.05, math.radians(3.0))


def test_frame_to_node_attachment():
    """Frame s <= t belongs to the first node at or after it, so frames t-1 and t share one correction; frames after t
    take none."""
    g = loop.PoseGraph(0)
    for k in (5, 10, 15):
        g.add_odometry(g.nodes()[-1], k, torch.eye(4, dtype=torch.float64))
    fn = g.frame_nodes(20, 15)
    assert fn[0] == 0
    assert fn[1:6] == [1] * 5 and fn[6:11] == [2] * 5 and fn[11:16] == [3] * 5
    assert fn[16:] == [-1] * 4
    assert fn[14] == fn[15]
    with pytest.raises(ValueError):
        g.add_odometry(10, 20, torch.eye(4))
    with pytest.raises(ValueError):
        g.add_loop(0, 7, torch.eye(4))


def test_sidecar_round_trips_the_edges():
    rng = np.random.default_rng(9)
    g = loop.PoseGraph(0)
    for k in (4, 8, 12):
        g.add_odometry(g.nodes()[-1], k, torch.from_numpy(_rand_pose(rng)))
    g.add_loop(0, 12, torch.from_numpy(_rand_pose(rng)))
    buf = io.BytesIO()
    np.savez(buf, **g.state())
    buf.seek(0)
    h = loop.PoseGraph.from_state(dict(np.load(buf)))
    assert h.nodes() == g.nodes() == [0, 4, 8, 12]
    assert len(h.edges) == 4
    for a, b in zip(g.edges, h.edges):
        assert a[:2] == b[:2] and a[3] == b[3]
        assert torch.equal(torch.as_tensor(a[2], dtype=torch.float64), b[2])


def test_abi_argument_checks():
    lib = _lib.load()
    d = 1                                                          # non-null dummy pointers, never dereferenced
    assert lib.sb_deform_gaussians(-1, d, d, d, 4, d, d, None) == 1
    assert lib.sb_deform_gaussians(10, d, d, d, 0, d, d, None) == 1
    assert lib.sb_deform_gaussians(10, None, d, d, 4, d, d, None) == 1
    assert lib.sb_deform_gaussians(10, d, d, d, 4, d, None, None) == 1
    assert lib.sb_deform_gaussians(0, None, None, None, 4, d, d, None) == 0      # an empty map: nothing to launch
    ne = lambda **kw: [kw.get(k, v) for k, v in dict(N=5, E=4, poses=d, edges=d, Z=d, w=d, res=d, jac=d, H=d, b=d,
                                                      stream=None).items()]
    assert lib.sb_pose_graph_normal_equations(*ne(N=1)) == 1
    assert lib.sb_pose_graph_normal_equations(*ne(E=0)) == 1
    assert lib.sb_pose_graph_normal_equations(*ne(H=None)) == 1
    assert lib.sb_pose_graph_normal_equations(*ne(edges=None)) == 1
    up = lambda **kw: [kw.get(k, v) for k, v in dict(N=5, E=4, T=20, poses=d, old=d, xi=d, edges=d, Z=d, fn=d, m=0.05,
                                                      rad=0.05, table=d, flag=d, err=d, stream=None).items()]
    assert lib.sb_pose_graph_update(*up(N=1)) == 1
    assert lib.sb_pose_graph_update(*up(T=0)) == 1
    assert lib.sb_pose_graph_update(*up(m=-1.0)) == 1
    assert lib.sb_pose_graph_update(*up(rad=float("nan"))) == 1
    assert lib.sb_pose_graph_update(*up(flag=None)) == 1


def test_cpu_tensors_raise():
    P, T = 8, 4
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        loop.deform_gaussians(torch.zeros(P, 3), torch.zeros(P, 4), torch.zeros(P), torch.zeros(T, 12),
                              torch.ones(1, dtype=torch.int32))
    frame = dict(depth=torch.ones(1, 8, 8))
    rots = torch.zeros(1, 4, 100)
    rots[:, 0] = 1
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        loop.candidates(frame, 90, [dict(id=0)], rots, torch.zeros(1, 3, 100), torch.eye(3), loop.config({}))


def _cpu_run(**kw):
    import splatam_b200 as SB
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(SB.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(3, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(3)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    torch.manual_seed(1); np.random.seed(1)
    return slam.run_slam(gt, frames, cam, render=cpu_render, fused=False, tracking_iters=2, mapping_iters=1,
                         keyframe_every=1, window=2, intrinsics=K, **kw)


@pytest.mark.parametrize("bad", [dict(min_gap=0), dict(max_dist=-1.0), dict(max_angle=200.0), dict(points=1.5),
                                 dict(min_overlap=1.5), dict(max_correction=(0.3,)), dict(loop_weights=(1.0, 0.0)),
                                 dict(iters=True), dict(max_rms=float("nan")), dict(unknown_key=1)])
def test_bad_loop_closure_settings_raise(bad):
    with pytest.raises(ValueError, match="loop_closure"):
        loop.config(bad)
    with pytest.raises(ValueError, match="loop_closure"):
        _cpu_run(loop_closure=bad)


def test_loop_closure_needs_cuda():
    assert loop.config({}) == dict(loop.DEFAULTS)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        _cpu_run(loop_closure={})
    with pytest.raises(ValueError, match="loop_closure"):
        _cpu_run(loop_closure=[("min_gap", 10)])


def test_default_run_never_reaches_the_loop_module(monkeypatch):
    """loop_closure=None: importing splatam_b200.loop would fail, and the run is the default's."""
    torch.set_num_threads(4)
    a = _cpu_run()
    monkeypatch.delattr(sys.modules["splatam_b200"], "loop", raising=False)
    monkeypatch.setitem(sys.modules, "splatam_b200.loop", None)
    b = _cpu_run(loop_closure=None)
    assert "loops" not in a and "loops" not in b
    for k in ("rots", "trans"):
        assert bits_equal(a[k].numpy(), b[k].numpy()), k
    for k in a["gauss"]:
        assert bits_equal(a["gauss"][k].numpy(), b["gauss"][k].numpy()), k
