"""CPU tests of the rows either side of the hot path (SURVEY.md 8(f) N3/N4): keyframe selection, checkpoint / PLY
formats, and the torch (reference-formulation) path of prune / grow -- all against fixtures produced by the
reference's own functions (tests/golden/host/make_golden_host.py)."""
import ast
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

G = np.load(os.path.join(HERE, "golden", "host", "host_ops.npz"), allow_pickle=True)
KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")


def test_keyframe_selection_matches_reference():
    from splatam_b200 import keyframes
    depth, K, w2c = (torch.from_numpy(G[k]) for k in ("kf_depth", "kf_K", "kf_w2c"))
    kfl = [{"est_w2c": torch.from_numpy(m)} for m in G["kf_list"]]
    torch.manual_seed(11); np.random.seed(12)
    sel = keyframes.keyframe_selection_overlap(depth, w2c, K, kfl, k=3, pixels=400)
    assert [int(i) for i in sel] == [int(i) for i in G["kf_selected"]]
    torch.manual_seed(11)
    valid = torch.stack(torch.where(depth[0] > 0), dim=1)
    pts = keyframes.get_pointcloud(depth, K, w2c, valid[torch.randint(valid.shape[0], (400,))])
    assert pts.shape == G["kf_pts"].shape and np.allclose(pts.numpy(), G["kf_pts"], rtol=1e-6, atol=1e-6)


def test_keyframe_selection_edge_cases():
    from splatam_b200 import keyframes
    depth, K, w2c = (torch.from_numpy(G[k]) for k in ("kf_depth", "kf_K", "kf_w2c"))
    assert keyframes.keyframe_selection_overlap(depth, w2c, K, [], k=3) == []
    behind = torch.eye(4); behind[0, 0] = behind[2, 2] = -1.0          # looks the other way: no overlap
    assert keyframes.keyframe_selection_overlap(depth, w2c, K, [{"est_w2c": behind}], k=3, pixels=200) == []
    same = [{"est_w2c": w2c.clone()} for _ in range(5)]
    sel = keyframes.keyframe_selection_overlap(depth, w2c, K, same, k=2, pixels=200)
    assert len(sel) == 2 and len(set(int(i) for i in sel)) == 2


def test_save_params_matches_reference_file(tmp_path):
    from splatam_b200 import formats
    ref = dict(np.load(os.path.join(HERE, "golden", "host", "ref_params.npz"), allow_pickle=True))
    g = torch.Generator().manual_seed(41)             # the same draws as make_golden_host.py
    params = dict(means3D=torch.randn(7, 3, generator=g), rgb_colors=torch.rand(7, 3, generator=g),
                  unnorm_rotations=torch.randn(7, 4, generator=g), logit_opacities=torch.randn(7, 1, generator=g),
                  log_scales=torch.randn(7, 1, generator=g), cam_unnorm_rots=torch.randn(1, 4, 5, generator=g),
                  cam_trans=torch.randn(1, 3, 5, generator=g), timestep=torch.arange(7).float(),
                  intrinsics=np.eye(3, dtype=np.float32), org_width=1200, org_height=680)
    path = formats.save_params({k: (torch.nn.Parameter(v) if isinstance(v, torch.Tensor) and v.dim() > 1 else v)
                                for k, v in params.items()}, str(tmp_path))
    assert os.path.basename(path) == "params.npz"
    ours = dict(np.load(path, allow_pickle=True))
    assert list(ours.keys()) == list(ref.keys())
    for k in ref:
        assert ours[k].dtype == ref[k].dtype and ours[k].shape == ref[k].shape, k
        assert np.array_equal(ours[k], ref[k]), k
    assert os.path.basename(formats.save_params_ckpt(params, str(tmp_path), 12)) == "params12.npz"
    back = formats.load_params(path, device="cpu")
    assert torch.equal(back["means3D"], params["means3D"]) and int(back["org_width"]) == 1200


def test_ply_export_layout_and_round_trip(tmp_path):
    from splatam_b200 import formats
    ref = dict(np.load(os.path.join(HERE, "golden", "host", "ref_params.npz"), allow_pickle=True))
    ply = formats.export_ply(os.path.join(HERE, "golden", "host", "ref_params.npz"), str(tmp_path / "splat.ply"))
    blob = open(ply, "rb").read()
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 7\n"
              + "".join(f"property float {a}\n" for a in formats.PLY_ATTRS) + "end_header\n").encode()
    assert blob.startswith(header) and len(blob) == len(header) + 7 * 17 * 4
    rec = np.frombuffer(blob[len(header):], dtype="<f4").reshape(7, 17)
    assert np.array_equal(rec[:, 0:3], ref["means3D"]) and np.all(rec[:, 3:6] == 0)
    assert np.array_equal(rec[:, 6:9], ((ref["rgb_colors"] - 0.5) / formats.C0).astype(np.float32))
    assert np.array_equal(rec[:, 9], ref["logit_opacities"][:, 0])
    assert all(np.array_equal(rec[:, 10 + k], ref["log_scales"][:, 0]) for k in range(3))     # isotropic -> tiled
    assert np.array_equal(rec[:, 13:17], ref["unnorm_rotations"])
    back = formats.load_ply(ply)
    assert np.allclose(back["rgb_colors"], ref["rgb_colors"], atol=1e-6)
    assert np.array_equal(back["unnorm_rotations"], ref["unnorm_rotations"])


def _mapper_after_one_step(fused, dev):
    from splatam_b200 import mapping as M
    init = {k: torch.from_numpy(G["prune_init_" + k]).to(dev) for k in KEYS}
    m = M.ShardedMapper(init, torch.zeros(1, 4, 3, device=dev), torch.zeros(1, 3, 3, device=dev),
                        lrs={k: 1e-3 for k in KEYS}, fused=fused)
    off = 0
    for k in KEYS:
        g = torch.from_numpy(G["prune_grad_" + k]).to(dev).reshape(-1)
        m.g.flat_grad[off:off + g.numel()].copy_(g)
        off += g.numel()
    m.opt.step()
    return m


@pytest.mark.parametrize("tag", ["a", "b"])
def test_prune_torch_path_matches_reference(tag):
    m = _mapper_after_one_step(False, "cpu")
    for k in KEYS:
        assert np.allclose(m.g.params[k].detach().numpy(), G[f"prune_{tag}_{k}_before"], rtol=1e-6, atol=1e-7), k
    prune_dict = ast.literal_eval(str(G[f"prune_{tag}_dict"][0]))
    P_new = m.prune_gaussians(int(G[f"prune_{tag}_iter"]), prune_dict, float(G["prune_scene_radius"]))
    assert P_new == G[f"prune_{tag}_means3D"].shape[0] and 0 < P_new < 400
    for k, (exp_avg, exp_avg_sq) in m.moments().items():
        assert np.allclose(m.g.params[k].detach().numpy(), G[f"prune_{tag}_{k}"], rtol=1e-6, atol=1e-7), k
        assert np.allclose(exp_avg.numpy(), G[f"prune_{tag}_{k}_exp_avg"], rtol=1e-6, atol=1e-9), k
        assert np.allclose(exp_avg_sq.numpy(), G[f"prune_{tag}_{k}_exp_avg_sq"], rtol=1e-6, atol=1e-12), k
    # the mapper keeps working on the smaller map: gradient views and the bucket follow the new size
    assert m.g.bucket.numel() == sum(p.numel() for p in m.g.params.values()) + P_new + 2
    m.g.flat_grad.fill_(0.5)
    m.opt.step()


def test_grow_torch_path_appends_rows_with_zero_moments():
    m = _mapper_after_one_step(False, "cpu")
    new = {k: torch.from_numpy(G["bp_iso_" + k]) for k in KEYS}
    n = new["means3D"].shape[0]
    before = {k: m.g.params[k].detach().clone() for k in KEYS}
    assert m.add_gaussians(new) == 400 + n
    for k, (exp_avg, _) in m.moments().items():
        p = m.g.params[k].detach()
        assert torch.equal(p[:400], before[k]) and torch.equal(p[400:], new[k].float().reshape(n, -1))
        assert exp_avg.shape[0] == 400 + n and float(exp_avg[400:].abs().sum()) == 0.0
        assert float(exp_avg[:400].abs().sum()) > 0.0


def test_oracle_backproject_and_prune_mask_match_reference():
    from oracle import map_ops_torch as O
    color, depth, K, w2c = (torch.from_numpy(G[k]) for k in ("bp_color", "bp_depth", "bp_K", "bp_w2c"))
    mask = torch.from_numpy(G["bp_mask"])
    for tag, sd in (("iso", 1), ("aniso", 3)):
        new, msd = O.backproject(color, depth, K, w2c, mask, scale_dim=sd)
        for k in KEYS:
            assert np.allclose(new[k].numpy(), G[f"bp_{tag}_{k}"], rtol=1e-6, atol=1e-6), (tag, k)
        assert np.allclose(msd.numpy(), G[f"bp_{tag}_mean_sq_dist"], rtol=1e-6)
    full, msd = O.backproject(color, depth, K, w2c, None)
    assert np.allclose(full["means3D"].numpy(), G["bp_full_pts"][:, :3], rtol=1e-6, atol=1e-6)
    lo, ls = torch.from_numpy(G["prune_a_logit_opacities_before"]), torch.from_numpy(G["prune_a_log_scales_before"])
    keep = O.prune_keep_mask(lo, ls, 0.05, 0.1 * 2.0)
    assert int(keep.sum()) == G["prune_a_means3D"].shape[0]


def test_operator_api_without_gaussians_needs_no_device():
    """P == 0: the reference returns zero images and R = 0 without launching (X/rasterize_points.cu:67-81); so does
    the host mirror, on any device, and the (empty) gradients come back on the inputs' device.  Both argument-check
    exceptions of the reference API fire before anything else."""
    import splatam_b200 as S
    rs = S.GaussianRasterizationSettings(8, 12, 1.0, 1.0, torch.zeros(3), 1.0, torch.eye(4)[None], torch.eye(4)[None], 0,
                                         torch.zeros(3), False)
    z = lambda *s: torch.zeros(*s, requires_grad=True)
    inp = dict(means3D=z(0, 3), means2D=z(0, 3), opacities=z(0, 1), colors_precomp=z(0, 3), scales=z(0, 3), rotations=z(0, 4))
    color, radii, depth = S.GaussianRasterizer(rs)(**inp)
    assert color.shape == (3, 8, 12) and depth.shape == (1, 8, 12) and radii.shape == (0,) and radii.dtype == torch.int32
    assert float(color.detach().abs().sum()) == 0.0
    color.sum().backward()
    assert inp["means3D"].grad.shape == (0, 3) and inp["rotations"].grad.shape == (0, 4)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        S.GaussianRasterizer(rs)(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), scales=z(1, 3), rotations=z(1, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        S.GaussianRasterizer(rs)(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3))
    with pytest.raises(S.SplatamB200Error, match="no CPU fallback"):
        S.GaussianRasterizer(rs)(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3),
                                 scales=z(1, 3), rotations=z(1, 4))


def test_pose_cache_follows_tensor_identity_and_version():
    from splatam_b200 import mapping as M
    rots = torch.zeros(1, 4, 3); rots[:, 0] = 1.0
    trans = torch.zeros(1, 3, 3)
    p = dict(means3D=torch.zeros(1, 3), cam_unnorm_rots=rots, cam_trans=trans)
    a = M.fused_pose_cached(p, 1)
    assert M.fused_pose_cached(p, 1) is a                      # same tensors, same versions -> cached
    trans[0, 0, 1] = 0.25                                      # in-place edit bumps the version
    b = M.fused_pose_cached(p, 1)
    assert b is not a and float(b[0][0, 3]) == 0.25
    p2 = dict(p, cam_trans=trans.clone())                      # another tensor object: never served from the cache
    c = M.fused_pose_cached(p2, 1)
    assert c is not b and torch.equal(c[0], b[0])
    ref = M.pose_matrices(p, 1)
    assert torch.equal(ref[0], b[0]) and torch.equal(ref[1], b[1])


def test_horn_aligned_ate_matches_reference():
    """slam.ate_horn == evaluate_ate of R/utils/eval_helpers.py:23-77 (run where the reference tree is present;
    the committed numbers below were produced by it)."""
    import torch
    from splatam_b200 import slam
    g = torch.Generator().manual_seed(4)

    def traj(n, noise):
        out = []
        for i in range(n):
            m = torch.eye(4)
            a = 0.05 * i
            m[:3, :3] = torch.tensor([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], dtype=torch.float32)
            m[:3, 3] = torch.tensor([0.1 * i, 0.02 * i * i, -0.05 * i]) + noise * torch.randn(3, generator=g)
            out.append(m)
        return out
    gt = traj(12, 0.0)
    # estimate = gt seen from a rotated / shifted frame + noise: Horn alignment must remove the rigid part
    Rz = torch.tensor([[0.8, -0.6, 0], [0.6, 0.8, 0], [0, 0, 1.0]])
    est = []
    for m in traj(12, 0.01):
        e = m.clone()
        e[:3, 3] = Rz @ m[:3, 3] + torch.tensor([1.0, -2.0, 0.5])
        est.append(e)
    ours = slam.ate_horn(gt, est)
    assert 0.002 < ours < 0.03
    assert abs(ours - 0.0127796377) < 2e-7, ours       # evaluate_ate(gt, est) of the reference on the same inputs
    import refsrc
    if refsrc.available():
        import types
        pkg = types.ModuleType("fake_rasterizer_pkg_ate")
        pkg.GaussianRasterizer, pkg.GaussianRasterizationSettings = object, object
        R = refsrc.load(pkg)
        assert abs(ours - float(R.eval_helpers.evaluate_ate(gt, est))) < 1e-6


def test_densify_matches_reference():
    """ShardedMapper.densify (torch path, CPU) == densify of R/utils/slam_external.py:191-243 on the fixture that the
    reference's own function produced (tests/golden/host/make_golden_densify.py): parameters and both Adam moments
    after an accumulate-only call and a clone + split + prune + opacity-reset call."""
    import torch
    from splatam_b200 import mapping as M
    G = np.load(os.path.join(HERE, "golden", "host", "densify.npz"))
    keys = M.GAUSSIAN_KEYS
    init = {k: torch.from_numpy(G["init_" + k]) for k in keys}
    m = M.ShardedMapper(init, torch.zeros(1, 4, 3), torch.zeros(1, 3, 3), lrs={k: 1e-3 for k in keys}, render=None, fused=False)
    for k in keys:
        m.g.params[k].grad.copy_(torch.from_numpy(G["grad_" + k]))
    m.opt.step()
    dd = eval(str(G["dict"][0]))
    for call in (0, 1):
        torch.manual_seed(70 + call)
        P = m.densify(int(G["iter_%d" % call]), dd, float(G["scene_radius"]), means2D_grad=torch.from_numpy(G["m2d_%d" % call]),
                      seen=torch.from_numpy(G["seen_%d" % call]))
    assert P == G["out_means3D"].shape[0] != 300
    for k, (exp_avg, exp_avg_sq) in m.moments().items():
        assert np.allclose(m.g.params[k].detach().numpy(), G["out_" + k], rtol=1e-6, atol=1e-7), k
        assert np.allclose(exp_avg.numpy(), G["out_" + k + "_exp_avg"], rtol=1e-6, atol=1e-9), k
        assert np.allclose(exp_avg_sq.numpy(), G["out_" + k + "_exp_avg_sq"], rtol=1e-6, atol=1e-12), k
