"""GPU parity tests of the map-maintenance kernels (csrc/map_ops.cu) through the C-ABI: prune mask, stream
compaction of the packed parameter buffer + Adam moments, add_new_gaussians' non-presence mask and the
back-projection -- against fixtures produced by the reference's own functions (tests/golden/host/host_ops.npz) and the
torch restatement oracle/map_ops_torch.py."""
import ast
import os
import sys

import numpy as np
import pytest
import torch

import scenes

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.gpu

G = np.load(os.path.join(HERE, "golden", "host", "host_ops.npz"), allow_pickle=True)
KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")


def test_compact_flat_equals_boolean_indexing(cuda_device):
    from splatam_b200 import map_ops
    dev = cuda_device
    g = torch.Generator().manual_seed(3)
    for P, widths, frac in ((100_003, [3, 3, 4, 1, 3], 0.37), (1, [3, 3, 4, 1, 1], 1.0), (4097, [5], 0.0), (777, [1, 2], 0.5)):
        flat = torch.randn(sum(widths) * P, generator=g).to(dev)
        keep = (torch.rand(P, generator=g) < frac).to(dev) if 0.0 < frac < 1.0 else torch.full((P,), frac == 1.0, device=dev)
        m8, dst, n = map_ops.compact_plan(keep)
        assert n == int(keep.sum())
        assert torch.equal(dst[:P][keep].long(), torch.arange(n, device=dev))
        out = map_ops.compact_flat(flat, P, widths, m8, dst, n)
        parts, off = [], 0
        for w in widths:
            parts.append(flat[off:off + w * P].view(P, w)[keep].reshape(-1))
            off += w * P
        assert torch.equal(out, torch.cat(parts))
    m8, dst, n = map_ops.compact_plan(torch.zeros(0, dtype=torch.bool, device=dev))
    assert n == 0


def test_prune_mask_equals_torch(cuda_device):
    from oracle import map_ops_torch as O
    from splatam_b200 import map_ops
    dev = cuda_device
    g = torch.Generator().manual_seed(4)
    for sd in (1, 3):
        lo = (4.0 * torch.randn(200_000, 1, generator=g)).to(dev)
        ls = torch.log(0.01 + 0.5 * torch.rand(200_000, sd, generator=g)).to(dev)
        for thr, big in ((0.005, None), (0.05, 0.2), (0.5, 0.45)):
            assert torch.equal(map_ops.prune_mask(lo, ls, thr, big), O.prune_keep_mask(lo, ls, thr, big)), (sd, thr, big)


def _fused_mapper_after_one_step(dev):
    from splatam_b200 import mapping as M
    init = {k: torch.from_numpy(G["prune_init_" + k]).to(dev) for k in KEYS}
    m = M.ShardedMapper(init, torch.zeros(1, 4, 3, device=dev), torch.zeros(1, 3, 3, device=dev),
                        lrs={k: 1e-3 for k in KEYS}, fused=True)
    off = 0
    for k in KEYS:
        g = torch.from_numpy(G["prune_grad_" + k]).to(dev).reshape(-1)
        m.g.flat_grad[off:off + g.numel()].copy_(g)
        off += g.numel()
    m.opt.step()
    return m


@pytest.mark.parametrize("tag", ["a", "b"])
def test_prune_fused_path_matches_reference(cuda_device, tag):
    m = _fused_mapper_after_one_step(cuda_device)
    prune_dict = ast.literal_eval(str(G[f"prune_{tag}_dict"][0]))
    P_new = m.prune_gaussians(int(G[f"prune_{tag}_iter"]), prune_dict, float(G["prune_scene_radius"]))
    assert P_new == G[f"prune_{tag}_means3D"].shape[0]
    off = 0
    for k, (exp_avg, exp_avg_sq) in m.moments().items():
        ref = G[f"prune_{tag}_{k}"]
        assert np.allclose(m.g.params[k].detach().cpu().numpy(), ref, rtol=2e-6, atol=1e-7), k
        assert np.allclose(exp_avg.cpu().numpy().reshape(ref.shape), G[f"prune_{tag}_{k}_exp_avg"], rtol=2e-6, atol=1e-9), k
        assert np.allclose(exp_avg_sq.cpu().numpy().reshape(ref.shape), G[f"prune_{tag}_{k}_exp_avg_sq"], rtol=2e-6, atol=1e-12), k
        off += ref.size
    assert m.opt.t == 1 and m.opt.m.numel() == m.g.flat.numel() == off
    m.g.flat_grad.fill_(0.5)
    m.opt.step()                                   # the fused optimizer keeps working on the compacted buffers
    assert torch.isfinite(m.g.flat).all()


def test_backproject_matches_reference_golden(cuda_device):
    from splatam_b200 import map_ops
    dev = cuda_device
    color, depth, w2c = (torch.from_numpy(G[k]).to(dev) for k in ("bp_color", "bp_depth", "bp_w2c"))
    K, mask = torch.from_numpy(G["bp_K"]), torch.from_numpy(G["bp_mask"]).to(dev)
    for tag, sd in (("iso", 1), ("aniso", 3)):
        new, msd = map_ops.backproject(color, depth, K, w2c, mask=mask, scale_dim=sd)
        for k in KEYS:
            a, b = new[k].cpu().numpy(), G[f"bp_{tag}_{k}"]
            assert a.shape == b.shape and np.allclose(a, b, rtol=2e-6, atol=2e-6), (tag, k, np.abs(a - b).max())
        assert np.allclose(msd.cpu().numpy(), G[f"bp_{tag}_mean_sq_dist"], rtol=1e-6)
    full, msd = map_ops.backproject(color, depth, K, w2c, mask=None)
    assert np.allclose(full["means3D"].cpu().numpy(), G["bp_full_pts"][:, :3], rtol=2e-6, atol=2e-6)
    assert np.array_equal(full["rgb_colors"].cpu().numpy(), G["bp_full_pts"][:, 3:6])
    assert np.allclose(msd.cpu().numpy(), G["bp_full_mean_sq_dist"], rtol=1e-6)


def _slam_problem(dev, P=30_000):
    import splatam_b200 as S
    sc = scenes.room(seed=33, P=P, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gauss = sc.splatam_params()
    gauss = {k: v.to(dev).contiguous() for k, v in gauss.items()}
    K = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])
    return sc, cam, gauss, K


def test_non_presence_mask_and_add_new_gaussians(cuda_device):
    from oracle import map_ops_torch as O
    from splatam_b200 import map_ops, mapping as M, slam
    dev = cuda_device
    sc, cam, gauss, K = _slam_problem(dev)
    rots, trans = slam.look_trajectory(3, dev)
    frame = slam.render_frame(gauss, rots, trans, 2, cam)                  # observation from the full scene
    part = {k: v[gauss["means3D"][:, 0] < 0.3].contiguous() for k, v in gauss.items()}     # the map misses a slab
    m = M.ShardedMapper(part, rots, trans, fused=True)
    P0 = m.g.shapes["means3D"][0]
    p = m.params()
    with torch.no_grad():
        tg = M.transform_to_frame(p, 2, gaussians_grad=False, camera_grad=False)
        depth_sil, _, _ = M.default_render(cam, **M.depth_sil_rendervar(p, frame["w2c"], tg))
    ref_mask = O.non_presence_mask(depth_sil, frame["depth"], 0.5)
    err = map_ops.depth_error(depth_sil, frame["depth"])
    assert torch.equal(err, O.depth_error(depth_sil, frame["depth"]))
    mask = map_ops.new_gaussian_mask(depth_sil, frame["depth"], 0.5, 50.0 * float(err.median()))
    assert torch.equal(mask, ref_mask) and 0 < int(mask.sum()) < mask.numel()
    curr_w2c = torch.eye(4, device=dev)
    curr_w2c[:3, :3] = M.build_rotation(torch.nn.functional.normalize(rots[..., 2]))[0]
    curr_w2c[:3, 3] = trans[0, :, 2]
    ref_new, _ = O.backproject(frame["im"], frame["depth"], K.to(dev), curr_w2c, ref_mask, scale_dim=1)
    n = m.add_new_gaussians(frame, 2, K, sil_thres=0.5)
    assert n == int(ref_mask.sum()) and m.g.shapes["means3D"][0] == P0 + n
    for k in KEYS:
        a, b = m.g.params[k].detach()[P0:], ref_new[k]
        assert torch.allclose(a, b, rtol=2e-6, atol=2e-6), (k, float((a - b).abs().max()))
        assert torch.equal(m.g.params[k].detach()[:P0], part[k].reshape(P0, -1))
    assert all(float(exp_avg.abs().sum()) == 0.0 for exp_avg, _ in m.moments().values())
    assert m.opt.m.numel() == m.g.flat.numel()
    # the grown map covers the frame: the silhouette hole is (mostly) gone, and mapping steps still run
    p = m.params()
    with torch.no_grad():
        tg = M.transform_to_frame(p, 2, gaussians_grad=False, camera_grad=False)
        ds2, _, _ = M.default_render(cam, **M.depth_sil_rendervar(p, frame["w2c"], tg))
    assert int(O.non_presence_mask(ds2, frame["depth"], 0.5).sum()) < 0.2 * n
    loss0, _, _ = m.step([frame])
    m.enable_graph([frame])
    for _ in range(3):
        loss, _, _ = m.step([frame])
    assert np.isfinite(float(loss)) and float(loss) <= float(loss0) * 1.05
    P1 = m.prune_gaussians(20, dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=20,
                                    removal_opacity_threshold=0.005, final_removal_opacity_threshold=0.6,
                                    reset_opacities=False, reset_opacities_every=500), scene_radius=3.0)
    assert 0 < P1 < P0 + n and m._graph is None      # the opacity-0.5 newcomers go
    loss, _, _ = m.step([frame])                      # eager again after the shape change
    assert np.isfinite(float(loss))


def test_densify_fused_path_matches_torch_path_and_reference_fixture(cuda_device):
    """densify over the packed buffer + fused Adam moments (compaction kernels) == the torch path on the GPU == the
    reference's own densify (fixture tests/golden/host/densify.npz, generated on the CPU: torch.normal draws differ
    between CPU and CUDA generators, so the split samples are compared fused-vs-torch with a shared CUDA generator and
    the reference fixture pins everything that does not depend on them: the final count)."""
    from splatam_b200 import mapping as M
    dev = cuda_device
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host", "densify.npz"))
    keys = M.GAUSSIAN_KEYS
    dd = eval(str(G["dict"][0]))
    res = {}
    for fused in (True, False):
        init = {k: torch.from_numpy(G["init_" + k]).to(dev) for k in keys}
        m = M.ShardedMapper(init, torch.zeros(1, 4, 3, device=dev), torch.zeros(1, 3, 3, device=dev),
                            lrs={k: 1e-3 for k in keys}, fused=fused)
        for k in keys:
            m.g.params[k].grad.copy_(torch.from_numpy(G["grad_" + k]).to(dev))
        m.opt.step()
        gen = torch.Generator(device=dev); gen.manual_seed(5)
        for call in (0, 1):
            P = m.densify(int(G["iter_%d" % call]), dd, float(G["scene_radius"]),
                          means2D_grad=torch.from_numpy(G["m2d_%d" % call]).to(dev),
                          seen=torch.from_numpy(G["seen_%d" % call]).to(dev), generator=gen)
        mom = m.moments()
        res[fused] = (P, {k: m.g.params[k].detach().clone() for k in keys},
                      {k: mom[k][0].clone() for k in keys}, {k: mom[k][1].clone() for k in keys})
    assert res[True][0] == res[False][0] == G["out_means3D"].shape[0]
    for k in keys:
        for i in (1, 2, 3):
            assert torch.allclose(res[True][i][k], res[False][i][k], rtol=2e-6, atol=1e-9), (k, i)
