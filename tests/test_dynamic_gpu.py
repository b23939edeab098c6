"""GPU suite of the motion masks: csrc/dynamic.cu bit for bit against oracle/dynamic_numpy.py, argument checks, the
masked losses against the unmasked kernels and a float64 statement, and tracking / SLAM with `dynamic`."""
import math

import numpy as np
import pytest
import torch

from oracle import dynamic_numpy as O
from splatam_b200 import _lib, dynamic as D
from scenes import motion_mask_frame as _frame

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.mark.parametrize("H,W", [(1, 1), (1, 17), (17, 1), (45, 97), (192, 320), (680, 1200)])
@pytest.mark.parametrize("radius", [0, 3, 8, 13, 17])
def test_kernels_equal_the_oracle(H, W, radius):
    ds, g = _frame(H, W, seed=H * 7 + radius, objects=4)
    for cfg in (dict(D.DEFAULTS, radius=radius), dict(D.DEFAULTS, radius=radius, k_high=1.0, k_low=0.5, dilate=0)):
        dyn, inc, st = O.motion_masks(ds, g, cfg["k_high"], cfg["k_low"], cfg["r_min"], cfg["tau"], cfg["radius"],
                                      cfg["dilate"])
        gd, gi, gs = D.motion_masks(torch.from_numpy(ds).to(DEV), torch.from_numpy(g).to(DEV), cfg)
        assert np.array_equal(gd.cpu().numpy(), dyn) and np.array_equal(gi.cpu().numpy(), inc)
        assert np.array_equal(gs.cpu().numpy().view(np.uint32), st.view(np.uint32)), (gs.cpu().numpy(), st)


def _serpentine(H, W):
    """A seed block at the top left and a 1-pixel-wide serpentine of weakly occluding candidates that crosses many
    32x32 tiles: growth follows it exactly `radius` steps."""
    g = np.full((H, W), 2.0, np.float32)
    d = np.full((H, W), 2.0, np.float32)
    d[:5, :3] = 3.0                                          # strong occluders: the seed block (r = 0.5)
    path = [(2, x) for x in range(3, W - 1)]                 # row 2 to the right, down, back to the left, ...
    y, x = 2, W - 2
    while y + 4 < H:
        path += [(yy, x) for yy in range(y + 1, y + 5)]
        y += 4
        xs = range(x - 1, 0, -1) if x > W // 2 else range(x + 1, W - 1)
        path += [(y, xx) for xx in xs]
        x = xs[-1]
    for yy, xx in path:
        d[yy, xx] = 2.4                                      # weak occluders (r = 0.2)
    return np.stack([d, np.ones_like(d), d * d]), g


@pytest.mark.parametrize("radius", [8, 9, 16, 17, 40, 100])
def test_growth_along_a_long_path_crossing_tiles_equals_the_oracle(radius):
    ds, g = _serpentine(70, 45)
    cfg = dict(k_high=0.0, k_low=0.0, r_min=0.3, tau=0.05, radius=radius, dilate=0)
    dyn, _, st = O.motion_masks(ds, g, **cfg)
    gd, _, gs = D.motion_masks(torch.from_numpy(ds).to(DEV), torch.from_numpy(g).to(DEV), D.config(cfg))
    assert int(dyn.sum()) > radius                          # the path carried the growth `radius` steps
    assert np.array_equal(gd.cpu().numpy(), dyn)
    assert np.array_equal(gs.cpu().numpy().view(np.uint32), st.view(np.uint32))


def test_an_empty_keep_set_gives_zero_losses_and_gradients():
    from splatam_b200.train_ops import image_loss, masked_l1
    x, y, ds, gd, _ = _loss_inputs()
    none = torch.zeros(x.shape[1:], dtype=torch.bool, device=DEV)
    l = image_loss(x, y, keep=none)
    c, _ = masked_l1(ds, gd, depth_mean=True, keep=none)
    (l + c).backward()
    assert float(l.detach()) == 0.0 and float(c.detach()) == 0.0
    assert not x.grad.any() and not ds.grad.any()


def test_motion_masks_reject_mismatched_shapes():
    ds = torch.zeros(3, 8, 8, device=DEV)
    with pytest.raises(ValueError):
        D.motion_masks(ds, torch.zeros(1, 8, 7, device=DEV), D.DEFAULTS)
    with pytest.raises(ValueError):
        D.motion_masks(ds[:2], torch.zeros(8, 8, device=DEV), D.DEFAULTS)


def test_bad_arguments_are_rejected():
    x = torch.zeros(3, 4, 4, device=DEV)
    u = torch.zeros(16, dtype=torch.uint8, device=DEV)
    h = torch.zeros(D.BINS, dtype=torch.int32, device=DEV)
    s = torch.zeros(6, device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_residual", 0, 4, x, x, 0.99, x, h, s, device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_residual", 4096, 4096, x, x, 0.99, x, h, s, device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_scale", None, s, device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_seeds", 4, 4, x, x, x, 0.99, float("nan"), 1.0, 0.1, u, u, s, device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_grow", 4, 4, x, u, 0.05, -1, u, u.clone(), device=DEV)
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_grow", 4, 4, x, u, 0.05, 3, u, u, device=DEV)        # dyn == tmp
    with pytest.raises(_lib.SplatamB200Error):
        _lib.call("sb_dynamic_dilate", 4, 4, u, u, 65, u, u, s, device=DEV)
    for name, args in (("sb_masked_l1_keep_forward", (None, x, x, None, None, 4, 4, 0.99, 1, s)),
                       ("sb_image_loss_keep_forward", (None, x, x, 3, 4, 4, x, s))):
        with pytest.raises(_lib.SplatamB200Error):
            _lib.call(name, *args, device=DEV)


def test_masks_can_be_captured_in_a_graph():
    ds, g = _frame(97, 45, seed=3, objects=3)
    dst, gt = torch.from_numpy(ds).to(DEV), torch.from_numpy(g).to(DEV)
    cfg = dict(D.DEFAULTS, radius=11)
    ref = D.motion_masks(dst, gt, cfg)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        D.motion_masks(dst, gt, cfg)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            out = D.motion_masks(dst, gt, cfg)
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(ref, out):
        assert torch.equal(a, b)


def _loss_inputs(H=45, W=97, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(3, H, W, generator=g).to(DEV).requires_grad_(True)
    y = torch.rand(3, H, W, generator=g).to(DEV)
    ds = torch.stack([torch.rand(H, W, generator=g) + 1, torch.rand(H, W, generator=g) * 0.02 + 0.985,
                      torch.rand(H, W, generator=g)]).to(DEV).requires_grad_(True)
    gd = (torch.rand(1, H, W, generator=g) + 1).to(DEV)
    keep = (torch.rand(H, W, generator=g) < 0.7).to(DEV)
    return x, y, ds, gd, keep


def test_masked_losses_with_every_pixel_kept_return_the_unmasked_bits():
    from splatam_b200.train_ops import image_loss, masked_l1
    x, y, ds, gd, _ = _loss_inputs()
    ones = torch.ones(x.shape[1:], dtype=torch.bool, device=DEV)
    outs = []
    for keep in (None, ones):
        x.grad = ds.grad = None
        l = image_loss(x, y, keep=keep)
        l.backward()
        a, b = masked_l1(ds, gd, x, y, use_sil=True, depth_mean=False, keep=keep)
        (a + b).backward()
        c, _ = masked_l1(ds, gd, depth_mean=True, keep=keep)
        outs.append((l.detach(), a.detach(), b.detach(), c.detach(), x.grad.clone(), ds.grad.clone()))
    for u, v in zip(*outs):
        assert torch.equal(u, v)


def test_masked_losses_match_a_float64_statement_and_repeat():
    from splatam_b200.mapping import ssim_map
    from splatam_b200.train_ops import image_loss, masked_l1
    x, y, ds, gd, keep = _loss_inputs(seed=1)
    runs = []
    for _ in range(2):
        x.grad = None
        l = image_loss(x, y, keep=keep)
        l.backward()
        runs.append((l.detach().clone(), x.grad.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    xd = x.detach().double().requires_grad_(True)
    k3 = keep.expand_as(xd)
    ref = 0.8 * (xd - y.double()).abs()[k3].mean() + 0.2 * (1 - ssim_map(xd, y.double())[k3].mean())
    ref.backward()
    assert abs(float(runs[0][0]) - float(ref)) < 1e-5
    assert torch.allclose(runs[0][1].double(), xd.grad, atol=1e-7, rtol=1e-3)
    ds.grad = None
    a, _ = masked_l1(ds, gd, depth_mean=True, keep=keep)
    a.backward()
    d = ds.detach()[0:1].double()
    m = (gd > 0) & keep
    ref = (gd.double() - d).abs()[m].mean()
    assert abs(float(a) - float(ref)) < 1e-6
    assert torch.equal(ds.grad[0] != 0, m[0])


@pytest.fixture(scope="module")
def problem():
    import scenes
    import splatam_b200 as S
    from splatam_b200 import slam
    sc = scenes.config1(seed=8, P=2048, w=128, h=96)
    cam = sc.settings(S.GaussianRasterizationSettings, DEV)
    gt = {k: v.to(DEV) for k, v in sc.splatam_params(opacity_clamp=(0.9, 0.99)).items()}
    T = 8
    rots, trans = slam.look_trajectory(T, DEV, step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    for t in range(2, T):
        x = 16 + 8 * t
        frames[t]["depth"][:, 30:70, x:x + 20] *= 0.6
        frames[t]["im"][:, 30:70, x:x + 20] = 0.5
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]], device=DEV)
    return cam, frames, gt, K, rots, trans


def test_graph_and_eager_tracking_agree_with_dynamic(problem):
    from splatam_b200 import mapping as M
    cam, frames, gt, K, rots, trans = problem
    cfg = D.config(dict(refresh_every=3))
    res = []
    for graph in (False, True):
        M._TRACK_GRAPHS.clear()
        r, tr = rots.clone(), trans.clone()
        r[..., 3], tr[..., 3] = r[..., 2], tr[..., 2]
        params = dict(gt, cam_unnorm_rots=r, cam_trans=tr)
        losses = M.track_frame(params, frames[3], num_iters=12, graph=graph, dynamic=cfg)
        with torch.no_grad():               # the mask at the tracked pose (the one run_slam keeps for the frame)
            _, ds, _, _ = M._render_pair(params, frames[3], M.default_render, True, camera_grad=False)
            dyn, inc, _ = D.motion_masks(ds, frames[3]["depth"], cfg)
        res.append((r[..., 3].detach().clone(), tr[..., 3].detach().clone(), losses, dyn | inc))
    graph_mask = next(iter(M._TRACK_GRAPHS.values())).motion["exclude"]    # refreshed at iteration 9 on the device
    assert graph_mask.any() and (graph_mask ^ res[1][3]).sum() <= 0.01 * graph_mask.sum()
    # the blend backward's float atomics make any two GPU tracking runs differ in the last bits
    print("graph - eager:", (res[0][0] - res[1][0]).abs().max().item(), (res[0][1] - res[1][1]).abs().max().item(),
          np.abs(np.array(res[0][2]) - np.array(res[1][2])).max())
    assert torch.allclose(res[0][0], res[1][0], atol=1e-4) and torch.allclose(res[0][1], res[1][1], atol=1e-4)
    assert np.allclose(res[0][2], res[1][2], rtol=1e-2)
    mismatch = int((res[0][3] ^ res[1][3]).sum())
    print("graph / eager masks: %d flagged, %d differ" % (int(res[0][3].sum()), mismatch))
    assert res[0][3].any() and mismatch <= 0.01 * int(res[0][3].sum())


@pytest.mark.parametrize("graph", [False, True])
def test_nothing_flagged_equals_the_run_without_dynamic_on_the_gpu(problem, graph):
    from splatam_b200 import mapping as M, slam
    cam, frames, gt, K, _, _ = problem
    kw = dict(tracking_iters=10, mapping_iters=4, keyframe_every=2, window=3, intrinsics=K, graph=graph,
              add_new_gaussians=True)
    outs = []
    for dyn in (None, dict(k_high=math.inf, k_low=math.inf, radius=0)):
        M._TRACK_GRAPHS.clear()
        torch.manual_seed(1); np.random.seed(1)
        outs.append(slam.run_slam(dict(gt), frames, cam, dynamic=dyn, **kw))
    a, b = outs
    assert all(r["dynamic_frac"] == 0 for r in b["dynamic"])
    # the blend backward's float atomics make two GPU runs differ in the last bits (tests/test_dynamic_cpu.py holds
    # the bit-for-bit statement on the torch path), so the bound is on the trajectory and the map's size
    print("nothing flagged - off:", (a["trans"] - b["trans"]).abs().max().item(), a["counts"], b["counts"])
    assert torch.allclose(a["rots"], b["rots"], atol=1e-4) and torch.allclose(a["trans"], b["trans"], atol=1e-4)
    assert a["counts"] == b["counts"]


def test_the_occluder_stays_out_of_the_map(problem):
    from splatam_b200 import slam
    cam, frames, gt, K, _, _ = problem
    kw = dict(tracking_iters=20, mapping_iters=10, keyframe_every=2, window=3, intrinsics=K, add_new_gaussians=True)
    torch.manual_seed(1); np.random.seed(1)
    off = slam.run_slam(dict(gt), frames, cam, **kw)
    torch.manual_seed(1); np.random.seed(1)
    on = slam.run_slam(dict(gt), frames, cam, dynamic={}, **kw)
    print("gaussians off/on:", off["counts"], on["counts"])
    print("dynamic:", on["dynamic"])
    assert on["counts"][-1] < off["counts"][-1]
    for r in on["dynamic"][1:]:
        assert r["dynamic_frac"] > 0.5 * 40 * 20 / (128 * 96), r


def test_end_to_end_on_the_moving_box_and_the_static_loop(tmp_path):
    """tools/run_slam_dataset.py (Replica's settings, ICP start) with and without --dynamic on
    scenes.write_dynamic_sequence (81 frames, 1200x680; the box enters, and with present_at_start it leaves) and on
    the static loop (tools/time_dynamic.end_to_end).  Bounds from two H100 measurements recorded in DESIGN.md
    ("Moving objects"), each with its margin.  With the mask the run repeats closely (18864 / 19153 ghost Gaussians);
    without it the run fails differently each time (281072 / 162311 ghosts, ATE 0.20 / 0.73 m), so the ghost ratio
    measured 14.9x and 8.5x: bound 5x, and at most 30000 ghosts with the mask.  Recall 0.9998 (bound 0.95); flagged
    static share 0.002 (bound 0.01); ATE and static-pixel PSNR no worse than off within 2 mm / 0.5 dB (measured
    0.013 against 0.20 / 0.73 m, 38.1-38.4 against 20.6 / 24.0 dB).  Static loop: median flagged share 0 (bound
    0.01), ATE 11.1-11.5 against 11.3-11.6 mm (bound: within 20 % + 2 mm of off)."""
    from util import load
    rows = load("tools/time_dynamic.py").end_to_end(str(tmp_path), 81)
    r = {(x["case"], x["dynamic"]): x for x in rows}
    off, on = r[("enters", False)], r[("enters", True)]
    print("enters:", off, on, "\nleaves (not a bar): ghosts off %d on %d" % (r[("leaves", False)]["ghosts"],
                                                                            r[("leaves", True)]["ghosts"]))
    assert on["ghosts"] * 5 <= off["ghosts"] and on["ghosts"] <= 30000
    assert on["mask_recall"] >= 0.95 and on["static_flagged"] <= 0.01
    assert on["ate_m"] <= off["ate_m"] + 0.002
    assert on["static_psnr_db"] >= off["static_psnr_db"] - 0.5
    s_off, s_on = r[("static", False)], r[("static", True)]
    assert s_on["dynamic_frac_median"] <= 0.01
    assert s_on["ate_m"] <= 1.2 * s_off["ate_m"] + 0.002
