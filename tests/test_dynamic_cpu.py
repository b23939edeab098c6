"""CPU suite of the motion masks (splatam_b200/dynamic.py): the numpy oracle against a plain breadth-first statement
of the growth rule, the torch statement against the oracle bit for bit, the scale against a sort, the options and
run_slam's behaviour with `dynamic` on the torch path."""
import collections
import math

import numpy as np
import pytest
import torch

import scenes
from oracle import dynamic_numpy as O
from splatam_b200 import dynamic as D

CFG = dict(k_high=3.0, k_low=1.2, r_min=0.05, tau=0.05, radius=5, dilate=1, refresh_every=1)


def _frame(H, W, seed, objects=2):
    return scenes.motion_mask_frame(H, W, seed, objects)


def _bfs(ds, g, cfg, sil=0.99):
    """The growth rule as a breadth-first search: pixels within `radius` 4-connected steps of a kept occ seed through
    candidates, each step depth-continuous; then the Chebyshev dilation."""
    r, valid, scale = O.scale_of(ds, g, sil)
    H, W = g.shape
    s = ds[1]
    f = np.float32
    hi = O._threshold(cfg["k_high"], scale, f(cfg["r_min"]))
    lo = O._threshold(cfg["k_low"], scale, f(cfg["r_min"]) * f(0.5))
    with np.errstate(invalid="ignore"):
        occ_raw = valid & (r > hi)
        cand = (g > 0) & ((valid & (r > lo)) | (s <= f(sil)))

    def kept(y, x):
        if not occ_raw[y, x]:
            return False
        n = sum(occ_raw[y + a, x + b] for a in (-1, 0, 1) for b in (-1, 0, 1)
                if (a or b) and 0 <= y + a < H and 0 <= x + b < W)
        return n >= 4

    dist = np.full((H, W), -1)
    q = collections.deque()
    for y in range(H):
        for x in range(W):
            if kept(y, x):
                dist[y, x] = 0
                q.append((y, x))
    while q:
        y, x = q.popleft()
        if dist[y, x] == cfg["radius"]:
            continue
        for a, b in ((-1, 0), (1, 0), (0, -1), (0, 1)):
            yy, xx = y + a, x + b
            if 0 <= yy < H and 0 <= xx < W and dist[yy, xx] < 0 and cand[yy, xx]:
                if abs(g[y, x] - g[yy, xx]) <= f(cfg["tau"]) * min(g[y, x], g[yy, xx]):
                    dist[yy, xx] = dist[y, x] + 1
                    q.append((yy, xx))
    grown = dist >= 0
    return O._dilate(grown, cfg["dilate"])


SIZES = [(1, 1), (1, 17), (17, 1), (9, 13), (24, 31), (45, 97)]


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_equals_bfs_and_torch_equals_oracle(H, W, seed):
    ds, g = _frame(H, W, seed)
    for cfg in (CFG, dict(CFG, radius=0, dilate=0), dict(CFG, radius=11, dilate=2, k_high=1.0, k_low=0.5)):
        dyn, inc, st = O.motion_masks(ds, g, cfg["k_high"], cfg["k_low"], cfg["r_min"], cfg["tau"], cfg["radius"],
                                      cfg["dilate"])
        assert np.array_equal(dyn, _bfs(ds, g, cfg))
        tdyn, tinc, tst = D.motion_masks_torch(torch.from_numpy(ds), torch.from_numpy(g), D.config(cfg))
        assert np.array_equal(tdyn.numpy(), dyn) and np.array_equal(tinc.numpy(), inc)
        assert np.array_equal(tst.numpy().view(np.uint32), st.view(np.uint32))


def test_path_of_exactly_radius_steps_and_a_depth_step():
    """A seed block at the left of a 1-pixel-high strip of weakly occluding candidates: growth reaches exactly
    `radius` pixels; a depth step beyond tau stops it."""
    H, W, rad = 5, 40, 7
    g = np.full((H, W), 2.0, np.float32)
    d = np.full((H, W), 2.0, np.float32)
    d[:, :3] = 3.0                                          # strong occluders: a 5x3 seed block
    d[2, 3:] = 2.4                                          # weak occluders along row 2 (r = 0.2)
    s = np.ones((H, W), np.float32)
    ds = np.stack([d, s, d * d])
    cfg = dict(k_high=0.0, k_low=0.0, r_min=0.3, tau=0.05, radius=rad, dilate=0)
    dyn, _, _ = O.motion_masks(ds, g, **cfg)
    assert dyn[2, :3 + rad].all()
    assert int(np.nonzero(dyn[2])[0].max()) == 2 + rad       # exactly radius steps from the seed at column 2
    dyn1, _, _ = O.motion_masks(ds, g, **dict(cfg, radius=rad + 1))
    assert int(np.nonzero(dyn1[2])[0].max()) == 3 + rad
    g2 = g.copy()
    g2[2, 6:] = 1.0                                          # a depth step at column 6
    dyn2, _, _ = O.motion_masks(np.stack([d, s, d * d]), g2, **dict(cfg, radius=rad + 1))
    assert int(np.nonzero(dyn2[2])[0].max()) == 5
    for x in (dyn, dyn1, dyn2):
        t, _, _ = D.motion_masks_torch(torch.from_numpy(ds), torch.from_numpy(g if x is not dyn2 else g2),
                                       D.config(dict(cfg, radius=rad + (x is not dyn))))
        assert np.array_equal(t.numpy(), x)


def test_residual_exactly_at_the_threshold_is_not_a_seed():
    H, W = 6, 6
    g = np.full((H, W), 2.0, np.float32)
    d = np.full((H, W), 2.0, np.float32)
    d[1:5, 1:5] = 2.5                       # r = 0.25 exactly
    ds = np.stack([d, np.ones_like(d), d * d])
    at, _, _ = O.motion_masks(ds, g, 0.0, 0.0, 0.25, 0.05, 0, 0)
    below, _, _ = O.motion_masks(ds, g, 0.0, 0.0, 0.2499, 0.05, 0, 0)
    assert not at.any() and below.sum() == 16 - 4         # the block's corners have 3 seed neighbours
    t, _, _ = D.motion_masks_torch(torch.from_numpy(ds), torch.from_numpy(g),
                                   D.config(dict(k_high=0.0, k_low=0.0, r_min=0.25, radius=0, dilate=0)))
    assert not t.any()


@pytest.mark.parametrize("seed", range(6))
def test_scale_is_the_top_16_bits_of_the_sorted_lower_median(seed):
    ds, g = _frame(23, 31, seed)
    r, valid, scale = O.scale_of(ds, g)
    a = np.sort(np.abs(r[valid]))
    med = a[(len(a) - 1) // 2]
    assert scale.view(np.uint32) == (med.view(np.uint32) >> 16) << 16
    _, _, st = D.motion_masks_torch(torch.from_numpy(ds), torch.from_numpy(g), D.config({}))
    assert st[1].numpy().view(np.uint32) == scale.view(np.uint32) and st[0] == valid.sum()


def test_config_rejects_bad_values():
    assert D.config({}) == D.DEFAULTS
    assert D.config(dict(k_high=math.inf))["k_high"] == math.inf
    for bad in (dict(foo=1), dict(k_high=float("nan")), dict(k_low=-1), dict(r_min=math.inf), dict(tau=-0.1),
                dict(radius=-1), dict(radius=1.5), dict(dilate=65), dict(refresh_every=0), dict(radius=True)):
        with pytest.raises(ValueError):
            D.config(bad)
    with pytest.raises(ValueError):
        D.config(None)


# ---- run_slam with `dynamic` on the torch path ----------------------------------------------------------------------
T = 6


@pytest.fixture(scope="module")
def problem():
    import scenes
    import splatam_b200 as S
    from splatam_b200 import slam
    from util import cpu_render
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=1024, w=64, h=64)          # dense enough that the map covers every pixel
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.9, 0.99))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    for t in range(2, T):         # a flat occluder 40 % nearer than the scene, moving right 4 px per frame
        x = 8 + 4 * t
        frames[t]["depth"][:, 20:40, x:x + 12] *= 0.6
        frames[t]["im"][:, 20:40, x:x + 12] = 0.5
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    kw = dict(render=cpu_render, fused=False, tracking_iters=10, mapping_iters=2, keyframe_every=2, window=3,
              intrinsics=K)
    return cam, frames, dict(gt), kw


def test_nothing_flagged_equals_the_run_without_dynamic(problem):
    from splatam_b200 import slam
    cam, frames, init, kw = problem
    torch.manual_seed(1); np.random.seed(1)
    ref = slam.run_slam(init, frames, cam, **kw)
    torch.manual_seed(1); np.random.seed(1)
    out = slam.run_slam(init, frames, cam, dynamic=dict(k_high=math.inf, k_low=math.inf, radius=0), **kw)
    assert all(r["dynamic_frac"] == 0.0 and r["inconsistent_frac"] == 0.0 for r in out["dynamic"])
    assert [r["frame"] for r in out["dynamic"]] == list(range(1, T))
    assert torch.equal(ref["rots"], out["rots"]) and torch.equal(ref["trans"], out["trans"])
    for k in ref["gauss"]:
        assert torch.equal(ref["gauss"][k], out["gauss"][k]), k
    assert ref["psnr"] == out["psnr"]


@pytest.fixture(scope="module")
def dyn_run(problem, tmp_path_factory):
    from splatam_b200 import slam
    cam, frames, init, kw = problem
    d = str(tmp_path_factory.mktemp("ckpt"))
    torch.manual_seed(1); np.random.seed(1)
    return slam.run_slam(init, frames, cam, checkpoint_dir=d, checkpoint_every=2, dynamic=dict(radius=4), **kw), d


def test_the_occluder_is_flagged_and_kept_out_of_the_keyframes(dyn_run):
    out, _ = dyn_run
    fr = {r["frame"]: r for r in out["dynamic"]}
    assert fr[1]["dynamic_frac"] == 0.0
    for t in range(2, T):
        assert fr[t]["dynamic_frac"] > 0.5 * (20 * 12) / 64 ** 2, fr[t]
    masks = dict(zip(out["keyframe_time_indices"], out["keyframe_dynamic"]))
    for t in (2, 4):
        box = np.zeros((64, 64), bool)
        box[20:40, 8 + 4 * t:20 + 4 * t] = True
        m = masks[t].numpy()
        assert (m & box).sum() == box.sum() and (m & ~box).sum() <= 24 * 16 - 20 * 12     # the box and its dilate=2 ring


def test_exact_resume_with_dynamic(problem, dyn_run):
    from splatam_b200 import formats, slam
    cam, frames, _, kw = problem
    out, d = dyn_run
    torch.manual_seed(77); np.random.seed(77)
    ckpt = formats.load_checkpoint(d, 2, "cpu")
    res = slam.run_slam(None, frames, cam, resume=ckpt, dynamic=dict(radius=4), **kw)
    assert torch.equal(out["rots"], res["rots"]) and torch.equal(out["trans"], res["trans"])
    for k in out["gauss"]:
        assert torch.equal(out["gauss"][k], res["gauss"][k]), k
    for a, b in zip(out["keyframe_dynamic"], res["keyframe_dynamic"]):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):            # a checkpoint of a run without masks
        slam.run_slam(None, frames, cam, resume=dict(ckpt, state={k: v for k, v in ckpt["state"].items()
                                                                  if not k.startswith("keyframe_dynamic")}),
                      dynamic={}, **kw)


def test_dynamic_with_relocalise_or_bad_options_raises(problem):
    from splatam_b200 import slam
    cam, frames, init, kw = problem
    with pytest.raises(ValueError):
        slam.run_slam(init, frames, cam, dynamic={}, relocalise={}, **kw)
    with pytest.raises(ValueError):
        slam.run_slam(init, frames, cam, dynamic=dict(radius=-1), **kw)


def test_dynamic_npz_round_trips(dyn_run, tmp_path):
    from splatam_b200 import formats
    out, _ = dyn_run
    path = formats.save_dynamic(str(tmp_path), out["dynamic"], out["keyframe_time_indices"], out["keyframe_dynamic"])
    assert path.endswith("dynamic.npz")
    d = formats.load_dynamic(path)
    assert d["frame"].tolist() == [r["frame"] for r in out["dynamic"]]
    assert np.array_equal(d["dynamic_frac"], np.array([r["dynamic_frac"] for r in out["dynamic"]], np.float32))
    assert d["keyframe_ids"].tolist() == out["keyframe_time_indices"]
    assert np.array_equal(d["keyframe_masks"], np.stack([m.numpy() for m in out["keyframe_dynamic"]]))
    with pytest.raises(ValueError):
        formats.save_dynamic(str(tmp_path), out["dynamic"], out["keyframe_time_indices"][:-1],
                             out["keyframe_dynamic"])
    np.savez(str(tmp_path / "bad.npz"), frame=np.zeros(1))
    with pytest.raises(ValueError):
        formats.load_dynamic(str(tmp_path / "bad.npz"))


def test_an_all_masked_keyframe_adds_a_zero_mapping_loss(problem):
    from splatam_b200 import mapping as M, slam
    from util import cpu_render
    cam, frames, init, kw = problem
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    p = {k: v.clone().requires_grad_(True) for k, v in init.items()}
    p.update(cam_unnorm_rots=rots, cam_trans=trans)
    fr = dict(frames[3], dynamic=torch.ones(64, 64, dtype=torch.bool))
    loss, _ = M.mapping_loss(p, fr, cpu_render)
    loss.backward()
    assert float(loss.detach()) == 0.0 and all(torch.isfinite(p[k].grad).all() for k in init)


def test_cli_flags_are_parsed_and_rejected(monkeypatch, capsys):
    import sys
    from util import load
    tool = load("tools/run_slam_dataset.py")
    base = ["run_slam_dataset.py", "--dataset", "replica", "--basedir", "x", "--sequence", "y", "--dynamic"]
    for extra in (["--relocalise"], ["--relocalise-photometric"]):
        monkeypatch.setattr(sys, "argv", base + extra)
        with pytest.raises(SystemExit) as e:
            tool.main()
        assert e.value.code == 2 and "--dynamic" in capsys.readouterr().err, extra
    seen = {}

    class Stop(Exception):
        pass

    def fake_run_slam(*a, **k):
        seen.update(k)
        raise Stop

    import splatam_b200.datasets as datasets
    import splatam_b200.slam as slam_mod

    class Seq:
        intrinsics, cam, w2c, width, height, load_wait_s = torch.eye(3), None, torch.eye(4), 4, 4, 0.0
        densify_height = densify_width = None

        def __init__(self, *a, **k):
            pass

        def __len__(self):
            return 3

        def __getitem__(self, t):
            return dict(depth=torch.ones(1, 4, 4), intrinsics=torch.eye(3), im=torch.zeros(3, 4, 4))

    monkeypatch.setattr(datasets, "RGBDSequence", Seq)
    monkeypatch.setattr(slam_mod, "initialize_map", lambda *a, **k: ({"means3D": torch.zeros(1, 3)}, 1.0))
    monkeypatch.setattr(slam_mod, "run_slam", fake_run_slam)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda d=None: None)
    for argv, want in ((base, {}), (base[:-1], None)):
        monkeypatch.setattr(sys, "argv", argv)
        seen.clear()
        with pytest.raises(Stop):
            tool.main()
        assert seen["dynamic"] == want
    demo = load("tools/run_iphone_demo.py")
    monkeypatch.setattr(sys, "argv", ["run_iphone_demo.py", "--source", "synthetic", "--out", "x", "--dynamic",
                                      "--capture-only"])
    with pytest.raises(SystemExit) as e:
        demo.main()
    assert e.value.code == 2 and "--dynamic" in capsys.readouterr().err
