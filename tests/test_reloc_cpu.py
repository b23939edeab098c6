"""Relocalisation without a GPU: the numpy restatement of the descriptors, scores, top-k and health record
(oracle/reloc_numpy.py) behaves as stated and retrieves the nearest view of an analytic scene; bad `relocalise`
settings, CPU tensors, a run without intrinsics and a multi-rank run are refused; tools/localise_sequence.py reports
bad arguments."""
import math

import numpy as np
import pytest
import torch

import scenes
from oracle import reloc_numpy as O
from util import cpu_render, load
from splatam_b200 import _lib, reloc, slam


def _img(H, W, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.1, 0.9, (3, H, W)).astype(np.float32), rng.uniform(0.5, 4.0, (H, W)).astype(np.float32)


def test_thumbnail_sizes():
    assert O.thumbnail_size(680, 1200)[:2] == (48, 85)
    assert O.thumbnail_size(480, 640)[:2] == (48, 64)
    assert O.thumbnail_size(45, 97)[:2] == (45, 97)


def test_constant_image_has_constant_grey():
    rgb = np.full((1, 3, 96, 128), 0.37, np.float32)
    d = np.full((1, 96, 128), 2.0, np.float32)
    t = O.thumbnails(rgb, d)
    assert t.shape == (1, 2, 48, 64)
    # constant up to the rounding of the blur's division (border pixels divide by 9 or 12 instead of 16)
    assert np.abs(t[0, 0] - np.float32(0.37)).max() <= 2 * np.spacing(np.float32(0.37)) and np.all(t[0, 1] == 2.0)


def test_grey_score_is_invariant_to_gain_and_offset():
    rgb, d = _img(96, 128, 1)
    a = O.thumbnails(rgb[None], d[None])[0]
    b = O.thumbnails((rgb * 0.5 + 0.2)[None], d[None])[0]
    s = O.score(a, b[None])[0]
    assert abs(s - 1.0) < 1e-6, s                     # the grey NCC stays 1 (to float rounding), depth is equal
    c = a.copy()
    c[1] = np.flip(c[1])                              # a different depth channel lowers only the depth part
    assert O.score(a, c[None])[0] < s


def test_invalid_samples():
    H, W = 96, 96                                     # s = 2: blocks of 4 samples
    rgb, d = _img(H, W, 2)
    d[0:2, 0:2] = [[np.nan, np.inf], [-1.0, 0.0]]     # every depth sample of block (0, 0) is invalid
    d[0:2, 2:4] = [[np.nan, 1.0], [1.0, 1.0]]         # 3 of 4 valid: block (1, 0) stays valid
    d[0:2, 4:6] = [[np.nan, np.inf], [1.0, 1.0]]      # 2 of 4 valid: still valid (at least half)
    m = O._block_means(rgb, d, None)
    assert np.isnan(m[1, 0, 0]) and m[1, 0, 1] == 1.0 and m[1, 0, 2] == 1.0
    assert not np.isnan(m[0, 0, 0])                   # grey does not depend on depth without a silhouette
    sil = np.ones((H, W), np.float32)
    sil[2:4, 0:2] = [[0.99, 0.5], [0.995, 1.0]]       # two samples of block (0, 1) unobserved: valid, 2 of 4
    sil[2:4, 2:4] = [[0.99, 0.5], [0.2, 1.0]]         # three unobserved: invalid in both channels
    m = O._block_means(rgb, d * sil, sil)
    assert not np.isnan(m[0, 1, 0]) and np.isnan(m[0, 1, 1]) and np.isnan(m[1, 1, 1])
    t = O.thumbnails(rgb[None], d[None])[0]
    assert np.isnan(t[1, 0, 0]) and not np.isnan(t[1, 0, 1])   # the blur keeps holes and skips them


def test_score_needs_overlap():
    rgb, d = _img(96, 96, 3)
    a = O.thumbnails(rgb[None], d[None])[0]
    b = a.copy()
    b[:, :30] = np.nan                                # fewer than half of the query's pixels valid in both
    assert O.score(a, b[None])[0] == -2.0
    b = a.copy()
    b[:, :20] = np.nan
    assert O.score(a, b[None])[0] > 0.99


def test_topk_breaks_ties_by_lower_index():
    s = np.array([0.5, 0.9, 0.5, 0.9, -2.0, np.nan, 0.7])
    idx, top = O.topk(s, 5)
    assert idx.tolist() == [1, 3, 6, 0, 2] and top.tolist() == [0.9, 0.9, 0.7, 0.5, 0.5]


def test_health_counts_on_hand_built_depth():
    H, W = 4, 5
    frame = np.full((H, W), 2.0, np.float32)
    frame[0, :] = [0.0, np.nan, np.inf, -1.0, 2.0]    # 4 invalid
    sil = np.ones((H, W), np.float32)
    sil[1, :2] = 0.5                                  # 2 valid, not covered
    dmap = np.full((H, W), 2.0, np.float32)
    dmap[2, :] = [2.03, 2.06, 1.96, 2.0, 3.0]         # tau = max(0.05, 0.02 * 2) = 0.05: 2.06 and 3.0 are outliers
    st = O.health(np.stack([dmap * sil, sil]), frame, 0.05, 0.02, 0.05, 0.5)
    assert st[:3].tolist() == [16.0, 14.0, 12.0] and st[4] == 1.0
    r = (dmap - frame)[sil > 0.99][np.isfinite(frame[sil > 0.99]) & (frame[sil > 0.99] > 0)]
    assert abs(st[3] - math.sqrt((r.astype(np.float64) ** 2).mean())) < 1e-6
    assert O.health(np.stack([dmap, sil]), frame, 0.05, 0.02, 0.05, 0.9)[4] == 0.0     # 12/14 inliers < 0.9
    assert O.health(np.stack([dmap, sil * 0.0]), frame, 0.05, 0.02, 0.05, 0.5)[4] == 0.0  # nothing covered
    zero = O.health(np.stack([dmap, sil]), np.zeros((H, W), np.float32), 0.05, 0.02, 0.05, 0.5)
    assert zero.tolist()[:3] == [0.0, 0.0, 0.0] and zero[4] == 0.0


def _analytic_view(shift, H=96, W=128):
    """A textured wall seen by a camera slid `shift` pixels to the side: colour and depth vary along x and y."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    u = x + shift
    g = 0.5 + 0.2 * np.sin(u * 0.09) + 0.15 * np.sin(y * 0.13 + u * 0.04)
    rgb = np.stack([g, g * 0.9, g * 1.1]).clip(0, 1).astype(np.float32)
    d = (2.0 + 0.4 * np.sin(u * 0.05) + 0.1 * np.cos(y * 0.07)).astype(np.float32)
    return rgb, d


def test_oracle_retrieval_ranks_the_nearest_view_first():
    shifts = np.arange(0, 200, 10)
    db = O.thumbnails(*map(np.stack, zip(*[_analytic_view(s) for s in shifts])))
    for q in (3, 47, 121, 188):
        desc = O.thumbnails(*[a[None] for a in _analytic_view(q)])[0]
        idx, _ = O.topk(O.score(desc, db), 3)
        assert shifts[idx[0]] == shifts[np.argmin(np.abs(shifts - q))], (q, shifts[idx])


@pytest.mark.parametrize("bad", [dict(k=0), dict(k=9), dict(k=2.5), dict(k=True), dict(tau_abs=0.0),
                                 dict(tau_rel=-1.0), dict(min_coverage=1.5), dict(min_inliers=float("nan")),
                                 dict(min_inlier_frac=-0.1), dict(max_rms=0.0), dict(unknown_key=1)])
def test_bad_relocalise_settings_raise(bad):
    with pytest.raises(ValueError, match="relocalise"):
        reloc.config(bad)
    with pytest.raises(ValueError, match="relocalise"):
        _cpu_run(relocalise=bad)


def test_relocalise_is_refused_on_cpu_without_intrinsics_and_on_several_ranks(monkeypatch):
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        _cpu_run(relocalise={})
    with pytest.raises(ValueError, match="intrinsics"):
        _cpu_run(relocalise={}, intrinsics=None)
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda *a: 2)
    with pytest.raises(ValueError, match="one rank"):
        _cpu_run(relocalise={})
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        reloc.thumbnails(torch.zeros(3, 8, 8), torch.ones(8, 8))


def _cpu_run(**kw):
    import splatam_b200 as SB
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(SB.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(3, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(3)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    kw = dict(dict(intrinsics=K), **kw)
    return slam.run_slam(gt, frames, cam, render=cpu_render, fused=False, tracking_iters=2, mapping_iters=1,
                         keyframe_every=1, window=2, **kw)


@pytest.mark.parametrize("argv,msg", [
    (["--dataset", "replica", "--basedir", "b", "--sequence", "s"], "--record"),
    (["--record", "{rec}", "--dataset", "replica", "--basedir", "b", "--sequence", "s", "--every", "0"], "--every"),
    (["--record", "{rec}", "--dataset", "replica", "--basedir", "b", "--sequence", "s", "--k", "9"], "--k"),
    (["--record", "{rec}", "--dataset", "replica", "--basedir", "b", "--sequence", "s", "--map-dataset", "replica"],
     "go together"),
    (["--record", "nowhere.npz", "--dataset", "replica", "--basedir", "b", "--sequence", "s"], "no such file"),
])
def test_localise_sequence_argument_errors(tmp_path, capsys, argv, msg):
    rec = tmp_path / "params.npz"
    np.savez(rec, x=np.zeros(1))
    tool = load("tools/localise_sequence.py")
    with pytest.raises(SystemExit):
        tool.parse_args([a.format(rec=rec) for a in argv])
    assert msg in capsys.readouterr().err
