"""GPU suite for map compaction (splatam_b200/contrib.py, sb_blend_stats): the statistics against the numpy oracle
(oracle/blend_stats_numpy.py), determinism, bit-identical re-renders of the lossless compaction, and the tool end to
end on a SplaTAM run record."""
import json
import os

import numpy as np
import pytest
import torch

import scenes
from util import load, run_tool

pytestmark = pytest.mark.gpu


def _scenes():
    d = dict(config1=scenes.config1, edge_cases=scenes.edge_cases, dense_opaque=scenes.dense_opaque)
    d.update(scenes.adversarial(small=True))
    return d


def _stats_of(render, P, dev):
    from splatam_b200 import contrib
    from splatam_b200.rasterizer import forward_states
    acc = contrib.BlendStats(P, dev)
    with torch.no_grad(), forward_states() as states:
        out = render()
    acc.add(states[-1])
    return acc.result(), out


def _host(st):
    return {k: v.cpu().numpy() for k, v in st.items()}


@pytest.mark.parametrize("name", sorted(_scenes()))
def test_statistics_match_the_oracle(cuda_device, name):
    """Counts equal the oracle's for every Gaussian it does not flag as near a threshold (EPS_ALPHA = 2e-6 relative on
    alpha, the accumulated bound on T; derived in oracle/blend_stats_numpy.py); max_weight within the oracle's
    per-Gaussian bound.  The plain, the two-set and the sync-free renders (at and above capacity) give the same
    statistics; an overflowed sync-free render adds nothing."""
    from oracle import blend_stats_numpy as BS
    import splatam_b200 as S
    sc = _scenes()[name]()
    rs = sc.settings(S.GaussianRasterizationSettings, cuda_device)
    inp = sc.inputs(cuda_device)
    P = sc.P
    plain, _ = _stats_of(lambda: S.GaussianRasterizer(rs)(**inp), P, cuda_device)
    extra = torch.rand(P, 3, generator=torch.Generator().manual_seed(1)).to(cuda_device)
    fused = lambda cap=None: lambda: S.GaussianRasterizer(rs, max_rendered=cap).forward_fused(
        inp["means3D"], inp["means2D"], inp["opacities"], inp["colors_precomp"], extra, inp["scales"],
        inp["rotations"])
    two, _ = _stats_of(fused(), P, cuda_device)
    o = sc.oracle()
    R = o.R
    for k in plain:
        assert torch.equal(plain[k], two[k]), k
    if R > 0:
        for cap in (R, R + 1000):
            sf, _ = _stats_of(fused(cap), P, cuda_device)
            for k in plain:
                assert torch.equal(plain[k], sf[k]), (k, cap)
        if R > 1:
            over, (im, _, _, _) = _stats_of(fused(R - 1), P, cuda_device)
            assert torch.isnan(im).all()
            for k in over:
                assert not over[k].any(), k
    ref = BS.blend_stats(o)
    got = _host(plain)
    ok = ~ref["flagged"]
    print("%s: %d Gaussians, %d used, %d flagged near a threshold (%.4f %%), %d end-only"
          % (name, P, int(((ref["blended"] > 0) | (ref["ended"] > 0)).sum()), int(ref["flagged"].sum()),
             100.0 * ref["flagged"].mean(), int(((ref["ended"] > 0) & (ref["blended"] == 0)).sum())))
    assert ref["flagged"].mean() < 0.02           # threshold_opacity puts alphas on 1/255 on purpose: 2 of 160
    np.testing.assert_array_equal(got["blended"][ok], ref["blended"][ok])
    np.testing.assert_array_equal(got["ended"][ok], ref["ended"][ok])
    err = np.abs(got["max_weight"][ok].astype(np.float64) - ref["max_weight"][ok])
    assert np.all(err <= ref["max_weight_tol"][ok]), float((err - ref["max_weight_tol"][ok]).max())


def _map(sc, T, dev):
    """A SplaTAM map of `sc` with T cameras along slam.look_trajectory (frame 0 the identity)."""
    from splatam_b200 import slam
    rots, trans = slam.look_trajectory(T, dev)
    g = sc.splatam_params(opacity_clamp=(1e-4, 1 - 1e-4))
    p = {k: v.to(dev).contiguous() for k, v in g.items()}
    p.update(cam_unnorm_rots=rots, cam_trans=trans)
    return p, sc.settings(__import__("splatam_b200").GaussianRasterizationSettings, dev), torch.eye(4, device=dev)


def _renders(params, cam, w2c0, ids, max_rendered=None):
    from splatam_b200 import contrib, mapping as M
    from splatam_b200.rasterizer import forward_states
    out = []
    with torch.no_grad():
        for t in ids:
            with forward_states() as states:
                im, ds, _, _ = M._render_pair(params, contrib._frame(t, cam, w2c0), M.default_render, True,
                                              camera_grad=False, max_rendered=max_rendered)
            st = states[-1]
            n = int(cam.image_height) * int(cam.image_width)
            tiles = ((int(cam.image_width) + 15) // 16) * ((int(cam.image_height) + 15) // 16)
            off = (tiles * 8 + 255) // 256 * 256          # carve_image: ranges, then final_T (256-B aligned)
            final_T = st.image[off:off + 4 * n].view(torch.float32).clone()
            out.append((im.clone(), ds.clone(), final_T))
    return out


def _drop(params, keep):
    from splatam_b200.formats import GAUSSIAN_KEYS
    return dict({k: params[k][keep].contiguous() for k in GAUSSIAN_KEYS}, cam_unnorm_rots=params["cam_unnorm_rots"],
                cam_trans=params["cam_trans"])


def _same(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for ra, rb in zip(a, b) for x, y in zip(ra, rb))


@pytest.mark.parametrize("scene", ["view_filling", "dense_opaque"])
def test_lossless_compaction_renders_bit_identically(cuda_device, scene):
    from splatam_b200 import contrib
    if scene == "view_filling":
        cam = dict(w=160, h=120, fx=80.0, fy=80.0, cx=79.5, cy=59.5)
        sc = scenes.view_filling(seed=3, cam=cam, P=30_000, margin=16, opacity=(0.85, 0.99))
    else:
        sc = scenes.dense_opaque()
    T = 10
    params, cam, w2c0 = _map(sc, T, cuda_device)
    ids = list(range(T))
    st = contrib.blend_stats(params, cam, ids, w2c0)
    st2 = contrib.blend_stats(params, cam, ids, w2c0)
    for k in st:                                             # determinism: integer and max atomics only
        assert torch.equal(st[k].view(torch.int32) if st[k].dtype == torch.float32 else st[k],
                           st2[k].view(torch.int32) if st2[k].dtype == torch.float32 else st2[k]), k
    cap = 32 * sc.P                                          # dense_opaque bins ~9.4 instances per Gaussian
    sf = contrib.blend_stats(params, cam, ids, w2c0, max_rendered=cap)
    assert not __import__("splatam_b200").GaussianRasterizer.last_counts(cuda_device)[1]
    for k in st:
        assert torch.equal(st[k], sf[k]), k
    keep = contrib.keep_mask(st)
    end_only = (st["blended"] == 0) & (st["ended"] > 0)
    print("%s: P %d, kept %d, end-only %d" % (scene, sc.P, int(keep.sum()), int(end_only.sum())))
    assert 0 < int(keep.sum()) < sc.P
    small = _drop(params, keep)
    ref = _renders(params, cam, w2c0, ids)
    assert _same(ref, _renders(small, cam, w2c0, ids))
    assert _same(_renders(params, cam, w2c0, ids, max_rendered=cap),
                 _renders(small, cam, w2c0, ids, max_rendered=cap))
    if scene == "dense_opaque":
        # the terminator count is load-bearing: dropping the end-only Gaussians too changes some pixel
        assert int(end_only.sum()) > 0
        assert not _same(ref, _renders(_drop(params, keep & ~end_only), cam, w2c0, ids))


def test_compact_record_end_to_end(cuda_device, tmp_path, monkeypatch, capsys):
    from splatam_b200 import contrib, datasets, formats, offline, viewer
    T = 6
    scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    data = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0"]
    run_dir = str(tmp_path / "run")
    run_tool(load("tools/run_slam_dataset.py"),
             ["run_slam_dataset.py"] + data + ["--tracking-iters", "10", "--mapping-iters", "10", "--out", run_dir],
             monkeypatch, capsys)
    src = os.path.join(run_dir, "params.npz")
    before = open(src, "rb").read()
    dst = str(tmp_path / "compact.npz")
    tool = load("tools/compact_record.py")
    line = run_tool(tool, ["compact_record.py", "--record", src, "--out", dst, "--every", "1"], monkeypatch, capsys)
    assert open(src, "rb").read() == before
    assert line["views"] == T and (line["width"], line["height"]) == (1200, 680)
    assert 0 < line["gaussians_after"] <= line["gaussians_before"]
    print("compact_record:", json.dumps(line))
    a, b = formats.read_record(src, formats.RECORD_KEYS), formats.read_record(dst, formats.RECORD_KEYS)
    assert list(a) == list(b)
    for k in a:
        assert a[k].dtype == b[k].dtype, k
        if k not in contrib.PER_GAUSSIAN_KEYS:
            assert a[k].tobytes() == b[k].tobytes(), k
    ev = load("tools/eval_record.py")
    per = []
    for rec, out in ((src, "eval_a"), (dst, "eval_b")):
        run_tool(ev, ["eval_record.py"] + data + ["--record", rec, "--out", str(tmp_path / out), "--no-frames",
                                                  "--frames", str(T)], monkeypatch, capsys)
        per.append({n: open(str(tmp_path / out / (n + ".txt"))).read() for n in ("psnr", "l1", "rmse", "ssim")})
    assert per[0] == per[1]                                  # per-frame PSNR, depth errors and MS-SSIM, bit for bit
    formats.export_ply(dst, str(tmp_path / "c.ply"))
    viewer.load_record(dst, cuda_device)
    with datasets.RGBDSequence("replica", str(tmp_path), "room0", desired_height=680, desired_width=1200,
                               device=cuda_device) as seq:
        params, cam, w2c0 = contrib.record_view(b, cuda_device)
        for f in ("image_height", "image_width", "tanfovx", "tanfovy", "scale_modifier", "sh_degree", "prefiltered"):
            assert getattr(cam, f) == getattr(seq.cam, f), f
        for f in ("bg", "viewmatrix", "projmatrix", "campos"):
            assert torch.equal(getattr(cam, f), getattr(seq.cam, f).to(cuda_device)), f
        frames = [seq[t] for t in range(T)]
        offline.from_record(dst, frames, list(range(T)), cuda_device)
    lossy = run_tool(tool, ["compact_record.py", "--record", src, "--out", str(tmp_path / "lossy.npz"), "--every", "1",
                            "--min-weight", "0.05"], monkeypatch, capsys)
    print("compact_record --min-weight 0.05:", json.dumps(lossy))
    assert lossy["gaussians_after"] <= line["gaussians_after"] and np.isfinite(lossy["psnr_db"])
    assert np.isfinite(lossy["depth_l1_m"])


def test_lossy_rule_splits_at_the_weight(cuda_device):
    from splatam_b200 import contrib
    sc = scenes.config1()
    params, cam, w2c0 = _map(sc, 4, cuda_device)
    st = contrib.blend_stats(params, cam, range(4), w2c0)
    for w in (0.01, 0.1, 0.5):
        keep = contrib.keep_mask(st, w)
        assert bool((st["max_weight"][keep] >= w).all()) and bool((st["max_weight"][~keep] < w).all())
    lossless = contrib.keep_mask(st)
    assert bool((contrib.keep_mask(st, 1e-30) <= lossless).all())
