"""GPU parity tests proper: the sm_90a path (through the C-ABI) against (1) the CPU oracle,
(2) the committed golden vectors, (3) what the unmodified reference extension computed on an H100 for the same
inputs (tests/golden/reference/), and (4) size-independent properties at BASELINE.json's full sizes.

Tolerances (BASELINE.json north_star): tile-ID/depth sort keys bit-identical; colour / depth /
silhouette / gradients within 1e-4 relative float32.
"""
import glob
import json
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, GRADS, REL, bits, check_against, check_against_reference, digest, l2_rel, \
    oracle_outputs, rel_err

pytestmark = pytest.mark.gpu

REF_GOLDEN = os.path.join(GOLDEN, "reference")      # written by tests/golden/make_golden_reference.py


def _golden(name):
    return np.load(os.path.join(REF_GOLDEN, name))


SMALL = [scenes.config1, scenes.edge_cases, lambda: scenes.dense_opaque(P=600, w=64, h=48),
         lambda: scenes.config1(seed=11, P=1000, w=200, h=120, bg=(0.3, 0.1, 0.9))]


@pytest.mark.parametrize("make", SMALL)
def test_cuda_vs_oracle(make, cuda_device):
    from gpu_harness import random_dL, run_ours
    sc = make()
    dL = random_dL(sc)
    ours = run_ours(sc, dL)
    check_against(ours, oracle_outputs(sc, dL), exact_images=False, tag=sc.name + " vs oracle")


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))) or [None])
def test_cuda_vs_golden(path, cuda_device):
    if path is None:
        pytest.skip("no golden fixtures committed yet")
    from gpu_harness import run_ours
    z = np.load(path)
    sc = scenes.Scene(str(z["name"]), int(z["w"]), int(z["h"]), float(z["fx"]), float(z["fy"]), float(z["cx"]),
                      float(z["cy"]), torch.from_numpy(z["means3D"]), torch.from_numpy(z["colors"]),
                      torch.from_numpy(z["opacities"]), torch.from_numpy(z["scales"]), torch.from_numpy(z["rotations"]),
                      w2c=torch.from_numpy(z["w2c"]), bg=tuple(z["bg"].tolist()))
    ours = run_ours(sc, z["dL_dcolor"])
    ref = {k[4:]: z[k] for k in z.files if k.startswith("ref_")}
    check_against(ours, ref, exact_images=True, tag=os.path.basename(path))


BIG = [("config1", scenes.config1), ("edge", scenes.edge_cases), ("dense", lambda: scenes.dense_opaque()),
       ("room50k", lambda: scenes.room(P=50_000)), ("tum_aniso", lambda: scenes.room(seed=9, P=200_000, cam=scenes.TUM_FR1, anisotropic=True)),
       ("config3_1M", lambda: scenes.config3()),
       ("splatam816k", lambda: scenes.view_filling(seed=12)),            # one Gaussian per pixel: every Gaussian in view
       ("replica50k", lambda: scenes.view_filling(seed=12, P=50_000, cover=True)),
       ("tum3m_aniso", lambda: scenes.view_filling(seed=15, P=3_000_000, cam=scenes.TUM_FR1, anisotropic=True))]


@pytest.mark.parametrize("name,make", BIG)
def test_cuda_vs_reference_extension(name, make, cuda_device):
    """Same inputs as the unmodified reference extension was given (tests/golden/reference/parity_<name>.npz): every
    output of check_against's exact branch bit for bit (as SHA-256 digests), the gradients on a seeded sample of the
    visible Gaussians within max(1e-4, 4 x the reference's own run-to-run atomics noise)."""
    from gpu_harness import random_dL, run_ours
    sc = make()
    check_against_reference(run_ours(sc, random_dL(sc)), _golden("parity_%s.npz" % name), sc.P, name)


def _err_stats(a, b):
    """Element-wise relative error with the SURVEY floor (1e-6 of the largest entry) + L2-relative error."""
    e = rel_err(a, b, 1e-6).reshape(-1)
    return dict(l2_rel=l2_rel(a, b), p50=float(np.percentile(e, 50)), p99=float(np.percentile(e, 99)),
                p999=float(np.percentile(e, 99.9)), max=float(e.max()), frac_gt_1e4=float((e > 1e-4).mean()),
                frac_gt_1e3=float((e > 1e-3).mean()))


def test_gradients_vs_double_oracle_full_size(cuda_device):
    """BASELINE config[2] (1M Gaussians, 1200x680): all six gradients against the C oracle, whose backward
    accumulates in DOUBLE and is deterministic, element by element.  The tail is held to the reference extension's
    own statistics against the same oracle (float atomics; tests/golden/reference/gradient_stats_config3.json)."""
    from gpu_harness import random_dL, run_ours
    sc = scenes.config3()
    dL = random_dL(sc)
    ours = run_ours(sc, dL, intermediates=False)
    o = sc.oracle()
    o.render()
    og = o.backward(dL)
    with open(os.path.join(REF_GOLDEN, "gradient_stats_config3.json")) as f:
        ref_stats = json.load(f)["reference_vs_oracle"]
    for k in GRADS:
        if k == "rotations":      # isotropic scene: mathematically zero, float noise in every implementation
            continue
        st = _err_stats(ours["grad_" + k], og[k])
        assert st["l2_rel"] < REL, (k, st)
        # element-wise: float32 sums with cancellation cannot hold 1e-4 on every entry (the reference's own atomics
        # do not either); the bulk must, and the tail must not be worse than the reference's tail
        assert st["p50"] < REL and st["frac_gt_1e3"] < 2e-3, (k, st)
        rs = ref_stats[k]
        assert st["p99"] <= max(2.0 * rs["p99"], REL), (k, st, rs)


def test_full_size_properties(cuda_device):
    """Size-independent properties at BASELINE config[2] (1M Gaussians, 1200x680)."""
    from gpu_harness import random_dL, run_ours
    sc = scenes.config3()
    dL1, dL2 = random_dL(sc, 3), random_dL(sc, 4)
    a = run_ours(sc, dL1)
    keys, lst = a["keys"], a["point_list"]
    assert np.all(keys[1:] >= keys[:-1])
    same = keys[1:] == keys[:-1]
    assert np.all(lst[1:][same] > lst[:-1][same])
    assert int(a["tiles_touched"].sum()) == a["num_rendered"] == int((a["ranges"][:, 1] - a["ranges"][:, 0]).sum())
    assert np.array_equal((keys & 0xFFFFFFFF).astype(np.uint32), bits(a["depths"])[lst])
    # forward is deterministic; backward is linear in dL/dcolor
    b = run_ours(sc, dL2, intermediates=False)
    c = run_ours(sc, dL1 + dL2, intermediates=False)
    assert np.array_equal(bits(a["color"]), bits(b["color"]))
    for k in GRADS:
        if k == "rotations":   # isotropic scene: the quaternion gradient is pure cancellation noise (~1e-12)
            assert np.abs(c["grad_" + k]).max() < 1e-6 * np.abs(c["grad_scales"]).max()
            continue
        assert l2_rel(c["grad_" + k], a["grad_" + k] + b["grad_" + k]) < 1e-5, k
    # a zero upstream gradient gives exactly zero gradients; transmittance is in (0, 1]
    z = run_ours(sc, np.zeros_like(dL1), intermediates=False)
    assert all(not z["grad_" + k].any() for k in GRADS)
    assert a["final_T"].min() >= 0 and a["final_T"].max() <= 1.0


def test_api_edge_cases(cuda_device):
    import splatam_b200 as S
    dev = cuda_device
    sc = scenes.config1()
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    rast = S.GaussianRasterizer(rs)
    inp = sc.inputs(dev)
    with pytest.raises(Exception, match="excatly one of either SHs"):
        rast(means3D=inp["means3D"], means2D=inp["means2D"], opacities=inp["opacities"], scales=inp["scales"],
             rotations=inp["rotations"])
    with pytest.raises(Exception, match="scale/rotation pair"):
        rast(means3D=inp["means3D"], means2D=inp["means2D"], opacities=inp["opacities"],
             colors_precomp=inp["colors_precomp"])
    # empty scene: background-free zero images like the reference (rasterize_points.cu:67-81)
    e = {k: v[:0] for k, v in inp.items()}
    color, radii, depth = rast(**e)
    assert color.shape == (3, sc.h, sc.w) and radii.numel() == 0 and not color.any()
    # everything behind the camera: R == 0, background only, depth default 15
    inp2 = sc.inputs(dev)
    inp2["means3D"][:, 2] = -1.0
    rs2 = rs._replace(bg=torch.tensor([0.25, 0.5, 0.75], device=dev))
    color, radii, depth = S.GaussianRasterizer(rs2)(**inp2)
    assert not radii.any() and torch.allclose(color[1], torch.tensor(0.5, device=dev)) and torch.all(depth == 15.0)
    # non-contiguous inputs (SplaTAM passes a strided view, utils/slam_helpers.py:288)
    inp3 = sc.inputs(dev)
    m4 = torch.cat([inp3["means3D"], torch.ones(sc.P, 1, device=dev)], 1)
    inp3["means3D"] = (torch.eye(4, device=dev) @ m4.T).T[:, :3]
    c3, _, _ = rast(**inp3)
    c0, _, _ = rast(**sc.inputs(dev))
    assert torch.equal(c3, c0)
    # markVisible
    vis = rast.markVisible(inp2["means3D"])
    assert vis.dtype == torch.bool and not vis.any()
    assert rast.markVisible(sc.inputs(dev)["means3D"]).all()


def _cov3d_scene():
    return scenes.config1(seed=13, P=2000, w=160, h=96)


def cov3d_run(mod, dev):
    """One fwd+bwd through the cov3D_precomp branch of `mod` (this repo or the reference extension)."""
    sc = _cov3d_scene()
    cov = torch.from_numpy(sc.oracle().geometry()["cov3D"]).to(dev)   # bit-exact Sigma of the scale/rot path
    dL = torch.randn(3, sc.h, sc.w, generator=torch.Generator().manual_seed(5)).to(dev)
    rs = sc.settings(mod.GaussianRasterizationSettings, dev)
    inp = sc.inputs(dev, requires_grad=True)
    c = cov.clone().requires_grad_(True)
    color, radii, depth = mod.GaussianRasterizer(rs)(means3D=inp["means3D"], means2D=inp["means2D"],
                                                     opacities=inp["opacities"], colors_precomp=inp["colors_precomp"],
                                                     cov3D_precomp=c)
    color.backward(dL)
    return (color.detach().cpu().numpy(), radii.cpu().numpy().astype(np.int32), c.grad.cpu().numpy(),
            inp["means3D"].grad.cpu().numpy())


def test_cov3d_precomp_branch_vs_reference(cuda_device):
    """The cov3D_precomp branch of the operator API (X/cuda_rasterizer/forward.cu:203-214,
    backward.cu:393-395): same images as the scale/rotation path, dL/dcov3D against the reference."""
    import splatam_b200 as S
    dev = cuda_device
    sc = _cov3d_scene()
    col, rad, gcov, gmean = cov3d_run(S, dev)
    # identical to the scale/rotation path
    c0, r0, _ = S.GaussianRasterizer(sc.settings(S.GaussianRasterizationSettings, dev))(**sc.inputs(dev))
    assert np.array_equal(col.view(np.uint32), c0.cpu().numpy().view(np.uint32)) and np.array_equal(rad, r0.cpu().numpy())
    z = _golden("branches.npz")
    assert digest(col) == str(z["cov_digest_color"]) and digest(rad) == str(z["cov_digest_radii"])
    idx = z["cov_index"]
    assert l2_rel(gcov[idx], z["cov_grad_cov3D"]) < REL and l2_rel(gmean[idx], z["cov_grad_means3D"]) < REL


@pytest.mark.parametrize("make", [scenes.config1, scenes.edge_cases, lambda: scenes.dense_opaque(),
                                  lambda: scenes.room(seed=9, P=100_000, cam=scenes.TUM_FR1, anisotropic=True)])
def test_fused_two_set_render_equals_two_passes(make, cuda_device):
    """N1: the fused RGB + depth/silhouette render against two plain renders over the same geometry."""
    import splatam_b200 as S
    dev = cuda_device
    sc = make()
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    rast = S.GaussianRasterizer(rs)
    g = torch.Generator().manual_seed(8)
    extra = torch.rand(sc.P, 3, generator=g).to(dev) * 3.0
    dL1 = torch.randn(3, sc.h, sc.w, generator=g).to(dev)
    dL2 = torch.randn(3, sc.h, sc.w, generator=g).to(dev)
    # two plain passes
    a = sc.inputs(dev, requires_grad=True)
    ex_a = extra.clone().requires_grad_(True)
    m2b = torch.zeros_like(a["means3D"], requires_grad=True)
    c1, r1, d1 = rast(**a)
    c2, _, _ = rast(means3D=a["means3D"], means2D=m2b, opacities=a["opacities"], colors_precomp=ex_a,
                    scales=a["scales"], rotations=a["rotations"])
    ((c1 * dL1).sum() + (c2 * dL2).sum()).backward()
    # fused
    b = sc.inputs(dev, requires_grad=True)
    ex_b = extra.clone().requires_grad_(True)
    f1, f2, rf, df = rast.forward_fused(means3D=b["means3D"], means2D=b["means2D"], opacities=b["opacities"],
                                        colors_precomp=b["colors_precomp"], colors_extra=ex_b, scales=b["scales"],
                                        rotations=b["rotations"])
    ((f1 * dL1).sum() + (f2 * dL2).sum()).backward()
    assert torch.equal(f1, c1) and torch.equal(f2, c2) and torch.equal(rf, r1) and torch.equal(df, d1)
    for k in ["means3D", "colors_precomp", "opacities", "scales", "rotations"]:
        ga, gb = a[k].grad.cpu().numpy(), b[k].grad.cpu().numpy()
        if k == "rotations" and np.abs(ga).max() < 1e-9:
            continue
        assert l2_rel(gb, ga) < 2e-5, (k, l2_rel(gb, ga))
    assert l2_rel(ex_b.grad.cpu().numpy(), ex_a.grad.cpu().numpy()) < 2e-5
    # means2D sink: first colour set only
    assert l2_rel(b["means2D"].grad.cpu().numpy(), a["means2D"].grad.cpu().numpy()) < 2e-5


def sh_run(mod, deg, dev):
    """One fwd+bwd through the shs / sh_degree branch of `mod` (this repo or the reference extension)."""
    sc = scenes.config1(seed=17, P=3000, w=160, h=96)
    g = torch.Generator().manual_seed(deg)
    M = 16
    shs = (torch.randn(sc.P, M, 3, generator=g) * 0.4).to(dev)
    dL = torch.randn(3, sc.h, sc.w, generator=g).to(dev)
    rs = sc.settings(mod.GaussianRasterizationSettings, dev)._replace(sh_degree=deg, campos=torch.tensor([0.1, -0.2, 0.05], device=dev))
    inp = sc.inputs(dev, requires_grad=True)
    sh = shs.clone().requires_grad_(True)
    color, radii, depth = mod.GaussianRasterizer(rs)(means3D=inp["means3D"], means2D=inp["means2D"], shs=sh,
                                                     opacities=inp["opacities"], scales=inp["scales"],
                                                     rotations=inp["rotations"])
    color.backward(dL)
    return (color.detach().cpu().numpy(), radii.cpu().numpy().astype(np.int32), sh.grad.cpu().numpy(),
            inp["means3D"].grad.cpu().numpy(), inp["opacities"].grad.cpu().numpy())


@pytest.mark.parametrize("deg", [0, 1, 3])
def test_sh_colour_branch_vs_reference(deg, cuda_device):
    """The shs / sh_degree branch of the operator (unused by SplaTAM) against the reference extension: radii bit for
    bit, colour on a seeded sample of 4096 values, gradients on a seeded sample of visible Gaussians."""
    import splatam_b200 as S
    col, rad, gsh, gmean, gop = sh_run(S, deg, cuda_device)
    z = _golden("branches.npz")
    t = "sh%d_" % deg
    assert digest(rad) == str(z[t + "digest_radii"])
    b = z[t + "color"]
    e = np.abs(col.reshape(-1)[z[t + "pixels"]] - b) / np.maximum(np.abs(b), 1e-3 * float(z[t + "color_absmax"]))
    assert (e > REL).mean() < 1e-4
    idx = z[t + "index"]
    for a, name in zip([gsh, gmean, gop], ["shs", "means3D", "opacities"]):
        assert l2_rel(a[idx], z[t + "grad_" + name]) < REL, (name, l2_rel(a[idx], z[t + "grad_" + name]))
    assert not gsh[:, (deg + 1) ** 2:, :].any(), "coefficients above sh_degree get no gradient"


def test_sync_free_forward_matches_and_graph_captures(cuda_device):
    """max_rendered (sync-free, fixed-capacity) mode: identical images, gradients within atomics noise, overflow
    flag when the capacity is too small, and forward+backward replayable from a CUDA graph."""
    import splatam_b200 as S
    dev = cuda_device
    sc = scenes.config3(P=200_000)
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    dL = torch.randn(3, sc.h, sc.w, generator=torch.Generator().manual_seed(3)).to(dev)
    a = sc.inputs(dev, requires_grad=True)
    c0, r0, d0 = S.GaussianRasterizer(rs)(**a)
    R = c0.grad_fn.state.num_rendered
    c0.backward(dL)
    rast = S.GaussianRasterizer(rs, max_rendered=int(R * 1.3))
    b = sc.inputs(dev, requires_grad=True)
    c1, r1, d1 = rast(**b)
    c1.backward(dL)
    assert rast.last_counts() == (R, False)
    assert torch.equal(c1, c0) and torch.equal(r1, r0) and torch.equal(d1, d0)
    for k in ["means3D", "colors_precomp", "opacities", "scales"]:
        assert l2_rel(b[k].grad.cpu().numpy(), a[k].grad.cpu().numpy()) < 1e-5, k
    # overflow is reported, not silent
    small = S.GaussianRasterizer(rs, max_rendered=R // 2)
    with torch.no_grad():
        small(**sc.inputs(dev))
    assert small.last_counts() == (R, True)
    # CUDA graph: capture forward + backward once, replay with new inputs in the static buffers
    static = sc.inputs(dev, requires_grad=True)
    leaves = [static[k] for k in ["means3D", "means2D", "colors_precomp", "opacities", "scales", "rotations"]]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            for t in leaves:
                t.grad = None
            rast(**static)[0].backward(dL)
    torch.cuda.current_stream().wait_stream(side)
    for t in leaves:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, _, _ = rast(**static)
        out.backward(dL)
    with torch.no_grad():
        static["colors_precomp"].mul_(0.5)           # change an input in place, replay
    graph.replay()
    torch.cuda.synchronize()
    ref_in = sc.inputs(dev, requires_grad=True)
    with torch.no_grad():
        ref_in["colors_precomp"].mul_(0.5)
    cr, _, _ = S.GaussianRasterizer(rs)(**ref_in)
    cr.backward(dL)
    assert torch.equal(out, cr)
    assert l2_rel(static["means3D"].grad.cpu().numpy(), ref_in["means3D"].grad.cpu().numpy()) < 1e-5


def test_more_than_65535_tiles_uses_32bit_tile_keys(cuda_device):
    """4112x4112 -> 257x257 = 66049 tiles: the tile-id sort switches to 32-bit keys (17 bits, as the reference's
    getHigherMsb gives); checked against the oracle in the synchronous and the sync-free mode."""
    import splatam_b200 as S
    from gpu_harness import random_dL, run_ours
    sc = scenes.config1(seed=21, P=1500, w=4112, h=4112)
    ours = run_ours(sc, random_dL(sc, 1))
    o = sc.oracle()
    geo, b, r = o.geometry(), o.binning(), o.render()
    assert np.array_equal(ours["radii"], geo["radii"])
    assert np.array_equal(ours["keys"], b["keys"]) and np.array_equal(ours["point_list"], b["point_list"])
    assert np.array_equal(ours["ranges"], b["ranges"])
    assert (ours["n_contrib"] != r["n_contrib"]).mean() < 1e-4
    assert (rel_err(ours["color"], r["color"], 1e-3) > REL).mean() < 1e-4
    dev = cuda_device
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    with torch.no_grad():
        c1, _, _ = S.GaussianRasterizer(rs, max_rendered=ours["num_rendered"] + 1000)(**sc.inputs(dev))
    assert S.GaussianRasterizer.last_counts() == (ours["num_rendered"], False)
    assert np.array_equal(c1.cpu().numpy().view(np.uint32), ours["color"].view(np.uint32))
