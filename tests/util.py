"""Shared helpers for the tests."""
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load(relpath):
    """Execute the file at `relpath` (relative to the repository root, or absolute) as a module. Every call returns
    a fresh module object, so a test that monkeypatches a tool changes nothing another test sees."""
    path = os.path.join(ROOT, relpath)
    spec = importlib.util.spec_from_file_location(os.path.splitext(os.path.basename(path))[0], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_tool(tool, argv, monkeypatch, capsys):
    """Run a tool module's main() with `argv` as sys.argv; return the last line it printed, parsed as JSON."""
    monkeypatch.setattr(sys, "argv", argv)
    tool.main()
    return json.loads(capsys.readouterr().out.strip().splitlines()[-1])


def cpu_render(settings, means3D, means2D, opacities, colors_precomp, scales, rotations):
    """The float32 brute-force composite of oracle/bruteforce_torch.py as the `render(settings, **rendervar)`
    callable the mapper and the SLAM loop take."""
    import torch
    from oracle import bruteforce_torch as BF
    out = BF.render(means3D, colors_precomp, opacities, scales, rotations, width=settings.image_width,
                    height=settings.image_height, tanfovx=settings.tanfovx, tanfovy=settings.tanfovy, bg=settings.bg,
                    viewmatrix=settings.viewmatrix[0], projmatrix=settings.projmatrix[0], means2D=means2D,
                    dtype=torch.float32)
    return out["color"], out["radii"], out["depth"]


def bits_equal(a, b):
    """Same shape, dtype and bytes, except that NaNs compare by position only: a NaN that arithmetic produces (the
    inverse of ScanNet's -inf pose, for one) has no portable sign or payload."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind in "fc":
        na, nb = np.isnan(a), np.isnan(b)
        if not np.array_equal(na, nb):
            return False
        a, b = np.where(na, 0, a), np.where(nb, 0, b)
    return a.tobytes() == b.tobytes()


def look_at(cam, target, up=(0.0, 1.0, 0.0)):
    """Float64 world-to-camera matrix of a camera at `cam` looking at `target`, x = fwd x up, y = fwd x x (image
    down for the default `up`); a view direction parallel to `up` takes x = fwd x (1, 0, 0) instead."""
    fwd = np.asarray(target, np.float64) - cam
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, up)
    if np.linalg.norm(right) < 1e-6:
        right = np.cross(fwd, [1.0, 0.0, 0.0])
    right /= np.linalg.norm(right)
    R = np.stack([right, np.cross(fwd, right), fwd])
    w2c = np.eye(4)
    w2c[:3, :3], w2c[:3, 3] = R, -R @ cam
    return w2c


def rel_err(a, b, floor_frac=1e-6):
    """|a-b| / max(|b|, floor_frac * max|b|)  (SURVEY.md section 7, hard part 3)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    floor = floor_frac * max(np.abs(b).max(), 1e-30)
    return np.abs(a - b) / np.maximum(np.abs(b), floor)


def l2_rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def digest(a):
    """SHA-256 of an array's bytes: how the golden data pins outputs that must match bit for bit."""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def exact_arrays(r):
    """The outputs of one render that must equal the reference's bit for bit (dtypes fixed so that digests of this
    repo's and the reference's arrays are comparable)."""
    vis = r["radii"] > 0
    out = dict(radii=np.asarray(r["radii"], np.int32), tiles_touched=np.asarray(r["tiles_touched"], np.uint32),
               depths=np.asarray(r["depths"], np.float32)[vis], means2D=np.asarray(r["means2D"], np.float32)[vis],
               conic_opacity=np.asarray(r["conic_opacity"], np.float32)[vis], keys=np.asarray(r["keys"], np.uint64),
               point_list=np.asarray(r["point_list"], np.uint32), ranges=np.asarray(r["ranges"], np.uint32),
               n_contrib=np.asarray(r["n_contrib"], np.uint32))
    for k in ("final_T", "color", "depth"):
        out[k] = np.asarray(r[k], np.float32)
    return out


GRADS = ["means3D", "means2D", "colors", "opacities", "scales", "rotations"]
REL = 1e-4      # BASELINE.json north_star: colour / depth / gradients within 1e-4 relative float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def oracle_outputs(scene, dL):
    """Everything check_against compares, from the C oracle (its backward accumulates in double)."""
    o = scene.oracle()
    geo, b, r = o.geometry(), o.binning(), o.render()
    g = o.backward(dL)
    ref = dict(radii=geo["radii"], tiles_touched=geo["tiles_touched"], depths=geo["depths"], means2D=geo["means2D"],
               conic_opacity=geo["conic_opacity"], keys=b["keys"], point_list=b["point_list"], ranges=b["ranges"],
               n_contrib=r["n_contrib"], final_T=r["final_T"], color=r["color"], depth=r["depth"])
    ref.update({"grad_" + k: g[k] for k in GRADS})
    return ref


def check_grads(ours, ref, tag, grad_tol=REL, keys=GRADS, tail=None):
    """Gradients element by element: L2-relative within grad_tol (one value, or one per gradient name), at most
    max(2e-3, 2 entries, tail[k]) of the entries off by 10 x grad_tol."""
    for k in keys:
        tol = grad_tol[k] if isinstance(grad_tol, dict) else grad_tol
        a, b = ours["grad_" + k].reshape(-1), ref["grad_" + k].reshape(-1)
        if k == "rotations" and np.abs(b).max() < 1e-6 * np.abs(ref["grad_scales"]).max():
            # isotropic scene: the quaternion gradient is mathematically zero and pure cancellation noise (~1e-10) in
            # every implementation (the reference's two runs differ by ~100 % here); only its smallness is meaningful
            assert np.abs(a).max() < 1e-6 * np.abs(ref["grad_scales"]).max(), (tag, k)
            continue
        assert l2_rel(a, b) < tol, (tag, k, l2_rel(a, b))
        # element-wise: entries that are sums with heavy cancellation carry float32 summation-order noise
        # (the reference's own atomics are order-nondeterministic), so floor at 1e-3 of the largest entry
        frac = (rel_err(a, b, 1e-3) > 10 * tol).mean()
        assert frac <= max(2e-3, 2.0 / a.size, tail[k] if tail else 0.0), (tag, k, frac)


def reference_grad_tol(z, floor=REL):
    """Per-gradient tolerance max(floor, 4 x the reference's own run-to-run noise) of a parity record: no float32
    implementation with atomic accumulation can match another more closely than the reference matches itself."""
    return {k: max(floor, 4 * float(z["noise_" + k] if "noise_" + k in z.files else z["noise"])) for k in GRADS}


def reference_tail(z):
    """Per-gradient fraction of entries two float32 implementations may have off by 10 x their tolerance against a
    third: twice the fraction of entries by which the reference itself misses the double-accumulating C oracle
    (`tail_<k>`, measured over every entry by make_golden_reference.py like gradient_stats); 0 for records without it."""
    return {k: 2.0 * float(z["tail_" + k]) if "tail_" + k in z.files else 0.0 for k in GRADS}


def check_against(ours, ref, exact_images, tag, grad_tol=REL, tail=None, grads=True):
    """One render of this repository (gpu_harness.run_ours) against full outputs of the oracle or the reference."""
    vis = ref["radii"] > 0
    assert np.array_equal(ours["radii"], ref["radii"]), tag
    assert np.array_equal(ours["tiles_touched"], ref["tiles_touched"]), tag
    assert np.array_equal(bits(ours["depths"][vis]), bits(ref["depths"][vis])), tag
    assert np.array_equal(bits(ours["means2D"][vis]), bits(ref["means2D"][vis])), tag
    assert np.array_equal(bits(ours["conic_opacity"][vis]), bits(ref["conic_opacity"][vis])), tag
    assert ours["num_rendered"] == len(ref["keys"]), tag
    assert np.array_equal(ours["keys"], ref["keys"]), tag + ": sorted (tile|depth) keys must be bit-identical"
    assert np.array_equal(ours["point_list"], ref["point_list"]), tag
    assert np.array_equal(ours["ranges"], ref["ranges"]), tag
    if exact_images:
        assert np.array_equal(ours["n_contrib"], ref["n_contrib"]), tag
        assert np.array_equal(bits(ours["final_T"]), bits(ref["final_T"])), tag
        assert np.array_equal(bits(ours["color"]), bits(ref["color"])), tag
        assert np.array_equal(bits(ours["depth"]), bits(ref["depth"])), tag
    else:  # CPU expf differs from libdevice expf by an ulp or two
        assert (ours["n_contrib"] != ref["n_contrib"]).mean() < 1e-3, tag
        assert (rel_err(ours["color"], ref["color"], 1e-3) > REL).mean() < 1e-3, tag
        assert (rel_err(ours["final_T"], ref["final_T"], 1e-3) > REL).mean() < 1e-3, tag
    if grads:
        check_grads(ours, ref, tag, grad_tol, tail=tail)


def check_against_reference(ours, z, P, tag, grads=True):
    """One render against a tests/golden/reference/parity_*.npz record of the unmodified reference extension: every
    output of exact_arrays bit for bit (as SHA-256 digests), the gradients on its seeded sample of the visible
    Gaussians within max(1e-4, 4 x the reference's own run-to-run atomics noise) -- per gradient where the record
    has it."""
    assert ours["num_rendered"] == int(z["num_rendered"]), tag
    for k, a in exact_arrays(ours).items():
        assert digest(a) == str(z["digest_" + k]), (tag, k, "must be bit-identical to the reference")
    tols, tails = reference_grad_tol(z), reference_tail(z)
    scale = float(z["max_grad_scales"])
    for k in GRADS if grads else []:
        grad_tol = tols[k]
        g = ours["grad_" + k].reshape(P, -1)
        if k == "rotations" and float(z["max_grad_rotations"]) < 1e-6 * scale:
            # isotropic scene: the quaternion gradient is mathematically zero (see check_grads)
            assert np.abs(g).max() < 1e-6 * scale, (tag, k)
            continue
        a, b = g[z["index"]].reshape(-1), z["grad_" + k].reshape(-1)
        assert l2_rel(a, b) < grad_tol, (tag, k, l2_rel(a, b))
        e = np.abs(a - b) / np.maximum(np.abs(b), 1e-3 * float(z["absmax_grad_" + k]))
        frac = (e > 10 * grad_tol).mean()
        assert frac <= max(2e-3, 2.0 / a.size, tails[k]), (tag, k, frac)


def sample_rows(mask, n, seed=0):
    """A fixed, seeded, sorted sample of at most n row indices among those where `mask` is true."""
    rows = np.flatnonzero(np.asarray(mask).reshape(-1))
    return np.sort(np.random.default_rng(seed).choice(rows, min(n, rows.size), replace=False))


def reference_extension():
    """The UNMODIFIED reference CUDA extension built into oracle/_ref by oracle/reference.py, or None."""
    from oracle import reference
    return reference.extension()


def _align(off, a=128):
    return (off + a - 1) // a * a


def parse_reference_buffers(geom, binning, img, P, R, W, H):
    """Decode the reference's three scratch byte buffers (GeometryState / BinningState / ImageState
    ::fromChunk, X/cuda_rasterizer/rasterizer_impl.cu:155-194; every chunk 128-B aligned)."""
    import torch
    out = {}
    g = geom.cpu().numpy()
    off = 0

    def take(buf, off, dtype, count):
        off = _align(off)
        n = np.dtype(dtype).itemsize * count
        return np.frombuffer(buf[off:off + n].tobytes(), dtype=dtype), off + n

    out["depths"], off = take(g, off, np.float32, P)
    _, off = take(g, off, np.uint8, 3 * P)           # clamped
    out["internal_radii"], off = take(g, off, np.int32, P)
    m2, off = take(g, off, np.float32, 2 * P)
    out["means2D"] = m2.reshape(P, 2)
    c3, off = take(g, off, np.float32, 6 * P)
    out["cov3D"] = c3.reshape(P, 6)
    co, off = take(g, off, np.float32, 4 * P)
    out["conic_opacity"] = co.reshape(P, 4)
    _, off = take(g, off, np.float32, 3 * P)         # rgb
    out["tiles_touched"], off = take(g, off, np.uint32, P)
    if R > 0:
        b = binning.cpu().numpy()
        off = 0
        out["point_list"], off = take(b, off, np.uint32, R)
        _, off = take(b, off, np.uint32, R)
        out["keys"], off = take(b, off, np.uint64, R)
    i = img.cpu().numpy()
    off = 0
    N = W * H
    ft, off = take(i, off, np.float32, N)
    out["final_T"] = ft.reshape(H, W)
    nc, off = take(i, off, np.uint32, N)
    out["n_contrib"] = nc.reshape(H, W)
    rg, off = take(i, off, np.uint32, 2 * N)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    out["ranges"] = rg.reshape(N, 2)[:tiles]
    return out
