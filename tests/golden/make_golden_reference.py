"""Generates tests/golden/reference/: what the GPU tests compare this repository against, produced by the UNMODIFIED
reference extension and the reference's own Python (both installed into oracle/_ref by oracle/reference.py).  Run on
an H100 with oracle/_ref built:

    python tests/golden/make_golden_reference.py OUT_DIR

then copy OUT_DIR/* into tests/golden/reference/.  `--only adversarial` writes only the parity_adv_*.npz records of
the adversarial scenes (scenes.adversarial), leaving the other records -- and the atomics noise sampled into them --
as they are.  The inputs are the tests' own seeded problems (imported from the
test modules), so a fixture and the test that reads it always see the same data.  Large outputs are stored as
SHA-256 digests of their bytes (for the bit-exact comparisons) and as a fixed, seeded sample of the Gaussians (for
the gradient tolerances), which keeps every file far below 1 MB.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import refsrc  # noqa: E402
import scenes  # noqa: E402
import test_parity_gpu as TP  # noqa: E402
import test_ref_glue_gpu as TG  # noqa: E402
import test_slam_gpu as TS  # noqa: E402
import test_tracking_gpu as TT  # noqa: E402
from gpu_harness import GRADS, random_dL, run_ref  # noqa: E402
from util import REL, digest, exact_arrays, l2_rel, oracle_outputs, reference_extension, rel_err, sample_rows  # noqa: E402,E501


def parity(name, make, out, tails=False):
    """test_cuda_vs_reference_extension: digests of every exact output, two runs' gradient noise (overall and per
    gradient), sampled gradients; with `tails`, the fraction of all entries by which the reference misses the
    double-accumulating C oracle at 10 x its tolerance (util.reference_tail)."""
    sc = make()
    dL = random_dL(sc)
    r1, r2 = run_ref(sc, dL), run_ref(sc, dL)
    idx = sample_rows(r1["radii"] > 0, 128)
    d = dict(num_rendered=r1["num_rendered"], index=idx,
             noise=max(l2_rel(r2["grad_" + k], r1["grad_" + k]) for k in GRADS),
             **{"noise_" + k: l2_rel(r2["grad_" + k], r1["grad_" + k]) for k in GRADS},
             max_grad_rotations=np.abs(r1["grad_rotations"]).max(), max_grad_scales=np.abs(r1["grad_scales"]).max())
    for k, a in exact_arrays(r1).items():
        d["digest_" + k] = digest(a)
    og = oracle_outputs(sc, dL) if tails else None
    for k in GRADS:
        g = r1["grad_" + k].reshape(sc.P, -1)
        d["grad_" + k] = g[idx]
        d["absmax_grad_" + k] = np.abs(g).max()
        if tails:
            # the reference's own element-wise miss of the double oracle over every entry, at the tests' threshold
            tol = max(REL, 4 * d["noise_" + k])
            d["tail_" + k] = float((rel_err(g, og["grad_" + k].reshape(sc.P, -1), 1e-3) > 10 * tol).mean())
    np.savez_compressed(os.path.join(out, "parity_%s.npz" % name), **d)


def adversarial(out):
    """test_raster_adversarial_gpu.test_adversarial_vs_reference_extension: one parity record per adversarial scene."""
    for name, make in sorted(scenes.adversarial().items()):
        parity("adv_" + name, make, out, tails=True)
        print("parity adv_" + name, flush=True)


def gradient_stats(out):
    """test_gradients_vs_double_oracle_full_size: the reference's own element-wise error against the double oracle."""
    sc = scenes.config3()
    dL = random_dL(sc)
    o = sc.oracle()
    o.render()
    og = o.backward(dL)
    r = run_ref(sc, dL)
    stats = {k: TP._err_stats(r["grad_" + k], og[k]) for k in GRADS if k != "rotations"}
    with open(os.path.join(out, "gradient_stats_config3.json"), "w") as f:
        json.dump({"workload": "config3 1M Gaussians 1200x680", "reference_vs_oracle": stats}, f, indent=1)


def branches(ref, out):
    """test_cov3d_precomp_branch_vs_reference and test_sh_colour_branch_vs_reference."""
    dev = torch.device("cuda:0")
    d = {}
    col, rad, gcov, gmean = TP.cov3d_run(ref, dev)
    idx = sample_rows(rad > 0, 256)
    d.update(cov_digest_color=digest(col), cov_digest_radii=digest(rad), cov_index=idx, cov_grad_cov3D=gcov[idx],
             cov_grad_means3D=gmean[idx])
    for deg in (0, 1, 3):
        col, rad, gsh, gmean, gop = TP.sh_run(ref, deg, dev)
        idx = sample_rows(rad > 0, 64)
        pix = np.sort(np.random.default_rng(deg).choice(col.size, 4096, replace=False))
        d.update({"sh%d_digest_radii" % deg: digest(rad), "sh%d_index" % deg: idx, "sh%d_pixels" % deg: pix,
                  "sh%d_color" % deg: col.reshape(-1)[pix], "sh%d_color_absmax" % deg: np.abs(col).max(),
                  "sh%d_grad_shs" % deg: gsh[idx], "sh%d_grad_means3D" % deg: gmean[idx],
                  "sh%d_grad_opacities" % deg: gop[idx]})
    np.savez_compressed(os.path.join(out, "branches.npz"), **d)


def loops(ref, out):
    """The loop-level tests: the reference's get_loss / optimizer / SLAM / tracking runs over the reference extension."""
    dev = torch.device("cuda:0")
    R = refsrc.load(ref)
    d = {}
    sc, params, gt_im, gt_d = TG._loop_problem(dev)
    for mode in ("mapping", "tracking"):
        loss, grads, variables, _ = TG._run_get_loss(R, sc, params, gt_im, gt_d, mode, dev)
        d["%s_loss" % mode] = loss
        d["%s_digest_seen" % mode] = digest(variables["seen"].cpu().numpy())
        d["%s_digest_max_2D_radius" % mode] = digest(variables["max_2D_radius"].cpu().numpy())
        idx = sample_rows(variables["seen"].cpu().numpy(), 256)
        d["%s_index" % mode] = idx
        for k in TG.loss_keys(mode):
            g = grads[k].cpu().numpy()
            d["%s_grad_%s" % (mode, k)] = g if k.startswith("cam_") else g[idx]
    ref_losses, p = TG.stock_mapping_iterations(R, sc, params, gt_im, gt_d, dev)
    d["stock_losses"] = np.array(ref_losses)
    idx = np.sort(np.random.default_rng(1).choice(sc.P, 512, replace=False))
    d["stock_index"] = idx
    for k in TG.UPDATE_KEYS:
        d["stock_update_" + k] = (p[k].detach() - params[k]).cpu().numpy()[idx]
    d.update({"tracking_run_" + k: v for k, v in TT.reference_run(ref, dev).items()})
    d.update({"slam_" + k: v for k, v in TS.reference_run(ref, dev).items()})
    np.savez_compressed(os.path.join(out, "loops.npz"), **d)


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("out", help="directory the records are written to")
    ap.add_argument("--only", choices=["adversarial"], help="write only this group of records")
    args = ap.parse_args()
    out = args.out
    os.makedirs(out, exist_ok=True)
    ref = reference_extension()
    assert ref is not None and refsrc.available(), "oracle/_ref is not built (oracle/reference.py)"
    if args.only == "adversarial":
        adversarial(out)
        print("adversarial records written to", out)
        sys.exit(0)
    for name, make in TP.BIG:
        parity(name, make, out)
        print("parity", name, flush=True)
    branches(ref, out)
    loops(ref, out)
    gradient_stats(out)
    adversarial(out)
    print("golden written to", out)
