"""GPU suite for the adversarial scenes (scenes.adversarial; what each one covers is asserted by
tests/test_raster_adversarial_cpu.py): needle splats, opacities at 1/255, near-plane and frustum-clamped giants,
translucent stacks thousands deep, depth ties across sort tiles and tiny images.  The blend kernels cull
(Gaussian, pixel) pairs with conservative boxes and the sort runs in two levels, where the reference evaluates every
pair of a tile and sorts (tile | depth) keys once; these are the inputs on which the two routes could part.

Each scene is checked against the unmodified reference extension's digests (tests/golden/reference/parity_adv_*.npz),
against the C oracle element by element (double-accumulated gradients), through the fused two-colour-set path with
SplaTAM's [depth, 1, depth^2] colours, and in sync-free mode at exactly its tile-instance capacity.  Every gradient
comparison allows 4 x the reference's own run-to-run noise of that gradient, which the needles' ill-conditioned
conics make large, and element-wise twice the fraction of entries by which the reference itself misses the oracle."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, GRADS, check_against, check_against_reference, check_grads, l2_rel, oracle_outputs, \
    reference_grad_tol, reference_tail

pytestmark = pytest.mark.gpu

ADV = scenes.adversarial()
NAMES = sorted(ADV)
# 2D condition numbers of 1e5-1e6: the float32 conic of such a needle is far from its float64 value, so its gradients
# are rounding noise in every float32 implementation (the reference's included); the scene is there for its forward
FORWARD_ONLY = {"box_edge_needles"}


def _golden(name):
    return np.load(os.path.join(GOLDEN, "reference", "parity_adv_%s.npz" % name))


@pytest.mark.parametrize("name", NAMES)
def test_adversarial_vs_reference_extension(name, cuda_device):
    from gpu_harness import random_dL, run_ours
    sc = ADV[name]()
    check_against_reference(run_ours(sc, random_dL(sc)), _golden(name), sc.P, name, grads=name not in FORWARD_ONLY)


@pytest.mark.parametrize("name", NAMES)
def test_adversarial_vs_oracle(name, cuda_device):
    from gpu_harness import random_dL, run_ours
    sc = ADV[name]()
    dL = random_dL(sc)
    check_against(run_ours(sc, dL), oracle_outputs(sc, dL), exact_images=False, tag=name + " vs oracle",
                  grad_tol=reference_grad_tol(_golden(name)), tail=reference_tail(_golden(name)),
                  grads=name not in FORWARD_ONLY)


def depth_colours(sc):
    """SplaTAM's second colour set: [z, 1, z^2] per Gaussian, z its camera-space depth."""
    p4 = torch.cat([sc.means3D, torch.ones(sc.P, 1)], 1)
    z = (p4 @ sc.view[0])[:, 2]
    return torch.stack([z, torch.ones_like(z), z * z], 1).contiguous()


@pytest.mark.parametrize("name", NAMES)
def test_adversarial_fused_two_set(name, cuda_device):
    """The fused RGB + depth/silhouette render: images identical to two single-set renders; gradients against the
    sum of the oracle's two single-set backwards (the colour gradients per set, means2D from the first set only)."""
    from oracle import oracle as O
    import splatam_b200 as S
    dev = cuda_device
    sc = ADV[name]()
    rast = S.GaussianRasterizer(sc.settings(S.GaussianRasterizationSettings, dev))
    extra = depth_colours(sc)
    g = torch.Generator().manual_seed(8)
    dL1, dL2 = torch.randn(3, sc.h, sc.w, generator=g), torch.randn(3, sc.h, sc.w, generator=g)
    b = sc.inputs(dev, requires_grad=True)
    ex = extra.to(dev).requires_grad_(True)
    f1, f2, rf, df = rast.forward_fused(means3D=b["means3D"], means2D=b["means2D"], opacities=b["opacities"],
                                        colors_precomp=b["colors_precomp"], colors_extra=ex, scales=b["scales"],
                                        rotations=b["rotations"])
    ((f1 * dL1.to(dev)).sum() + (f2 * dL2.to(dev)).sum()).backward()
    with torch.no_grad():
        c1, r1, d1 = rast(**sc.inputs(dev))
        c2, _, _ = rast(**dict(sc.inputs(dev), colors_precomp=extra.to(dev)))
    assert torch.equal(f1, c1) and torch.equal(f2, c2) and torch.equal(rf, r1) and torch.equal(df, d1), name
    if name in FORWARD_ONLY:
        return

    o1 = sc.oracle()
    o1.render()
    g1 = o1.backward(dL1.numpy())
    o2 = O.Oracle(sc.oracle_cam(), sc.means3D.numpy(), extra.numpy(), sc.opacities.numpy(), sc.scales.numpy(),
                  sc.rotations.numpy())
    o2.render()
    g2 = o2.backward(dL2.numpy())
    names = {"colors": "colors_precomp"}
    ours = {"grad_" + k: b[names.get(k, k)].grad.cpu().numpy() for k in GRADS}
    ref = {"grad_" + k: g1[k] + g2[k] for k in ("means3D", "opacities", "scales", "rotations")}
    ref.update(grad_means2D=g1["means2D"], grad_colors=g1["colors"])
    tol, tail = reference_grad_tol(_golden(name)), reference_tail(_golden(name))
    check_grads(ours, ref, name + " fused", tol, tail=tail)
    check_grads({"grad_colors": ex.grad.cpu().numpy()}, {"grad_colors": g2["colors"]}, name + " fused set 2", tol,
                keys=["colors"], tail=tail)


@pytest.mark.parametrize("name", NAMES)
def test_adversarial_sync_free_at_capacity(name, cuda_device):
    """max_rendered == R renders exactly what the synchronous path renders and reports no overflow; R - 1 reports
    overflow."""
    import splatam_b200 as S
    dev = cuda_device
    sc = ADV[name]()
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    dL = torch.randn(3, sc.h, sc.w, generator=torch.Generator().manual_seed(3)).to(dev)
    a = sc.inputs(dev, requires_grad=True)
    c0, r0, d0 = S.GaussianRasterizer(rs)(**a)
    R = c0.grad_fn.state.num_rendered
    c0.backward(dL)
    rast = S.GaussianRasterizer(rs, max_rendered=R)
    b = sc.inputs(dev, requires_grad=True)
    c1, r1, d1 = rast(**b)
    c1.backward(dL)
    assert rast.last_counts() == (R, False), name
    assert torch.equal(c1, c0) and torch.equal(r1, r0) and torch.equal(d1, d0), name
    tol = reference_grad_tol(_golden(name), floor=1e-5)
    for k in [] if name in FORWARD_ONLY else ["means3D", "colors_precomp", "opacities", "scales"]:
        assert l2_rel(b[k].grad.cpu().numpy(), a[k].grad.cpu().numpy()) < tol[{"colors_precomp": "colors"}.get(k, k)], \
            (name, k)
    short = S.GaussianRasterizer(rs, max_rendered=R - 1)
    with torch.no_grad():
        short(**sc.inputs(dev))
    assert short.last_counts() == (R, True), name
