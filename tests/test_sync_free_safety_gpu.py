"""The sync-free (fixed-capacity, CUDA-graph) mode must never pass a truncated render for a valid one: on overflow
the images are NaN, the device flag is raised, the guarded Adam step is a no-op, and the mapper re-captures with a
larger capacity and carries on -- ending where an eager run of the same effective steps ends."""
import numpy as np
import pytest
import torch

import scenes

pytestmark = pytest.mark.gpu


def test_overflow_poisons_images_and_is_reported(cuda_device):
    import splatam_b200 as S
    dev = cuda_device
    sc = scenes.config1(seed=3, P=2000, w=160, h=96)
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    inp = sc.inputs(dev)
    color, radii, depth = S.GaussianRasterizer(rs)(**inp)
    torch.cuda.synchronize()
    R = int(color.grad_fn.state.num_rendered) if color.grad_fn is not None else None
    small = S.GaussianRasterizer(rs, max_rendered=64)
    c2, _, _ = small(**inp)
    n_r, overflow = small.last_counts(dev)
    assert overflow and n_r > 64 and (R is None or n_r == R)
    # the capacity probe of the CUDA-graph paths: the forward's first stage alone counts the same instances
    assert S.GaussianRasterizer(rs).num_rendered(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"]) == n_r
    assert torch.isnan(c2).all(), "a truncated render must be poisoned"
    big = S.GaussianRasterizer(rs, max_rendered=n_r + 10)
    c3, _, _ = big(**inp)
    n_r3, overflow3 = big.last_counts(dev)
    assert not overflow3 and n_r3 == n_r and torch.equal(c3, color)


def _problem(dev):
    import splatam_b200 as S
    sc = scenes.view_filling(seed=41, cam=dict(w=256, h=160, fx=128.0, fy=128.0, cx=127.5, cy=79.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    g = torch.Generator().manual_seed(2)
    gauss = sc.splatam_params(dev)
    rots = torch.zeros(1, 4, 1); rots[:, 0] = 1.0
    trans = torch.zeros(1, 3, 1)
    frames = [dict(id=0, cam=cam, w2c=torch.eye(4, device=dev), im=torch.rand(3, sc.h, sc.w, generator=g).to(dev),
                   depth=(1.5 + 2.0 * torch.rand(1, sc.h, sc.w, generator=g)).to(dev))]
    return gauss, rots.to(dev), trans.to(dev), frames


def test_mapper_recovers_from_capacity_overflow(cuda_device):
    from splatam_b200 import mapping as M
    dev = cuda_device
    gauss, rots, trans, frames = _problem(dev)
    n_steps = 6
    eager = M.ShardedMapper(gauss, rots, trans, seed=1, fused=True)
    eager_losses = [eager.step(frames)[0] for _ in range(n_steps)]
    graphed = M.ShardedMapper(gauss, rots, trans, seed=1, fused=True)
    graphed.enable_graph(frames, capacity=1000)           # far too small on purpose: the first replays overflow
    losses, guard = [], 0
    while graphed.effective_steps()[0] < n_steps and guard < 40:
        losses.append(float(graphed.step(frames)[0]))
        guard += 1
    graphed.poll_overflow(frames, block=True)
    applied, skipped = graphed.effective_steps()
    assert applied == n_steps and skipped >= 1 and graphed.overflow_events >= 1, (applied, skipped, graphed.overflow_events)
    assert any(np.isnan(l) for l in losses), "overflowed steps report a NaN loss"
    good = [l for l in losses if not np.isnan(l)]
    assert np.allclose(good[:n_steps], eager_losses, rtol=1e-3), (good, eager_losses)
    for k in ("means3D", "rgb_colors", "logit_opacities", "log_scales"):
        init = gauss[k]
        du, dr = graphed.g.params[k].detach() - init, eager.g.params[k].detach() - init
        assert float((du - dr).norm() / dr.norm()) < 0.05, k
    assert torch.isfinite(graphed.g.flat).all()
