"""GPU: the depth-loss rule of mapping.track_frame (the reference's use_depth_loss_thres, R/scripts/splatam.py:727-738)
on test_tracking_gpu.py's problem, eager and graph-replayed.  A threshold that is always met must give the run of
num_iters iterations without the rule, a threshold of 0 the run of 2 * num_iters, within test_tracking_gpu.py's bounds:
the backward accumulates with float atomics, so two runs of the same loop are not bit-identical on the GPU (the
bit-for-bit check of the rule is tests/test_tracking_rule_cpu.py, over a deterministic renderer)."""
import numpy as np
import pytest
import torch

from test_tracking_gpu import _pose_params, _problem

pytestmark = pytest.mark.gpu

N = 20


def _track(gauss, frame, dev, num_iters, graph, **kw):
    from splatam_b200 import mapping as M
    r0, t0 = _pose_params(dev, [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    p = dict({k: v.detach() for k, v in gauss.items()}, cam_unnorm_rots=r0, cam_trans=t0)
    losses = M.track_frame(p, dict(frame), num_iters=num_iters, fused=True, graph=graph, **kw)
    return losses, p["cam_unnorm_rots"][..., 1].detach().clone(), p["cam_trans"][..., 1].detach().clone()


def _close(got, ref, n):
    assert len(got[0]) == n
    assert np.allclose(got[0][:8], ref[0][:8], rtol=1e-3)
    assert (got[1] - ref[1]).abs().max() < 1e-3 and (got[2] - ref[2]).abs().max() < 2e-3


def test_rule_eager_matches_fixed_iteration_runs(cuda_device):
    dev = cuda_device
    _, gauss, frame = _problem(dev)
    base_n, base_2n = _track(gauss, frame, dev, N, False), _track(gauss, frame, dev, 2 * N, False)
    _close(_track(gauss, frame, dev, N, False, depth_loss_thres=float("inf")), base_n, N)
    _close(_track(gauss, frame, dev, N, False, depth_loss_thres=0.0), base_2n, 2 * N)


def test_rule_graphed_matches_fixed_iteration_runs(cuda_device):
    from splatam_b200 import mapping as M
    dev = cuda_device
    _, gauss, frame = _problem(dev)
    base_n, base_2n = _track(gauss, frame, dev, N, True), _track(gauss, frame, dev, 2 * N, True)
    met = _track(gauss, frame, dev, N, True, depth_loss_thres=float("inf"))
    never = _track(gauss, frame, dev, N, True, depth_loss_thres=0.0)
    _close(met, base_n, N)
    _close(never, base_2n, 2 * N)
    # the decision is taken per frame on the device: a cached graph serves both outcomes
    again = _track(gauss, frame, dev, N, True, depth_loss_thres=float("inf"))
    assert len(again[0]) == N
    # graphs are cached per learning rates and rule, so other rates are never replayed with a stale graph
    p = dict(gauss, cam_unnorm_rots=torch.zeros(1, 4, 2, device=dev), cam_trans=torch.zeros(1, 3, 2, device=dev))
    keys = {M._tracking_key(p, frame, N, lr_rot, lr_trans, thres)
            for lr_rot, lr_trans, thres in ((0.0004, 0.002, None), (0.001, 0.004, None), (0.001, 0.004, 20000.0))}
    assert len(keys) == 3
