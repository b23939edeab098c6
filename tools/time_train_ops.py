"""Times the training-step kernels with CUDA events: the Gaussian preparation forward + backward (with the camera-pose
gradient) at SplaTAM's map size, through autograd and as the bare backward kernel, the fused image loss and the masked
L1 at 1200x680.  Prints one JSON line of
median microseconds per call over `--reps` calls, `--runs` times.

    python tools/time_train_ops.py [--P 816000] [--reps 200] [--runs 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_info import gpu_info  # noqa: E402


def median_us(fn, reps):
    fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) * 1e3 for a, b in ev)
    return t[len(t) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=816_000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    from splatam_b200.prepare import prepare_gaussians
    from splatam_b200.train_ops import image_loss, masked_l1
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    P = a.P
    mk = lambda *s: torch.randn(*s, device=dev, generator=g)
    leaves = [mk(P, 3), mk(P, 4), mk(P, 1), mk(P, 3) * 0.3 - 3]
    rel = torch.eye(4, device=dev).requires_grad_(True)
    cr = torch.tensor([[1.0, 0.0, 0.0, 0.0]], device=dev).requires_grad_(True)
    w2c0 = torch.eye(4, device=dev)
    ups = [mk(P, n) for n in (3, 4, 1, 3, 3)]
    outs = prepare_gaussians(*leaves, rel, cr, w2c0)

    def prep_bwd():
        torch.autograd.grad(outs, [rel, cr], ups, retain_graph=True)

    # the backward kernel alone, through the C ABI (no autograd bookkeeping): what the pose reduction costs
    from splatam_b200 import _lib
    gm, gu, gl, gs = (torch.empty_like(t) for t in leaves[:2] + leaves[2:4])
    pose = torch.empty(16, dtype=torch.float64, device=dev)
    means_cam, _, opac, sc3, _ = (o.detach() for o in outs)
    flat = [t.contiguous() for t in leaves[:2]] + [rel.detach(), cr.detach().reshape(4), w2c0, means_cam, opac, sc3]

    def prep_bwd_kernel():
        _lib.call("sb_prepare_backward", P, 3, 1, *flat, *ups, gm, gu, gl, gs, pose, device=dev)

    x = torch.rand(3, 680, 1200, device=dev, generator=g).requires_grad_(True)
    y = torch.rand(3, 680, 1200, device=dev, generator=g)

    def img():
        image_loss(x, y).backward()

    ds = torch.rand(3, 680, 1200, device=dev, generator=g).requires_grad_(True)
    gd = torch.rand(1, 680, 1200, device=dev, generator=g)
    im = torch.rand(3, 680, 1200, device=dev, generator=g).requires_grad_(True)

    def masked():
        ld, li = masked_l1(ds, gd, im, y, use_sil=True, depth_mean=False)
        (ld + li).backward()

    res = {k: [] for k in ("prepare_fwd_us", "prepare_bwd_pose_us", "prepare_bwd_kernel_us", "image_loss_fwd_bwd_us",
                           "masked_l1_fwd_bwd_us")}
    for _ in range(a.runs):
        res["prepare_fwd_us"].append(median_us(lambda: prepare_gaussians(*leaves, rel, cr, w2c0), a.reps))
        res["prepare_bwd_pose_us"].append(median_us(prep_bwd, a.reps))
        res["prepare_bwd_kernel_us"].append(median_us(prep_bwd_kernel, a.reps))
        res["image_loss_fwd_bwd_us"].append(median_us(img, a.reps))
        res["masked_l1_fwd_bwd_us"].append(median_us(masked, a.reps))
    res.update(P=P, gpu=gpu_info())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
