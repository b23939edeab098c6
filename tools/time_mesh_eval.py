#!/usr/bin/env python
"""Times mesh evaluation on one GPU (splatam_b200/mesh_eval.py) on seeded synthetic data and prints one JSON line with
the card's name and power limit:

  * the ground truth: a wavy floor of --side x --side vertices (about 1M by default) over 10 m x 10 m, and a
    reconstruction: the same surface, sampled with another seed and displaced by 5 mm of noise
  * culling (sb_points_visible): --frames frames at 1200x680 from cameras 1.5 m above the floor looking down, in
    batches of 8 and 32, for 2x10^5 and 10^6 ground-truth samples; the bare launches and visible_mask with its copies
  * the grid build (NearestGrid, including its host read of the box) and the queries (sb_nn_query) both ways, at
    2x10^5 and 10^6 samples per mesh

  python tools/time_mesh_eval.py [--side 1000] [--frames 2000] [--reps 5]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import time_viewer as TV  # noqa: E402
from gpu_info import gpu_info  # noqa: E402

H, W = 680, 1200
K = np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]], np.float32)


def floor_mesh(side):
    """A 10 m x 10 m height field z = 0.05 sin(x) cos(y) of side x side vertices, two triangles per quad."""
    x, y = np.meshgrid(np.linspace(-5, 5, side), np.linspace(-5, 5, side))
    v = np.c_[x.ravel(), y.ravel(), (0.05 * np.sin(x) * np.cos(y)).ravel()].astype(np.float32)
    q = np.arange(side - 1)
    i = (q[:, None] * side + q[None, :]).ravel()
    f = np.concatenate([np.c_[i, i + 1, i + side + 1], np.c_[i, i + side + 1, i + side]])
    return v, f


def cameras(T, dev, seed=0):
    """T w2c of cameras 1.5 m above the floor looking straight down, walking a lawnmower path, and 32 depth images
    of the floor (1.5 m plus noise)."""
    g = np.random.default_rng(seed)
    s = np.linspace(0, 1, T)
    cx, cy = 8 * (s * 4 % 1) - 4, 8 * s - 4
    w2c = np.tile(np.eye(4, dtype=np.float32), (T, 1, 1))
    w2c[:, :3, :3] = np.diag([1.0, -1.0, -1.0])                 # camera z along world -z
    w2c[:, :3, 3] = -(w2c[:, :3, :3] @ np.c_[cx, cy, np.full(T, 1.5)][..., None])[..., 0]
    depth = (1.5 + 0.02 * g.standard_normal((32, H, W))).astype(np.float32)
    return torch.from_numpy(w2c).to(dev), torch.from_numpy(depth).to(dev)


def events_ms(fn, reps):
    return TV.events_us(fn, reps) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--side", type=int, default=1000, help="ground-truth vertices per side")
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from splatam_b200 import _lib, mesh_eval as E
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = dict(gpu=gpu_info(), frame=[W, H], frames=a.frames)
    gv, gf = floor_mesh(a.side)
    out["gt_mesh_V_F"] = [len(gv), len(gf)]
    w2c, depth = cameras(a.frames, dev)
    for n in (200_000, 1_000_000):
        gen = torch.Generator(dev).manual_seed(1)
        gt, _ = E.sample_surface(gv, gf, n, gen, dev)
        pred, _ = E.sample_surface(gv, gf, n, gen, dev)
        pred += 0.005 * torch.randn(pred.shape, device=dev, generator=gen)
        r = dict()
        for B in (8, 32):
            mask = torch.zeros(n, dtype=torch.uint8, device=dev)

            def cull():
                mask.zero_()
                for b0 in range(0, a.frames, B):
                    nb = min(B, a.frames - b0)
                    _lib.call("sb_points_visible", n, gt, nb, H, W, depth[:nb], w2c[b0:b0 + nb], float(K[0, 0]),
                              float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 0.03, mask, device=dev)
            r["cull_launches_b%d_ms" % B] = events_ms(cull, a.reps)
            r["seen_fraction"] = float(mask.float().mean())
            frames = [dict(depth=depth[t % 32], gt_w2c=w2c[t]) for t in range(a.frames)]
            r["visible_mask_b%d_ms" % B] = events_ms(lambda: E.visible_mask(gt, frames, K, 0.03, batch=B), a.reps)
        for name, ref, q in (("gt", gt, pred), ("pred", pred, gt)):
            E.NearestGrid(ref)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.reps):
                grid = E.NearestGrid(ref)
            torch.cuda.synchronize()
            r["build_%s_ms" % name] = (time.perf_counter() - t0) * 1e3 / a.reps
            r["grid_%s_cells_cell" % name] = [int(np.prod(grid.dims)), grid.cell]
            r["query_to_%s_ms" % name] = events_ms(lambda: grid.query(q), a.reps)
        out["samples_%d" % n] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
