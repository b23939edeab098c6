#!/usr/bin/env python
"""Times mesh extraction on one GPU (splatam_b200/mesh.py) and prints one JSON line:

  * integration time per 1200x680 frame into 256^3 and 512^3 volumes at batch 1 / 8 / 32 (sb_tsdf_integrate), with
    the cameras looking into the volume so that the frustum covers most of it and a tenth of it lies in the band
  * extraction time (sb_mc_count + the count read + sb_mc_emit) of the volumes' meshes
  * the whole mesh_record on a synthetic record of --gaussians Gaussians and --frames poses (time_viewer.py's record)

  python tools/time_mesh.py [--gaussians 1000000] [--frames 2000] [--voxel 0.02] [--reps 20]"""
import argparse
import json
import os
import sys
import tempfile
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


def frames(B, dev, seed=0):
    """B frames of a wavy wall 2.5-3.5 m ahead, from cameras near the origin looking along +z."""
    g = np.random.default_rng(seed)
    u = np.arange(W)[None, :] / W
    v = np.arange(H)[:, None] / H
    depth = np.stack([3.0 + 0.3 * np.sin(6 * u + b) * np.cos(4 * v) + 0.01 * g.standard_normal((H, W))
                      for b in range(B)]).astype(np.float32)
    w2c = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    w2c[:, :3, 3] = g.uniform(-0.05, 0.05, (B, 3))
    rgb = g.uniform(0, 1, (B, 3, H, W)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(dev)
    return t(depth), t(rgb), t(w2c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--voxel", type=float, default=0.02, help="voxel size of the mesh_record run")
    ap.add_argument("--batch", type=int, default=32, help="batch of the mesh_record run")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    from splatam_b200.mesh import TSDFVolume, mesh_record
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = dict(gpu=gpu_info(), frame=[W, H])
    depth, rgb, w2c = frames(32, dev)
    for n in (256, 512):
        # a 4 m cube from z = 0.5: the frustum holds most of it, the wall's band a tenth
        vox = 4.0 / n
        vol = TSDFVolume((-2.0, -2.0, 0.5, -2.0 + (n - 1) * vox, -2.0 + (n - 1) * vox, 0.5 + (n - 1) * vox), vox,
                         device=dev)
        assert (vol.nx, vol.ny, vol.nz) == (n, n, n), (vol.nx, vol.ny, vol.nz)
        for B in (1, 8, 32):
            us = TV.events_us(lambda: vol.integrate(depth[:B], rgb[:B], K, w2c[:B]), a.reps)
            out["integrate_%d_b%d_us_per_frame" % (n, B)] = us / B
        touched = float((vol.weight > 0).float().mean())
        band = float(((vol.weight > 0) & (vol.tsdf < 1)).float().mean())
        out["fraction_%d_in_frustum" % n], out["fraction_%d_in_band" % n] = touched, band
        for _ in range(2):
            vol.extract()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            v, c, f = vol.extract()
        torch.cuda.synchronize()
        out["extract_%d_ms" % n] = (time.perf_counter() - t0) * 1e3 / a.reps
        out["mesh_%d_V_F" % n] = [int(v.shape[0]), int(f.shape[0])]
        del vol, v, c, f
        torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        path = TV.synthetic_record(d, a.gaussians, a.frames)
        mesh_record(path, a.voxel, every=500, batch=a.batch, device=dev)     # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v, c, f, info = mesh_record(path, a.voxel, batch=a.batch, device=dev)
        wall = time.perf_counter() - t0
    out["record"] = dict(gaussians=a.gaussians, frames=a.frames, voxel=a.voxel, batch=a.batch, voxels=info["voxels"],
                         dims=list(info["dims"]), V=int(v.shape[0]), F=int(f.shape[0]), wall_s=wall,
                         render_ms=info["render_ms"], integrate_ms=info["integrate_ms"],
                         extract_ms=info["extract_ms"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
