#!/usr/bin/env python
"""Times mesh depth rendering on one GPU (sb_mesh_depth, splatam_b200/mesh_eval.py) on seeded synthetic meshes and
prints one JSON line with the card's name and power limit:

  * sb_mesh_depth at batch 1, 8 and 32, at 500x500 (fx = 300) and 1200x680 (fx = 600), for
      - floor_far:  the wavy floor of tools/time_mesh_eval.py (--side^2 vertices, about 2M faces) from 1.5 m above,
                    looking down
      - floor_near: the same floor from 5 cm above, pitched 60 degrees from straight down: large faces, many of them
                    crossing the near plane
      - screen:     two triangles that fill the image, 1 m in front (load balance: two faces, every pixel)
  * depth_l1 end to end: --views accepted views of the floor against a coarser floor, culled by --frames frames at
    1200x680, split into render and cull time (its own device timers), with the view centres 1-2 m above the floor

  python tools/time_mesh_depth.py [--side 1000] [--frames 2000] [--views 1000] [--reps 5]"""
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
import time_mesh_eval as TME  # noqa: E402
from gpu_info import gpu_info  # noqa: E402


floor_mesh = TME.floor_mesh

SIZES = {"500x500": (500, 500, np.array([[300.0, 0, 249.5], [0, 300.0, 249.5], [0, 0, 1]])),
         "1200x680": (680, 1200, np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]]))}


def look(B, height, pitch_deg, seed=0):
    """B w2c [B,4,4] at `height` above z = 0 along the line x = 0 (where the floor is at z = 0), camera z pitched
    `pitch_deg` from straight down towards +y."""
    g = np.random.default_rng(seed)
    a = np.radians(pitch_deg)
    z = np.array([0.0, np.sin(a), -np.cos(a)])
    x = np.array([1.0, 0.0, 0.0])
    R = np.stack([x, np.cross(z, x), z])
    w2c = np.tile(np.eye(4), (B, 1, 1))
    for b in range(B):
        c = np.array([0.0, g.uniform(-3, 3), height])
        w2c[b, :3, :3] = R
        w2c[b, :3, 3] = -R @ c
    return w2c.astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--side", type=int, default=1000, help="floor vertices per side")
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--views", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from splatam_b200 import mesh_eval as E
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = dict(gpu=gpu_info())
    fv, ff = floor_mesh(a.side)
    out["floor_V_F"] = [len(fv), len(ff)]
    screen_v = np.array([[-10, -10, 1], [10, -10, 1], [10, 10, 1], [-10, 10, 1]], np.float32)
    screen_f = np.array([[0, 1, 2], [0, 2, 3]])
    meshes = {"floor_far": (E.MeshDepth(fv, ff, dev), 1.5, 0.0), "floor_near": (E.MeshDepth(fv, ff, dev), 0.05, 60.0),
              "screen": (E.MeshDepth(screen_v, screen_f, dev), None, None)}
    for name, (m, height, pitch) in meshes.items():
        r = dict()
        for size, (H, W, K) in SIZES.items():
            for B in (1, 8, 32):
                w = look(B, height, pitch) if height is not None else np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
                w = torch.from_numpy(w).to(dev)
                d, _ = m.render(w, K, H, W)
                ms = TME.events_ms(lambda: m.render(w, K, H, W), a.reps)
                r["%s_b%d" % (size, B)] = dict(ms=ms, ms_per_view=ms / B, covered=float((d > 0).float().mean()))
        out[name] = r
    # depth_l1 end to end
    pv, pf = floor_mesh(max(2, a.side // 4))
    w2c, depth = TME.cameras(a.frames, dev)
    frames = [dict(depth=depth[t % 32], gt_w2c=w2c[t]) for t in range(a.frames)]
    box = torch.tensor([[-4.0, -4.0, 1.0], [4.0, 4.0, 2.0]], device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = E.depth_l1((pv, pf), (fv, ff), frames, TME.K, views=a.views, seed=0, gt_kept=box, device=dev)
    torch.cuda.synchronize()
    r["wall_s"] = time.perf_counter() - t0
    r["frames"] = a.frames
    out["depth_l1"] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
