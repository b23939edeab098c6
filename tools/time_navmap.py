#!/usr/bin/env python
"""Times the navigation-map kernels on one GPU (csrc/navmap.cu) and prints one JSON line with the card's name and
power limit:

  * sb_nav_labels on 256^3 and 512^3 volumes
  * sb_esdf on 256^3 and 512^3 label grids, random (each sample occupied / free / unknown at random) and room-like
    (a closed box of walls, seen from inside, with unknown space behind the walls), both obstacle rules
  * sb_esdf_query of 1M and 16M random points in the room-like grid

Each time is the mean over --reps launches between device events, after warm-up launches.  Beside each is the bytes
the kernel has to move (the model below) and that traffic's time at 3.35 TB/s (the H100 SXM data sheet's HBM3
bandwidth) as a fraction of the measured time.

  python tools/time_navmap.py [--reps 20]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
import time_viewer as TV  # noqa: E402
from gpu_info import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


# bytes per sample (per point for the query) each kernel must read and write, whatever its algorithm:
#   labels   tsdf 4 + weight 4 in, label 1 out
#   esdf     pass x: the labels once per sign (2) in, both squared-distance buffers (8) out; pass y: both buffers in
#            and out (16); pass z: both buffers in (8), sd2 and esdf out (8).  The envelope stacks come on top: their
#            traffic depends on the map (one 8-B entry written and read back per site kept on a line's envelope).
#   query    the point 12 in, dist 4 + grad 12 out; the 8 corners are gathered from the esdf through the caches
MODEL = dict(labels=9, esdf=42, query=28)


def bound_fraction(kind, count, us):
    nbytes = MODEL[kind] * count
    return dict(us=us, bytes=nbytes, hbm_fraction=nbytes / HBM_BYTES_PER_S / (us * 1e-6))


def room_labels(n, dev):
    """A box room filling the middle 80 % of the grid: walls two samples thick are occupied, the inside free, the
    band behind the walls unknown (never seen), beyond it unknown too."""
    g = torch.arange(n, device=dev)
    lo, hi = int(0.1 * n), int(0.9 * n)
    inside = lambda a: (a > lo) & (a < hi)
    wall = lambda a: ((a >= lo - 1) & (a <= lo)) | ((a >= hi) & (a <= hi + 1))
    z, y, x = torch.meshgrid(g, g, g, indexing="ij")
    within = (x >= lo - 1) & (x <= hi + 1) & (y >= lo - 1) & (y <= hi + 1) & (z >= lo - 1) & (z <= hi + 1)
    lab = torch.zeros((n, n, n), dtype=torch.uint8, device=dev)
    lab[inside(x) & inside(y) & inside(z)] = 1
    lab[within & (wall(x) | wall(y) | wall(z))] = 2
    return lab


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    from splatam_b200 import _lib
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = dict(gpu=gpu_info(), model_bytes=MODEL)
    gen = torch.Generator(device=dev).manual_seed(0)
    for n in (256, 512):
        N = n ** 3
        tsdf = torch.rand((n, n, n), generator=gen, device=dev) * 2 - 1
        weight = (torch.rand((n, n, n), generator=gen, device=dev) * 3).floor()
        lab = torch.empty((n, n, n), dtype=torch.uint8, device=dev)
        us = TV.events_us(lambda: _lib.call("sb_nav_labels", n, n, n, tsdf, weight, 0.2, 1.0, 0.025, lab, device=dev),
                          a.reps)
        out["labels_%d" % n] = bound_fraction("labels", N, us)
        del tsdf, weight
        sd2 = torch.empty((n, n, n), dtype=torch.int32, device=dev)
        esdf = torch.empty((n, n, n), dtype=torch.float32, device=dev)
        nb = _lib.nbytes("sb_esdf_workspace_bytes", n, n, n)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        out["esdf_%d_workspace_bytes" % n] = nb
        for kind, labels in (("random", lab), ("room", room_labels(n, dev))):
            for uio in (1, 0):
                us = TV.events_us(lambda: _lib.call("sb_esdf", n, n, n, labels, 0.02, uio, ws, nb, sd2, esdf,
                                                    device=dev), a.reps)
                out["esdf_%d_%s_%s" % (n, kind, "unknown_obstacle" if uio else "unknown_free")] = \
                    bound_fraction("esdf", N, us)
        # the room grid with unknown space free was the last one built: query it
        for m in (1 << 20, 1 << 24):
            pts = torch.rand((m, 3), generator=gen, device=dev) * (0.02 * (n - 1))
            dist = torch.empty(m, dtype=torch.float32, device=dev)
            grad = torch.empty((m, 3), dtype=torch.float32, device=dev)
            us = TV.events_us(lambda: _lib.call("sb_esdf_query", n, n, n, 0.0, 0.0, 0.0, 0.02, esdf, m, pts, dist,
                                                grad, device=dev), a.reps)
            out["query_%d_%dM" % (n, m >> 20)] = bound_fraction("query", m, us)
            del pts, dist, grad
        del lab, sd2, esdf, ws
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
