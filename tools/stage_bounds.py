"""Per-stage HBM floors of the rasterizer's streaming stages against their measured time on one GPU, and prints the
card's name and power limit first.

For one `bench.py` workload (the scene comes from bench.make_scene, i.e. scenes.py) it
(a) times every stage of the eager operator (forward + backward with a dense dL/dcolor) with sb_profile_begin/end, the
    CUDA events bench.py's profile pass uses, mean over `--steps` steps;
(b) counts, from the measured R (tile instances) and V (Gaussians with radius > 0), the bytes each streaming stage has
    to move: the algorithmic bytes, and the sector-level bytes (a random 4-16 B load costs one 32-B sector; a random
    12-B colour row 1.25 sectors on average), and prints the achieved GB/s and the fraction of the H100 SXM data sheet's
    3.35 TB/s (not a measured peak) for both;
(c) builds, in a temporary directory, a variant of the library whose project_kernel computes everything but stores
    nothing except radii (project.cu compiled with -DSB_PROBE_PROJECT_RADII_ONLY, linked with the objects `make`
    left in splatam_b200/csrc), and times the project stage of both libraries through sb_forward_geometry.  The
    variant's time is the projection's arithmetic and input traffic without its geometry stores.

Byte model (per launch; DESIGN.md section 5), the workspace layout of DESIGN.md section 2:
  project            44 P in; radii 4 + depth key 4 + tile count 4 for every Gaussian, 32-B geometry + 8-B rect for V
  emit_instances     sorted_idx + offsets 8 P, the 8-B rect of each of the V Gaussians (1 sector), 8 R out
  ranges_records     tile_sorted + point_list 8 R, 32-B geometry (1 sector), colour 12 B (1.25 sectors), 48 R out
  geometry_backward  radii 4 P; accum 48 + inputs 40 for V; 68 P out

Needs a CUDA device; there is no CPU path.
Run:  python tools/stage_bounds.py [--workload config3] [--steps 100]"""
import argparse
import ctypes
import glob
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from gpu_info import gpu_info  # noqa: E402

PEAK_GBS = 3350.0


def stage_bytes(P, V, R):
    """{stage: (algorithmic bytes, sector-level bytes)} per launch of the single-colour-set eager operator."""
    return {
        "project": (44 * P + 12 * P + 40 * V,) * 2,
        "emit_instances": (8 * P + 8 * V + 8 * R, 8 * P + 32 * V + 8 * R),
        "ranges_records": (8 * R + 32 * R + 12 * R + 48 * R, 8 * R + 32 * R + 40 * R + 48 * R),
        "geometry_backward": (4 * P + 88 * V + 68 * P,) * 2,
    }


def profiled(lib, fn, steps):
    """Mean ms per call of every sb_profile stage over `steps` calls of fn()."""
    names = [lib.sb_stage_name(i).decode() for i in range(10)]
    lib.sb_profile_begin()
    for _ in range(steps):
        fn()
    ms, calls = (ctypes.c_float * 10)(), (ctypes.c_int * 10)()
    rc = lib.sb_profile_end(ms, calls)
    assert rc == 0, "sb_profile_end failed"
    return {n: ms[i] / max(calls[i], 1) for i, n in enumerate(names)}


def run_quiet(cmd):
    """Runs a compiler command; its output is printed only when it fails."""
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("failed: " + " ".join(cmd))


def build_probe(tmp):
    """libsplatam_b200 with project.cu compiled as the radii-only variant, in tmp."""
    csrc = os.path.join(ROOT, "splatam_b200", "csrc")
    objs = [cu[:-3] + ".o" for cu in sorted(glob.glob(os.path.join(csrc, "*.cu")))]
    missing = [o for o in objs if not os.path.exists(o)]
    assert not missing, "build the library first (make): missing %s" % missing
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    probe_o = os.path.join(tmp, "project_probe.o")
    run_quiet([nvcc, "-O3", "-std=c++17", *arch, "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
               "--expt-relaxed-constexpr", "-DSB_PROBE_PROJECT_RADII_ONLY", "-c", os.path.join(csrc, "project.cu"),
               "-o", probe_o])
    so = os.path.join(tmp, "libprobe.so")
    objs = [probe_o if os.path.basename(o) == "project.o" else o for o in objs]
    run_quiet([nvcc, *arch, "-shared", "-o", so, *objs, "-lcudart_static", "-Xcompiler", "-fvisibility=hidden"])
    lib = ctypes.CDLL(so)
    from splatam_b200 import _lib
    for name in ("sb_forward_geometry", "sb_geometry_workspace_bytes"):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _lib._SIGNATURES[name]
    for name in ("sb_profile_begin", "sb_profile_end", "sb_stage_name"):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _lib._SIGNATURES[name]
    return lib


def project_time(lib, pack, inp, P, dev, steps):
    """Mean project-stage ms of `lib` over `steps` sb_forward_geometry calls (legacy default stream)."""
    n = ctypes.c_size_t(0)
    assert lib.sb_geometry_workspace_bytes(P, ctypes.byref(n)) == 0
    geom = torch.zeros(n.value, dtype=torch.uint8, device=dev)
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    R = ctypes.c_int(0)
    args = [ctypes.byref(pack.c), P] + [inp[k].data_ptr() for k in ("means3D", "opacities", "scales", "rotations")] + \
        [None, radii.data_ptr(), geom.data_ptr(), geom.numel(), ctypes.byref(R), None]
    torch.cuda.synchronize(dev)
    for _ in range(3):
        assert lib.sb_forward_geometry(*args) == 0
    return profiled(lib, lambda: lib.sb_forward_geometry(*args), steps)["project"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config3",
                    choices=["config3", "replica50k", "splatam816k", "tum3m", "room50k", "room3m"])
    ap.add_argument("--gaussians", type=int, default=0)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stage_bounds.py measures on a CUDA device; there is no CPU path"
    print(gpu_info(), flush=True)
    dev = torch.device("cuda", 0)
    scene, desc = bench.make_scene(args)
    import splatam_b200 as S
    from splatam_b200 import _lib
    from splatam_b200.rasterizer import _settings_pack
    step, inp, _, _ = bench.gpu_step_fn(scene, dev, S.GaussianRasterizer, S.GaussianRasterizationSettings, graph=False)
    for _ in range(5):
        color = step()
    torch.cuda.synchronize(dev)
    P, R = scene.P, int(color.grad_fn.state.num_rendered)
    _, radii, _ = S.GaussianRasterizer(scene.settings(S.GaussianRasterizationSettings, dev))(
        **{k: v.detach() for k, v in inp.items()})
    V = int((radii > 0).sum().item())
    lib = _lib.load()
    ms = profiled(lib, step, args.steps)
    bytes_ = stage_bytes(P, V, R)

    print("%s  P=%d V=%d R=%d, mean of %d eager steps" % (desc, P, V, R, args.steps))
    print("%-18s %9s %10s %10s %8s %8s %10s %7s" % ("stage", "ms", "alg MB", "sector MB", "alg GB/s", "frac",
                                                   "floor ms", "x floor"))
    rows = {}
    for name, t in ms.items():
        if name not in bytes_:
            print("%-18s %9.4f" % (name, t))
            continue
        alg, sec = bytes_[name]
        floor = sec / (PEAK_GBS * 1e9) * 1e3
        gbs = alg / (t * 1e-3) / 1e9
        rows[name] = dict(ms=round(t, 4), alg_bytes=alg, sector_bytes=sec, alg_gbs=round(gbs, 1),
                          frac=round(gbs / PEAK_GBS, 3), sector_frac=round(sec / (t * 1e-3) / 1e9 / PEAK_GBS, 3),
                          sector_floor_ms=round(floor, 4), over_floor=round(t / floor, 2))
        print("%-18s %9.4f %10.1f %10.1f %8.0f %8.3f %10.4f %7.2f" % (name, t, alg / 1e6, sec / 1e6, gbs,
                                                                      gbs / PEAK_GBS, floor, t / floor))

    pack = _settings_pack(scene.settings(S.GaussianRasterizationSettings, dev), dev)
    raw = {k: v.detach().contiguous() for k, v in inp.items()}
    with tempfile.TemporaryDirectory() as tmp:
        probe = build_probe(tmp)
        t_full = project_time(lib, pack, raw, P, dev, args.steps)
        t_probe = project_time(probe, pack, raw, P, dev, args.steps)
    print("project via sb_forward_geometry: %.4f ms with every store, %.4f ms storing radii only "
          "(the stores cost %.4f ms)" % (t_full, t_probe, t_full - t_probe))
    print(json.dumps(dict(tool="stage_bounds", gpu=gpu_info(), workload=desc, P=P, V=V, R=R, steps=args.steps,
                          peak_gbs=PEAK_GBS, peak_source="H100 SXM data sheet, not measured",
                          stage_ms={k: round(v, 4) for k, v in ms.items()}, streaming=rows,
                          project_probe=dict(all_stores_ms=round(t_full, 4), radii_only_ms=round(t_probe, 4)))))


if __name__ == "__main__":
    main()
