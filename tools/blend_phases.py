"""Where blend_backward's time goes, phase by phase, on one GPU; prints the card's name and power limit first.

It builds, in a temporary directory, a variant of the library whose blend_backward.cu is compiled with
-DSB_PROBE_BLEND_PHASES (linked with the objects `make` left in splatam_b200/csrc; the shipped library has no probe).
In that build every consumer warp of the backward sums clock64() deltas over its phases:
  wait      mbar_wait on the record ring (the TMA producer has not staged the next batch yet)
  gather    ballot-culling staged records by coverage bit and compacting survivors into the window
  evaluate  the lock-step G / alpha / skip pass over the window's slots
  chain     each lane's back-to-front T / A / dL/dalpha walk over its own contributors
  reduce    the per-slot moment and colour sums, the half-warp combine and the vector reductions
and each CTA records its %globaltimer start and end.  The tool runs the eager operator (forward + backward with the
bench's dense dL/dcolor) of one `bench.py` workload and writes one JSON line: the warp-cycles per phase summed over
the timed steps and their shares, the last launch's CTA span (first start to last end) and mean CTA duration, and the
probe build's blend_backward stage time (sb_profile events; the probe itself adds clock reads, so this time is a little
above the shipped kernel's).

--src takes another blend_backward.cu that defines the same probe (to attribute a change phase by phase, the
instrumented parent is measured the same way).  Needs a CUDA device; there is no CPU path.
Run:  python tools/blend_phases.py [--workload config3] [--steps 50] [--src FILE] [--label NAME] [--out FILE.jsonl]"""
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

PHASES = ("wait", "gather", "evaluate", "chain", "reduce")   # enum ProbePhase in blend_backward.cu
KERNEL = "blend_backward_kernel"


def run_quiet(cmd):
    """Runs a compiler command; its output is printed only when it fails."""
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("failed: " + " ".join(cmd))


def build_probe(tmp, src):
    """libsplatam_b200 with `src` compiled as the instrumented blend_backward, in tmp; returns its path."""
    csrc = os.path.join(ROOT, "splatam_b200", "csrc")
    objs = [cu[:-3] + ".o" for cu in sorted(glob.glob(os.path.join(csrc, "*.cu")))]
    missing = [o for o in objs if not os.path.exists(o)]
    assert not missing, "build the library first (make): missing %s" % missing
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    probe_o = os.path.join(tmp, "blend_backward_probe.o")
    run_quiet([nvcc, "-O3", "-std=c++17", *arch, "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
               "--expt-relaxed-constexpr", "-I", csrc, "-I", os.path.join(ROOT, "include"),
               "-DSB_PROBE_BLEND_PHASES", "-c", src, "-o", probe_o])
    so = os.path.join(tmp, "libsplatam_b200.so")
    objs = [probe_o if os.path.basename(o) == "blend_backward.o" else o for o in objs]
    run_quiet([nvcc, *arch, "-shared", "-o", so, *objs, "-lcudart_static", "-Xcompiler", "-fvisibility=hidden"])
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config3",
                    choices=["config3", "replica50k", "splatam816k", "tum3m", "room50k", "room3m"])
    ap.add_argument("--gaussians", type=int, default=0)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--src", default=os.path.join(ROOT, "splatam_b200", "csrc", "blend_backward.cu"))
    ap.add_argument("--label", default="this")
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "blend_phases.py measures on a CUDA device; there is no CPU path"
    gpu = gpu_info()
    print(gpu, flush=True)
    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp:
        so = build_probe(tmp, args.src)
        from splatam_b200 import _lib
        assert _lib._lib is None, "the library was loaded before the probe build"
        _lib.LIB_PATH = so
        lib = _lib.load()
        u64 = ctypes.c_ulonglong
        probe = lib.sb_probe_blend_phases
        probe.restype, probe.argtypes = ctypes.c_int, [ctypes.POINTER(u64)] * 3 + [ctypes.c_int]

        import splatam_b200 as S
        scene, desc = bench.make_scene(args)
        step, _, _, _ = bench.gpu_step_fn(scene, dev, S.GaussianRasterizer, S.GaussianRasterizationSettings,
                                          graph=False)
        for _ in range(5):
            color = step()
        torch.cuda.synchronize(dev)
        R = int(color.grad_fn.state.num_rendered)
        tiles = ((scene.w + 15) // 16) * ((scene.h + 15) // 16)
        cyc, t0, t1 = (u64 * len(PHASES))(), (u64 * tiles)(), (u64 * tiles)()
        assert probe(cyc, t0, t1, tiles) == 0                      # zeroes the phase totals
        names = [lib.sb_stage_name(i).decode() for i in range(10)]
        lib.sb_profile_begin()
        for _ in range(args.steps):
            step()
        ms, calls = (ctypes.c_float * 10)(), (ctypes.c_int * 10)()
        assert lib.sb_profile_end(ms, calls) == 0, "sb_profile_end failed"
        torch.cuda.synchronize(dev)
        assert probe(cyc, t0, t1, tiles) == 0
        stage_ms = {n: ms[i] / max(calls[i], 1) for i, n in enumerate(names)}

    total = sum(cyc)
    per_step = {p: cyc[i] / args.steps for i, p in enumerate(PHASES)}
    start, end = min(t0), max(t1)
    durs = [b - a for a, b in zip(t0, t1)]
    line = dict(tool="blend_phases", label=args.label, gpu=gpu, workload=desc, R=R, tiles=tiles, steps=args.steps,
                warp_cycles_per_step={p: round(v) for p, v in per_step.items()},
                share={p: round(cyc[i] / total, 4) for i, p in enumerate(PHASES)},
                cta_span_us=round((end - start) / 1e3, 2), cta_mean_us=round(sum(durs) / len(durs) / 1e3, 2),
                cta_max_us=round(max(durs) / 1e3, 2),
                probe_blend_backward_ms=round(stage_ms["blend_backward"], 4),
                src=os.path.relpath(os.path.abspath(args.src), ROOT))
    print("%s  R=%d, %d steps, probe build of %s" % (desc, R, args.steps, line["src"]))
    for p in PHASES:
        print("%-9s %14.0f warp-cycles/step %6.1f %%" % (p, per_step[p], 100.0 * line["share"][p]))
    print("CTA span %.1f us, mean CTA %.1f us, probe blend_backward %.4f ms" % (
        line["cta_span_us"], line["cta_mean_us"], line["probe_blend_backward_ms"]))
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(args.out, "a") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
