"""world_size-2 gloo test (CPU) of checkpoint / resume in the SLAM loop: only rank 0 writes the checkpoint files,
both ranks resume from them, and the resumed run equals the uninterrupted one on both ranks, with identical
`timestep` replicas.  The raster op is the float32 brute-force composite from oracle/."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenes
from util import cpu_render
from splatam_b200 import formats, slam

T = 6
PRUNE = dict(start_after=2, remove_big_after=0, stop_after=20, prune_every=1, removal_opacity_threshold=0.06,
             final_removal_opacity_threshold=0.06, reset_opacities=False, reset_opacities_every=500)
DENSIFY = dict(start_after=0, remove_big_after=0, stop_after=1, densify_every=2, grad_thresh=2e-6, num_to_split_into=2,
               removal_opacity_threshold=0.06, final_removal_opacity_threshold=0.06, reset_opacities=False,
               reset_opacities_every=100)


def _problem():
    import splatam_b200 as S
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    init = dict(gt)
    init["rgb_colors"] = (gt["rgb_colors"] + 0.2).clamp(0, 1)
    kw = dict(render=cpu_render, fused=False, tracking_iters=2, mapping_iters=3, keyframe_every=2, window=4,
              intrinsics=K, prune_dict=PRUNE, densify_dict=DENSIFY, scene_radius=0.5, select_keyframes=True, seed=3)
    return cam, frames, init, kw


def _pack(out):
    return dict(rots=out["rots"].numpy().copy(), trans=out["trans"].numpy().copy(),
                gauss={k: v.numpy().copy() for k, v in out["gauss"].items()}, timestep=out["timestep"].numpy().copy(),
                kti=list(out["keyframe_time_indices"]), counts=list(out["counts"]), psnr=out["psnr"])


def _worker(rank, world, port, root, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    cam, frames, init, kw = _problem()
    torch.manual_seed(1); np.random.seed(1)
    full = slam.run_slam(init, frames, cam, checkpoint_dir=os.path.join(root, "rank%d" % rank), checkpoint_every=2, **kw)
    dist.barrier()                                        # rank 0's files are complete
    ckpt = formats.load_checkpoint(os.path.join(root, "rank0"), 2, "cpu")
    torch.manual_seed(50 + rank); np.random.seed(50 + rank)
    resumed = slam.run_slam(None, frames, cam, resume=ckpt, **kw)
    q.put((rank, _pack(full), _pack(resumed)))
    dist.barrier()
    dist.destroy_process_group()


def _same(a, b):
    assert np.array_equal(a["rots"], b["rots"]) and np.array_equal(a["trans"], b["trans"])
    for k in a["gauss"]:
        assert np.array_equal(a["gauss"][k], b["gauss"][k]), k
    assert np.array_equal(a["timestep"], b["timestep"])
    assert a["kti"] == b["kti"] and a["counts"] == b["counts"] and a["psnr"] == b["psnr"]


def test_resume_on_two_ranks(tmp_path):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=600) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, full0, resumed0), (_, full1, resumed1) = res
    _same(full0, resumed0)
    _same(full1, resumed1)
    _same(full0, full1)                                  # the replicas, timestep included, are identical
    assert len(set(full0["counts"])) > 1
    names = {"params%d.npz" % t for t in (0, 2, 4)} | {"keyframe_time_indices%d.npy" % t for t in (0, 2, 4)}
    names |= {"run_state%d.npz" % t for t in (0, 2, 4)} | {"params.npz"}
    assert set(os.listdir(tmp_path / "rank0")) == names
    assert not (tmp_path / "rank1").exists()             # only rank 0 writes
