"""Times relocalisation (splatam_b200/reloc.py) on the GPU and prints one JSON line:

  thumbnails_ms          sb_reloc_thumbnails per 1200x680 frame (batch of 1 and of 32)
  score_us[N]            sb_reloc_score of one 85x48 query against N = 400, 2000, 10000 entries, with the byte bound
                         (N * 2 * 85 * 48 * 4 bytes read once, at 3.35 TB/s) and its share
  topk_us                sb_reloc_topk, k = 5 of 10000
  health_ms              sb_track_health at 1200x680 (kernel only); health_alternated_ms: it and sb_track_health_rgb
                         alternated three times; health_frame_ms: the depth/silhouette render of
                         the loop room at 320x192 plus the check and its host read, as run_slam pays per frame
  relocalise_ms          one reloc.relocalise call in the loop room at k = 5 (40 tracking iterations)
  slam_ms_per_frame      run_slam on scenes.write_replica_sequence (12 frames), relocalise=None and {} alternated twice

The card's name and power limit are read in the same call."""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def _events(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    import scenes
    import splatam_b200 as SB
    from splatam_b200 import reloc, slam
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = dict(gpu=smi[0] if smi else torch.cuda.get_device_name(dev))
    g = torch.Generator().manual_seed(0)
    H, W = 680, 1200
    for B in (1, 32):
        im = torch.rand(B, 3, H, W, generator=g).to(dev)
        d = (torch.rand(B, H, W, generator=g) * 3 + 0.5).to(dev)
        out["thumbnails_ms_per_frame_b%d" % B] = _events(lambda: reloc.thumbnails(im, d), 20) / B
    q = reloc.thumbnails(im[:1], d[:1])[0]
    out["score_us"] = {}
    for N in (400, 2000, 10_000):
        db = torch.rand(N, 2, 48, 85, generator=g).to(dev)
        us = 1e3 * _events(lambda: reloc.score(q, db), 50)
        bound = N * 2 * 48 * 85 * 4 / 3.35e12 * 1e6
        out["score_us"][N] = dict(us=round(us, 2), bound_us=round(bound, 2), share=round(bound / us, 3))
    s = reloc.score(q, db)
    out["topk_us"] = 1e3 * _events(lambda: reloc.topk(s, 5), 50)
    ds = torch.stack([d[0], torch.ones_like(d[0])])
    cfg = reloc.config({})
    out["health_ms"] = _events(lambda: reloc._health_of(ds, d[0], cfg), 50)
    cfg_rgb = reloc.config(dict(photometric=True))
    hm, hr = [], []
    for _ in range(3):                              # alternated: depth-only and photometric health
        hm.append(_events(lambda: reloc._health_of(ds, d[0], cfg), 50))
        hr.append(_events(lambda: reloc._health_rgb_of(ds, im[0], d[0], im[1], cfg_rgb), 50))
    out["health_alternated_ms"] = dict(depth=[round(x, 4) for x in hm], rgb=[round(x, 4) for x in hr])

    sc = scenes.loop_room()
    cam = sc.settings(SB.GaussianRasterizationSettings, dev)
    gt = {k: v.contiguous() for k, v in sc.splatam_params(dev).items()}
    rots, trans = scenes.loop_trajectory(81, dev)
    p = dict(gt, cam_unnorm_rots=rots.clone(), cam_trans=trans.clone())
    f = slam.render_frame(gt, rots, trans, 13, cam)
    f["depth"] = torch.where(f["sil"] > 0.9, f["depth"] / f["sil"].clamp(min=1e-6), torch.zeros_like(f["depth"]))
    del f["sil"]
    reloc.read_health(reloc.health(p, f, 13, cfg))
    t0 = time.perf_counter()
    for _ in range(20):
        reloc.read_health(reloc.health(p, f, 13, cfg))
    out["health_frame_ms"] = 1e3 * (time.perf_counter() - t0) / 20
    db = reloc.Database.from_record(dict(gt, cam_unnorm_rots=rots, cam_trans=trans), range(0, 81, 5), cam)
    K = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])
    lat = []
    for rep in range(4):
        q = dict(p, cam_unnorm_rots=rots.clone(), cam_trans=trans.clone())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rec = reloc.relocalise(q, f, 13, db, K, tracking=dict(num_iters=40))
        torch.cuda.synchronize()
        lat.append(1e3 * (time.perf_counter() - t0))
    out["relocalise_ms"] = dict(first=round(lat[0], 2), steady=round(float(np.median(lat[1:])), 2),
                                accepted=rec["accepted"])

    with tempfile.TemporaryDirectory() as tmp:
        scenes.write_replica_sequence(tmp + "/seq", 12, dev)
        from splatam_b200 import datasets
        K_r = None
        with datasets.RGBDSequence("replica", tmp, "seq", dict(camera_params=dict(
                image_height=680, image_width=1200, fx=600.0, fy=600.0, cx=599.5, cy=339.5, png_depth_scale=6553.5)),
                device=dev) as seq:
            frames = [seq[t] for t in range(len(seq))]
            K_r, cam_r = seq.intrinsics, seq.cam
        res = {"none": [], "on": []}
        for rep in range(2):
            for mode in ("none", "on"):
                init, radius = slam.initialize_map(frames[0], K_r)
                timing = {}
                torch.manual_seed(0); np.random.seed(0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                o = slam.run_slam(init, frames, cam_r, intrinsics=K_r, fused=True, tracking_iters=40, mapping_iters=12,
                                  first_frame_iters=12, add_new_gaussians=True, keyframe_every=5, timing=timing,
                                  relocalise=None if mode == "none" else {})
                torch.cuda.synchronize()
                res[mode].append(dict(ms_per_frame=round(1e3 * (time.perf_counter() - t0) / len(frames), 2),
                                      health_ms_per_frame=round(1e3 * timing.get("health_s", 0.0) / (len(frames) - 1),
                                                                3), lost=o.get("reloc_lost")))
        out["slam"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
