#!/usr/bin/env python
"""CPU-side cost of one mapping step (torch.profiler self CPU time per op) -- where the host overhead goes."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import scenes  # noqa: E402
import splatam_b200 as S  # noqa: E402
from splatam_b200 import mapping as M  # noqa: E402

dev = torch.device("cuda:0")
sc = scenes.room(seed=4, P=1_000_000)
cam = sc.settings(S.GaussianRasterizationSettings, dev)
g = torch.Generator().manual_seed(0)
gauss = sc.splatam_params(dev)
rots = torch.zeros(1, 4, 8); rots[:, 0] = 1.0
trans = 0.02 * torch.randn(1, 3, 8, generator=g)
frames = [dict(id=t, cam=cam, w2c=torch.eye(4, device=dev), im=torch.rand(3, sc.h, sc.w, generator=g).to(dev),
               depth=(1.0 + 2.0 * torch.rand(1, sc.h, sc.w, generator=g)).to(dev)) for t in range(8)]
mapper = M.ShardedMapper(gauss, rots.to(dev), trans.to(dev), seed=11, fused=True)
for _ in range(5):
    mapper.step(frames)
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(20):
    mapper.step(frames)
torch.cuda.synchronize()
print("wall ms/step", (time.perf_counter() - t0) / 20 * 1e3)
# pure host time: no sync at the end of the loop body except the one inside the forward
t0 = time.perf_counter()
for _ in range(20):
    mapper.step(frames)
print("host-issue ms/step", (time.perf_counter() - t0) / 20 * 1e3)
torch.cuda.synchronize()
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        mapper.step(frames)
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="self_cpu_time_total", row_limit=28, max_name_column_width=48))
