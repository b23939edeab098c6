"""Run one raster fwd(+bwd) through (a) the product C-ABI path and (b) the unmodified reference
extension, returning numpy dicts with the same keys, intermediates included."""
import ctypes

import numpy as np
import torch

import splatam_b200 as S
from splatam_b200 import _lib
from splatam_b200 import rasterizer as RZ
from util import parse_reference_buffers, reference_extension

GRADS = ["means3D", "means2D", "colors", "opacities", "scales", "rotations"]


def run_ours(scene, dL=None, device="cuda:0", intermediates=True):
    dev = torch.device(device)
    rs = scene.settings(S.GaussianRasterizationSettings, dev)
    inp = scene.inputs(dev, requires_grad=dL is not None)
    rast = S.GaussianRasterizer(rs)
    color, radii, depth = rast(**inp)
    out = dict(color=color.detach().cpu().numpy(), radii=radii.cpu().numpy(), depth=depth.cpu().numpy())
    node = color.grad_fn
    if intermediates and dL is not None and scene.P > 0:
        st = node.state
        P, W, H, R = scene.P, scene.w, scene.h, st.num_rendered
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        t = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        depths, m2, co, tt = t(P, torch.float32), t((P, 2), torch.float32), t((P, 4), torch.float32), t(P, torch.int32)
        _lib.call("sb_export_geometry", P, st.geom, st.geom.numel(), depths, m2, co, tt, device=dev)
        keys, lst = t(max(R, 1), torch.int64), t(max(R, 1), torch.int32)
        ranges, fT, nc = t((tiles, 2), torch.int32), t((H, W), torch.float32), t((H, W), torch.int32)
        _lib.call("sb_export_binning", ctypes.byref(st.settings.c), P, R, st.geom, st.geom.numel(), st.binning,
                  st.binning.numel(), st.image, st.image.numel(), keys, lst, ranges, fT, nc, device=dev)
        torch.cuda.synchronize(dev)
        out.update(depths=depths.cpu().numpy(), means2D=m2.cpu().numpy(), conic_opacity=co.cpu().numpy(),
                   tiles_touched=tt.cpu().numpy().view(np.uint32), keys=keys.cpu().numpy().view(np.uint64)[:R],
                   point_list=lst.cpu().numpy().view(np.uint32)[:R], ranges=ranges.cpu().numpy().view(np.uint32),
                   final_T=fT.cpu().numpy(), n_contrib=nc.cpu().numpy().view(np.uint32), num_rendered=R)
    if dL is not None:
        color.backward(torch.as_tensor(dL, device=dev))
        out.update({"grad_" + k: inp[{"colors": "colors_precomp"}.get(k, k)].grad.cpu().numpy() for k in GRADS})
    return out


def run_ref(scene, dL=None, device="cuda:0"):
    ref = reference_extension()
    assert ref is not None
    dev = torch.device(device)
    rs = scene.settings(ref.GaussianRasterizationSettings, dev)
    inp = scene.inputs(dev, requires_grad=dL is not None)
    rast = ref.GaussianRasterizer(rs)
    color, radii, depth = rast(**inp)
    out = dict(color=color.detach().cpu().numpy(), radii=radii.cpu().numpy(), depth=depth.detach().cpu().numpy())
    if dL is not None and scene.P > 0:
        node = color.grad_fn
        saved = node.saved_tensors
        geom, binning, img = saved[7], saved[8], saved[9]
        R = node.num_rendered
        out.update(parse_reference_buffers(geom, binning, img, scene.P, R, scene.w, scene.h))
        out["num_rendered"] = R
    if dL is not None:
        color.backward(torch.as_tensor(dL, device=dev))
        out.update({"grad_" + k: inp[{"colors": "colors_precomp"}.get(k, k)].grad.cpu().numpy() for k in GRADS})
    return out


def random_dL(scene, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(3, scene.h, scene.w, generator=g).numpy()
