"""GPU suite for the per-instance coverage masks (csrc/binning.cu, cover_mask) read back with sb_export_cover: every
(warp, Gaussian) pair with a pixel that blends has its bit set, every mask is a subset of the box test, and the masks
equal the numpy restatement (tools/lane_packing_model.py) wherever no decision lies within 1e-6 of its threshold.
Also in the sync-free mode with a binning capacity of exactly the instances the scene needs."""
import ctypes

import numpy as np
import pytest
import torch

import scenes
from test_cover_mask_cpu import M, blended_pairs

pytestmark = pytest.mark.gpu


def _export(sc, st, R, radii, dev):
    from splatam_b200 import _lib
    P, W, H = sc.P, sc.w, sc.h
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    t = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    depths, m2, co, tt = t(P, torch.float32), t((P, 2), torch.float32), t((P, 4), torch.float32), t(P, torch.int32)
    _lib.call("sb_export_geometry", P, st.geom, st.geom.numel(), depths, m2, co, tt, device=dev)
    lst, ranges = t(max(R, 1), torch.int32), t((tiles, 2), torch.int32)
    _lib.call("sb_export_binning", ctypes.byref(st.settings.c), P, R, st.geom, st.geom.numel(), st.binning,
              st.binning.numel(), st.image, st.image.numel(), None, lst, ranges, None, None, device=dev)
    cover = t(max(R, 1), torch.uint8)
    _lib.call("sb_export_cover", ctypes.byref(st.settings.c), R, st.binning, st.binning.numel(), cover, device=dev)
    torch.cuda.synchronize(dev)
    return dict(radii=radii.cpu().numpy(), means2D=m2.cpu().numpy(), conic_opacity=co.cpu().numpy(),
                point_list=lst.cpu().numpy().view(np.uint32)[:R], ranges=ranges.cpu().numpy().view(np.uint32),
                cover=cover.cpu().numpy()[:R])


def _check(sc, ex, n_tiles=60, seed=0):
    xy, co, radii, plist, ranges = ex["means2D"], ex["conic_opacity"], ex["radii"], ex["point_list"], ex["ranges"]
    cover = ex["cover"]
    grid_x = (sc.w + 15) // 16
    R = plist.size
    tile = np.empty(R, np.int64)
    for t in np.nonzero(ranges[:, 1] > ranges[:, 0])[0]:
        tile[ranges[t, 0]:ranges[t, 1]] = t
    hx, hy = M.cull_half_extents_f32(co[:, :3], co[:, 3], radii)
    mask, box, near = M.cover_masks(xy[plist], co[plist, :3], hx[plist], hy[plist], tile, grid_x)
    assert not (cover & ~(box | near)).any(), "a device coverage bit outside the box test"
    diff = (cover ^ mask) & ~near
    assert not diff.any(), "%d instances differ from the restatement away from a threshold" % int((diff != 0).sum())
    nonempty = np.nonzero(ranges[:, 1] > ranges[:, 0])[0]
    rng = np.random.default_rng(seed)
    for t in (nonempty if nonempty.size <= n_tiles else rng.choice(nonempty, size=n_tiles, replace=False)):
        lo, hi = int(ranges[t, 0]), int(ranges[t, 1])
        ids = plist[lo:hi]
        blend = blended_pairs(xy[ids], co[ids], np.full(ids.shape, t), grid_x, sc.w, sc.h)
        assert not (blend & ~cover[lo:hi]).any(), "tile %d: a blended pair with its coverage bit clear" % t


def _render(sc, dev):
    import splatam_b200 as S
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    inp = sc.inputs(dev, requires_grad=True)
    color, radii, _ = S.GaussianRasterizer(rs)(**inp)
    st = color.grad_fn.state
    return _export(sc, st, st.num_rendered, radii, dev)


SCENES = {"config3": lambda: scenes.config3(), "view_filling": lambda: scenes.view_filling(),
          "view_filling_aniso": lambda: scenes.view_filling(anisotropic=True)}
SCENES.update(scenes.adversarial())


@pytest.mark.parametrize("name", sorted(SCENES))
def test_device_masks_cover_blended_pairs_and_match_the_restatement(name, cuda_device):
    sc = SCENES[name]()
    _check(sc, _render(sc, cuda_device))


def test_sync_free_masks_at_exact_capacity(cuda_device):
    import splatam_b200 as S
    dev = cuda_device
    sc = scenes.view_filling(anisotropic=True)
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    inp = sc.inputs(dev)
    R = S.GaussianRasterizer(rs).num_rendered(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"])
    color, radii, _ = S.GaussianRasterizer(rs, max_rendered=R)(**inp)
    n_r, overflow = S.GaussianRasterizer.last_counts(dev)
    assert n_r == R and not overflow and not torch.isnan(color).any()
    _check(sc, _export(sc, S.GaussianRasterizer.last_state(dev), R, radii, dev))
