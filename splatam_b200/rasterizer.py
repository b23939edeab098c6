"""Host-side mirror of the reference operator API.

Same names, kwargs, return tuple and error behaviour as
``diff_gaussian_rasterization`` (reference: X/diff_gaussian_rasterization/__init__.py:17-196), but
every stage runs in the hand-written sm_90a kernels behind ``libsplatam_b200.so``; torch is only
used for device memory, the current stream and autograd bookkeeping.
"""
import contextlib
import ctypes
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib


class GaussianRasterizationSettings(NamedTuple):
    # field-for-field the reference's NamedTuple (__init__.py:134-145)
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool


def _given(t):
    """False for the reference's "not provided": None or an empty tensor (__init__.py:173-183)."""
    return t is not None and t.numel() != 0


def _f32c(t, name):
    if not _given(t):
        return t
    if not t.is_cuda:
        raise _lib.SplatamB200Error(f"{name} must be a CUDA tensor (there is no CPU fallback)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


class _SettingsPack:
    """sb_settings plus the tensors that keep its device pointers alive."""

    def __init__(self, rs: GaussianRasterizationSettings, device):
        self.bg = _f32c(rs.bg.to(device), "bg")
        self.view = _f32c(rs.viewmatrix.to(device), "viewmatrix")
        self.proj = _f32c(rs.projmatrix.to(device), "projmatrix")
        self.campos = _f32c(rs.campos.to(device), "campos") if rs.campos is not None else None
        self.c = _lib.SbSettings(
            int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy),
            self.bg.data_ptr(), float(rs.scale_modifier), self.view.data_ptr(), self.proj.data_ptr(),
            int(rs.sh_degree), _lib.ptr(self.campos), int(bool(rs.prefiltered)))


_PACK_CACHE = {}


def _settings_pack(rs, device):
    """sb_settings for a GaussianRasterizationSettings tuple, cached: SplaTAM builds the camera once per
    resolution (R/utils/recon_helpers.py:4-27) and passes the same tuple to every call.  The cache entry
    keeps the tuple alive (so ids stay unique) and is invalidated if a tensor is modified in place."""
    key = (id(rs), str(device))
    ver = (rs.bg._version, rs.viewmatrix._version, rs.projmatrix._version,
           rs.campos._version if isinstance(rs.campos, torch.Tensor) else -1)
    hit = _PACK_CACHE.get(key)
    if hit is not None and hit[0] is rs and hit[1] == ver:
        return hit[2]
    if len(_PACK_CACHE) > 64:
        _PACK_CACHE.clear()
    pack = _SettingsPack(rs, device)
    _PACK_CACHE[key] = (rs, ver, pack)
    return pack


_SIZE_CACHE = {}
_R_HINT = {}
_LAST_ASYNC_STATE = {}      # device index -> state of the most recent sync-free forward on that device
_STATE_SINKS = []           # the lists of the open `forward_states` blocks, innermost last


@contextlib.contextmanager
def forward_states():
    """Yields a list that collects, in call order, the workspace `_State` of every forward this module runs while the
    block is open (plain, two-set and sync-free alike), so a caller can read what a render left in its workspaces
    (e.g. contrib.BlendStats) without changing what the render returns.  A collected state keeps its workspaces
    alive until the list is dropped."""
    sink = []
    _STATE_SINKS.append(sink)
    try:
        yield sink
    finally:
        _STATE_SINKS.remove(sink)


def _sizes(P, W, H, sets):
    """(geometry, image, backward) workspace bytes of one problem shape."""
    key = (P, W, H, sets)
    hit = _SIZE_CACHE.get(key)
    if hit is None:
        if len(_SIZE_CACHE) > 256:
            _SIZE_CACHE.clear()
        hit = _SIZE_CACHE[key] = (_lib.nbytes("sb_geometry_workspace_bytes", P),
                                  _lib.nbytes("sb_image_workspace_bytes", W, H),
                                  _lib.nbytes("sb_backward_workspace_bytes", P, sets))
    return hit


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def _binning_ws(num_rendered, W, H, sets, device):
    return _ws(_lib.nbytes("sb_binning_workspace_bytes", num_rendered, W, H, sets), device)


class _State:
    """Scratch kept alive between forward and backward (the reference saves its three byte buffers
    on the autograd ctx, __init__.py:82-84)."""
    __slots__ = ("geom", "binning", "image", "num_rendered", "settings", "P", "sync_free")

    def header(self):
        """int32 view [num_rendered, num_visible, overflow flag] of the device-side counters (no synchronisation)."""
        return self.geom[:12].view(torch.int32)

    def counts(self):
        """(num_rendered, overflowed) of a sync-free forward; synchronises the current stream."""
        r, o = ctypes.c_int(0), ctypes.c_int(0)
        _lib.call("sb_read_counts", self.geom, self.geom.numel(), self.P, ctypes.byref(r), ctypes.byref(o),
                  device=self.geom.device)
        return r.value, bool(o.value)


def _forward_impl(means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                  colors2=None, capacity=None):
    """One or two colour sets (`colors2`) over one geometry.  Returns (color, color2 or None, radii, depth, state,
    saved): `saved` is the tuple of inputs _backward_impl reads, None where not provided."""
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        # rasterize_points.cu:56-58
        raise _lib.SplatamB200Error("means3D must have dimensions (num_points, 3)")
    device = means3D.device
    if not means3D.is_cuda:
        raise _lib.SplatamB200Error("means3D must be a CUDA tensor (there is no CPU fallback)")
    P = means3D.shape[0]
    H, W = int(raster_settings.image_height), int(raster_settings.image_width)
    means3D = _f32c(means3D, "means3D")
    colors_precomp = _f32c(colors_precomp, "colors_precomp")
    opacities = _f32c(opacities, "opacities")
    scales = _f32c(scales, "scales")
    rotations = _f32c(rotations, "rotations")
    cov3Ds_precomp = _f32c(cov3Ds_precomp, "cov3D_precomp")
    colors2 = _f32c(colors2, "colors_extra")
    sets = 2 if colors2 is not None else 1

    pack = _settings_pack(raster_settings, device)
    color = torch.empty((3, H, W), dtype=torch.float32, device=device)
    depth = torch.empty((1, H, W), dtype=torch.float32, device=device)
    radii = torch.empty((P,), dtype=torch.int32, device=device)
    state = _State()
    state.settings = pack
    state.P = P
    state.sync_free = capacity is not None
    if _STATE_SINKS:
        _STATE_SINKS[-1].append(state)
    geom_bytes, img_bytes, _ = _sizes(P, W, H, sets)
    state.geom = _ws(geom_bytes, device)
    state.image = _ws(img_bytes, device)
    color2 = torch.empty((3, H, W), dtype=torch.float32, device=device) if sets == 2 else None
    saved = (means3D, colors_precomp, scales, rotations, cov3Ds_precomp, colors2)
    if capacity is not None:
        # sync-free mode: fixed-capacity binning workspace, num_rendered stays on the device (CUDA-graph safe)
        capacity = int(capacity)
        state.binning = _binning_ws(capacity, W, H, sets, device)
        _lib.call("sb_forward_async", ctypes.byref(pack.c), P, means3D, opacities, scales, rotations, cov3Ds_precomp,
                  colors_precomp, colors2, radii, state.geom, state.geom.numel(), state.binning, state.binning.numel(),
                  capacity, state.image, state.image.numel(), color, color2, depth, device=device)
        state.num_rendered = capacity
        _LAST_ASYNC_STATE[device.index] = state
        return color, color2, radii, depth, state, saved
    # binning workspace sized from the last num_rendered seen for this problem shape (+12 % slack): the
    # whole forward is then ONE library call and the GPU only waits for the num_rendered read-back itself
    hint_key = (P, W, H, sets, device.index)
    hint = _R_HINT.get(hint_key, 0)
    state.binning = _binning_ws(int(hint * 1.125) + 4096, W, H, sets, device) if hint > 0 else None
    R = ctypes.c_int(0)
    p = _lib.ptr
    with _lib.on_device(device):
        # called directly, not through _lib.call: SB_ERR_BINNING_TOO_SMALL is a status to act on, not a failure
        rc = _lib.load().sb_forward(
            ctypes.byref(pack.c), P, p(means3D), p(opacities), p(scales), p(rotations), p(cov3Ds_precomp),
            p(colors_precomp), p(colors2), p(radii), p(state.geom), state.geom.numel(), p(state.binning),
            0 if state.binning is None else state.binning.numel(), p(state.image), state.image.numel(), p(color),
            p(color2), p(depth), ctypes.byref(R), _lib.stream(device))
    if rc == 5:      # SB_ERR_BINNING_TOO_SMALL: stage 1 is done, the guess was too small -> size exactly and finish
        state.binning = _binning_ws(R.value, W, H, sets, device)
        _lib.call("sb_forward_render", ctypes.byref(pack.c), P, R.value, colors_precomp, colors2, state.geom,
                  state.geom.numel(), state.binning, state.binning.numel(), state.image, state.image.numel(), color,
                  color2, depth, device=device)
    else:
        _lib.check(rc, "sb_forward")
    if state.binning is None:
        state.binning = _ws(16, device)
    state.num_rendered = R.value
    _R_HINT[hint_key] = R.value
    if len(_R_HINT) > 256:
        _R_HINT.clear()
    return color, color2, radii, depth, state, saved


def _backward_impl(state, saved, radii, grad_out_color, grad_out_color2=None):
    """Gradients (means3D, means2D, colors, colors2, opacities, scales, rotations, cov3D) of the forward that made
    `state` and `saved`; colors2 is None for one colour set, cov3D is None unless cov3D_precomp was given, scales
    and rotations are zeros when it was."""
    means3D, colors_precomp, scales, rotations, cov3Ds_precomp, colors2 = saved
    sets = 2 if colors2 is not None else 1
    device = means3D.device
    P = means3D.shape[0]
    pack = state.settings
    grad_out_color = _f32c(grad_out_color, "grad_out_color")
    grad_out_color2 = _f32c(grad_out_color2, "grad_out_color2")
    e = lambda *shape: torch.empty(shape, dtype=torch.float32, device=device)
    g_means3D, g_means2D, g_colors, g_opac = e(P, 3), e(P, 3), e(P, 3), e(P, 1)
    have_sr = _given(scales)
    g_scales = e(P, 3) if have_sr else torch.zeros((P, 3), dtype=torch.float32, device=device)
    g_rot = e(P, 4) if have_sr else torch.zeros((P, 4), dtype=torch.float32, device=device)
    g_cov3D = None if have_sr else e(P, 6)     # only the cov3D_precomp branch has a consumer for it
    g_colors2 = e(P, 3) if sets == 2 else None
    bwd_ws = _ws(_sizes(P, int(pack.c.image_width), int(pack.c.image_height), sets)[2], device)
    _lib.call("sb_backward", ctypes.byref(pack.c), P, state.num_rendered, means3D, colors_precomp, scales, rotations,
              cov3Ds_precomp, radii, state.geom, state.geom.numel(), state.binning, state.binning.numel(), state.image,
              state.image.numel(), bwd_ws, bwd_ws.numel(), grad_out_color, grad_out_color2, g_means3D, g_means2D,
              g_colors, g_colors2, g_opac, g_scales if have_sr else None, g_rot if have_sr else None, g_cov3D,
              device=device)
    return g_means3D, g_means2D, g_colors, g_colors2, g_opac, g_scales, g_rot, g_cov3D


def _sh_forward(sh, means3D, raster_settings):
    """SH colours -> rgb for the colours-precomp path (forward.cu:241-247).  Returns (rgb, what _sh_backward needs)."""
    sh_c = _f32c(sh, "shs")
    m_c = _f32c(means3D, "means3D")
    P, M = sh_c.shape[0], sh_c.shape[1]
    deg = int(raster_settings.sh_degree)
    rgb = torch.empty((P, 3), dtype=torch.float32, device=m_c.device)
    clamped = torch.empty((P,), dtype=torch.uint8, device=m_c.device)
    campos = _f32c(raster_settings.campos.to(m_c.device), "campos")
    _lib.call("sb_sh_forward", P, deg, M, m_c, campos, sh_c, rgb, clamped, device=m_c.device)
    return rgb, (sh_c, clamped, campos, M, deg, sh.shape)


def _sh_backward(sh_saved, means3D, radii, g_colors, g_means3D):
    """dL/dshs from dL/drgb; adds the view-direction term to g_means3D in place."""
    sh_c, clamped, campos, M, deg, sh_shape = sh_saved
    P = means3D.shape[0]
    g_sh = torch.empty((P, M, 3), dtype=torch.float32, device=means3D.device)
    _lib.call("sb_sh_backward", P, deg, M, means3D, campos, sh_c, clamped, g_colors, radii, g_sh, g_means3D,
              device=means3D.device)
    return g_sh.reshape(sh_shape)


class _RasterizeGaussians(torch.autograd.Function):
    """autograd node with the reference's argument order and gradient tuple (__init__.py:40-132)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, capacity=None):
        ctx.empty = means3D.shape[0] == 0
        if ctx.empty:
            H, W = int(raster_settings.image_height), int(raster_settings.image_width)
            dev = means3D.device
            ctx.dev = dev
            ctx.shapes = (means3D.shape, means2D.shape, colors_precomp.shape, opacities.shape, scales.shape,
                          rotations.shape)
            # rasterize_points.cu:67-75,81: P == 0 returns the zero-filled images without launching
            return (torch.zeros((3, H, W), device=dev), torch.zeros((0,), dtype=torch.int32, device=dev),
                    torch.zeros((1, H, W), device=dev))
        ctx.sh = None
        if _given(sh):
            colors_precomp, ctx.sh = _sh_forward(sh, means3D, raster_settings)
        color, _, radii, depth, ctx.state, saved = _forward_impl(
            means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, capacity=capacity)
        ctx.opac_shape = opacities.shape
        ctx.save_for_backward(radii, *saved)
        ctx.mark_non_differentiable(radii, depth)
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii, _grad_depth):
        # depth carries no gradient (the reference drops it, __init__.py:88)
        if ctx.empty:
            z = [torch.zeros(s, device=ctx.dev) for s in ctx.shapes]
            return z[0], z[1], None, z[2], z[3], z[4], z[5], None, None, None
        radii, *saved = ctx.saved_tensors
        g_means3D, g_means2D, g_colors, _, g_opac, g_scales, g_rot, g_cov3D = _backward_impl(
            ctx.state, saved, radii, grad_out_color)
        g_sh = None
        if ctx.sh is not None:
            g_sh, g_colors = _sh_backward(ctx.sh, saved[0], radii, g_colors, g_means3D), None
        needs_cov = _given(saved[4])
        return (g_means3D, g_means2D, g_sh, g_colors, g_opac.reshape(ctx.opac_shape),
                g_scales if not needs_cov else None, g_rot if not needs_cov else None,
                g_cov3D if needs_cov else None, None, None)


class _RasterizeGaussiansFused(torch.autograd.Function):
    """Two colour sets over one geometry in one pass (SURVEY.md 8(f) N1): returns (color, color_extra, radii,
    depth).  Equivalent to two _RasterizeGaussians calls that share every input except colors_precomp;
    the means2D gradient carries the first set's share only (SplaTAM's densification statistic)."""

    @staticmethod
    def forward(ctx, means3D, means2D, colors_precomp, colors_extra, opacities, scales, rotations, raster_settings,
                capacity=None):
        if means3D.shape[0] == 0:
            raise _lib.SplatamB200Error("fused render needs at least one Gaussian")
        color, color2, radii, depth, ctx.state, saved = _forward_impl(
            means3D, colors_precomp, opacities, scales, rotations, None, raster_settings, colors2=colors_extra,
            capacity=capacity)
        ctx.opac_shape = opacities.shape
        ctx.save_for_backward(radii, *saved)
        ctx.mark_non_differentiable(radii, depth)
        return color, color2, radii, depth

    @staticmethod
    def backward(ctx, grad_color, grad_color2, _grad_radii, _grad_depth):
        radii, *saved = ctx.saved_tensors
        if grad_color is None:
            grad_color = torch.zeros_like(grad_color2)
        if grad_color2 is None:
            grad_color2 = torch.zeros_like(grad_color)
        g_means3D, g_means2D, g_colors, g_colors2, g_opac, g_scales, g_rot, _ = _backward_impl(
            ctx.state, saved, radii, grad_color, grad_color2)
        return (g_means3D, g_means2D, g_colors, g_colors2, g_opac.reshape(ctx.opac_shape), g_scales, g_rot, None, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, capacity=None):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, capacity)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings, max_rendered=None):
        """`max_rendered` (extension): fixed capacity, in tile instances, of the binning workspace.  When given,
        the forward never synchronises with the host (num_rendered stays on the device) and forward + backward
        can be captured into a CUDA graph; `last_counts()` reports the true count and whether it overflowed."""
        super().__init__()
        self.raster_settings = raster_settings
        self.max_rendered = max_rendered

    @staticmethod
    def last_state(device=None):
        """Workspace state of the most recent sync-free forward on `device` (default: the current device)."""
        idx = torch.cuda.current_device() if device is None else torch.device(device).index
        return _LAST_ASYNC_STATE.get(idx)

    @staticmethod
    def last_counts(device=None):
        """(num_rendered, overflowed) of the most recent sync-free forward on `device` (default: the current
        device); synchronises.  On overflow the images of that forward are NaN."""
        st = GaussianRasterizer.last_state(device)
        return None if st is None else st.counts()

    def num_rendered(self, means3D, opacities, scales, rotations):
        """Tile instances a render of these Gaussians bins, from the forward's first stage alone (sb_forward_geometry:
        projection and depth ordering, the count a synchronous forward renders with); synchronises."""
        dev, P = means3D.device, means3D.shape[0]
        pack = _settings_pack(self.raster_settings, dev)
        geom = _ws(_lib.nbytes("sb_geometry_workspace_bytes", P), dev)
        R = ctypes.c_int(0)
        _lib.call("sb_forward_geometry", ctypes.byref(pack.c), P, _f32c(means3D, "means3D"), _f32c(opacities, "opacities"),
                  _f32c(scales, "scales"), _f32c(rotations, "rotations"), None,
                  torch.empty((P,), dtype=torch.int32, device=dev), geom, geom.numel(), ctypes.byref(R), device=dev)
        return R.value

    def markVisible(self, positions):
        """Boolean mask ``view_z > 0.2`` per point (reference __init__.py:152-161)."""
        with torch.no_grad():
            rs = self.raster_settings
            pos = _f32c(positions, "positions")
            P = pos.shape[0]
            present = torch.zeros((P,), dtype=torch.bool, device=pos.device)
            if P:
                view = _f32c(rs.viewmatrix.to(pos.device), "viewmatrix")
                proj = _f32c(rs.projmatrix.to(pos.device), "projmatrix")
                _lib.call("sb_mark_visible", P, pos, view, proj, present, device=pos.device)
        return present

    def forward_fused(self, means3D, means2D, opacities, colors_precomp, colors_extra, scales, rotations):
        """One pass, two colour sets (e.g. SplaTAM's RGB and [depth, 1, depth^2]); see _RasterizeGaussiansFused."""
        return _RasterizeGaussiansFused.apply(means3D, means2D, colors_precomp, colors_extra, opacities, scales,
                                              rotations, self.raster_settings, self.max_rendered)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        raster_settings = self.raster_settings
        # the two argument checks of the reference, same exception type and text (__init__.py:167-171)
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if shs is None:
            shs = torch.Tensor([])
        if colors_precomp is None:
            colors_precomp = torch.Tensor([])
        if scales is None:
            scales = torch.Tensor([])
        if rotations is None:
            rotations = torch.Tensor([])
        if cov3D_precomp is None:
            cov3D_precomp = torch.Tensor([])
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, raster_settings, self.max_rendered)
