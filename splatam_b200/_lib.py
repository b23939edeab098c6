"""ctypes binding of the C-ABI library (include/splatam_b200.h).

The product path has NO fallback: if ``libsplatam_b200.so`` is missing or fails to load, importing
the rasterizer raises.  Build it with ``python -c "import __graft_entry__ as g; g.build()"`` or ``make``.
Every wrapper module calls the library through ``call`` (and ``nbytes`` for size queries), the one place that turns
tensors into ABI arguments, picks the device and stream of a launch and reports a failed status.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsplatam_b200.so")

SB_OK = 0


class SbSettings(ctypes.Structure):
    """Mirror of ``sb_settings`` == GaussianRasterizationSettings
    (reference: diff_gaussian_rasterization/__init__.py:134-145)."""
    _fields_ = [
        ("image_height", ctypes.c_int32),
        ("image_width", ctypes.c_int32),
        ("tanfovx", ctypes.c_float),
        ("tanfovy", ctypes.c_float),
        ("bg", ctypes.c_void_p),
        ("scale_modifier", ctypes.c_float),
        ("viewmatrix", ctypes.c_void_p),
        ("projmatrix", ctypes.c_void_p),
        ("sh_degree", ctypes.c_int32),
        ("campos", ctypes.c_void_p),
        ("prefiltered", ctypes.c_int32),
    ]


class SplatamB200Error(RuntimeError):
    pass


_vp, _sz, _i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
_SIGNATURES = {
    # name: (restype, argtypes)  -- must list every symbol include/splatam_b200.h declares
    "sb_abi_version": (_i, []),
    "sb_status_string": (ctypes.c_char_p, [_i]),
    "sb_last_cuda_error": (ctypes.c_char_p, []),
    "sb_geometry_workspace_bytes": (_i, [_i, ctypes.POINTER(_sz)]),
    "sb_image_workspace_bytes": (_i, [_i, _i, ctypes.POINTER(_sz)]),
    "sb_binning_workspace_bytes": (_i, [_i, _i, _i, _i, ctypes.POINTER(_sz)]),
    "sb_backward_workspace_bytes": (_i, [_i, _i, ctypes.POINTER(_sz)]),
    "sb_forward_geometry": (_i, [ctypes.POINTER(SbSettings), _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz,
                                 ctypes.POINTER(_i), _vp]),
    "sb_forward": (_i, [ctypes.POINTER(SbSettings), _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _sz,
                        _vp, _sz, _vp, _vp, _vp, ctypes.POINTER(_i), _vp]),
    "sb_forward_async": (_i, [ctypes.POINTER(SbSettings), _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _sz,
                              _i, _vp, _sz, _vp, _vp, _vp, _vp]),
    "sb_read_counts": (_i, [_vp, _sz, _i, ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    "sb_forward_render": (_i, [ctypes.POINTER(SbSettings), _i, _i, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _sz,
                               _vp, _vp, _vp, _vp]),
    "sb_backward": (_i, [ctypes.POINTER(SbSettings), _i, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                         _vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz,
                         _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sb_mark_visible": (_i, [_i, _vp, _vp, _vp, _vp, _vp]),
    "sb_export_geometry": (_i, [_i, _vp, _sz, _vp, _vp, _vp, _vp, _vp]),
    "sb_adam_step": (_i, [_vp, _vp, _vp, _vp, _sz, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double), _i,
                          _i, ctypes.c_double, ctypes.c_double, ctypes.c_double, _vp]),
    "sb_adam_clock_bytes": (_sz, []),
    "sb_adam_step_guarded": (_i, [_vp, _vp, _vp, _vp, _sz, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double),
                                  _i, _vp, _vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, _vp]),
    "sb_image_loss_workspace_floats": (_sz, [_i, _i, _i]),
    "sb_image_loss_forward": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "sb_image_loss_backward": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, ctypes.c_float, ctypes.c_float, _vp, _vp]),
    "sb_prepare_forward": (_i, [_i, _i] + [_vp] * 12 + [_vp]),
    "sb_prepare_backward": (_i, [_i, _i, _i] + [_vp] * 18 + [_vp]),
    "sb_sh_forward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sb_sh_backward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sb_masked_l1_forward": (_i, [_vp, _vp, _vp, _vp, _i, _i, ctypes.c_float, _i, _vp, _vp]),
    "sb_masked_l1_backward": (_i, [_vp, _vp, _vp, _vp, _i, _i, ctypes.c_float, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sb_prune_mask": (_i, [_i, _vp, _vp, _i, ctypes.c_float, ctypes.c_float, _vp, _vp]),
    "sb_compact_plan_bytes": (_i, [_i, ctypes.POINTER(ctypes.c_size_t)]),
    "sb_compact_plan": (_i, [_i, _vp, _vp, _vp, _sz, ctypes.POINTER(ctypes.c_int), _vp]),
    "sb_compact_flat": (_i, [_i, _i, _vp, _vp, _i, ctypes.POINTER(ctypes.c_int), _vp, _vp, _vp]),
    "sb_densify_accumulate": (_i, [_i, _vp, _i, _vp, _vp, _vp, _vp]),
    "sb_depth_error": (_i, [_i, _i, _vp, _vp, _vp, _vp]),
    "sb_new_gaussian_mask": (_i, [_i, _i, _vp, _vp, ctypes.c_float, ctypes.c_float, _vp, _vp]),
    "sb_backproject": (_i, [_i, _i, _vp, _vp, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                            ctypes.POINTER(ctypes.c_float), _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "sb_frame_metrics_workspace_bytes": (_i, [_i, _i, ctypes.POINTER(_sz)]),
    "sb_frame_metrics": (_i, [_vp, _vp, _vp, _vp, _i, _i, ctypes.c_float, _i, _vp, _vp, _vp, _sz, _vp, _vp]),
    "sb_ms_ssim_workspace_bytes": (_i, [_i, _i, _i, _i, ctypes.POINTER(_sz)]),
    "sb_ms_ssim": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.c_double, _vp, _sz, _vp, _vp, _vp]),
    "sb_lpips_weights_floats": (_i, [ctypes.POINTER(_sz)]),
    "sb_lpips_workspace_bytes": (_i, [_i, _i, _i, ctypes.POINTER(_sz)]),
    "sb_lpips": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp, _vp, _vp]),
    "sb_eval_frames_u8": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "sb_ingest_rgbd": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, ctypes.c_double, _vp, _vp, _vp]),
    "sb_profile_begin": (_i, []),
    "sb_profile_end": (_i, [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)]),
    "sb_stage_name": (ctypes.c_char_p, [_i]),
    "sb_export_binning": (_i, [ctypes.POINTER(SbSettings), _i, _i, _vp, _sz, _vp, _sz, _vp, _sz,
                               _vp, _vp, _vp, _vp, _vp, _vp]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises if the CUDA library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SplatamB200Error(
            f"{LIB_PATH} is missing: the sm_90a CUDA library is not built "
            "(run `make` or `__graft_entry__.build()`); there is no CPU fallback")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.sb_abi_version() != 4:
        raise SplatamB200Error("libsplatam_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc, what):
    if rc != SB_OK:
        lib = load()
        name = lib.sb_status_string(rc).decode()
        detail = lib.sb_last_cuda_error().decode() if name == "SB_ERR_CUDA" else ""
        raise SplatamB200Error(f"{what} failed: {name} {detail}".strip())


def ptr(a):
    """ABI argument for `a`: a tensor's device pointer, or NULL for None or an empty tensor (the reference's "not
    provided", X/diff_gaussian_rasterization/__init__.py:173-183); anything else (ints, floats, byref out-parameters,
    host ctypes arrays) unchanged."""
    if isinstance(a, torch.Tensor):
        return a.data_ptr() if a.numel() else None
    return a


def stream(device):
    return torch.cuda.current_stream(device).cuda_stream


class on_device:
    """torch.cuda.device(dev) only when dev is not already current (the context manager costs ~10 us)."""

    def __init__(self, device):
        self.ctx = None if torch.cuda.current_device() == device.index else torch.cuda.device(device)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *a):
        if self.ctx is not None:
            self.ctx.__exit__(*a)


def call(name, *args, device=None):
    """Calls entry point `name` with every argument passed through `ptr`; raises SplatamB200Error on a non-zero
    status.  With `device`, that device is made current for the call and its current stream is appended as the
    trailing `void* stream`."""
    fn = getattr(load(), name)
    args = [ptr(a) for a in args]
    if device is None:
        check(fn(*args), name)
        return
    with on_device(device):
        check(fn(*args, stream(device)), name)


def nbytes(name, *args):
    """Size written by a `*_workspace_bytes` / `sb_compact_plan_bytes` query through its trailing size_t*."""
    n = ctypes.c_size_t(0)
    call(name, *args, ctypes.byref(n))
    return n.value


def need_cuda(what, *tensors):
    for t in tensors:
        if not t.is_cuda:
            raise SplatamB200Error(f"{what} needs CUDA tensors (there is no CPU fallback)")
