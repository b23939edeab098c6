"""CPU suite: the C-ABI library loads, exports every symbol include/splatam_b200.h declares, sizes
workspaces sanely, validates arguments, and FAILS LOUDLY (no CPU fallback) without a GPU."""
import ctypes
import os
import re

import pytest
import torch

from splatam_b200 import _lib
import splatam_b200 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "splatam_b200.h")).read()
    return sorted(set(re.findall(r"SB_API\s+(?:const\s+char\*|int|size_t)\s+(sb_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol_of_abi_4():
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(lib, name), name
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared, "python binding table out of sync with the header"
    assert lib.sb_abi_version() == 4
    assert lib.sb_status_string(0) == b"SB_OK" and lib.sb_status_string(3) == b"SB_ERR_CUDA"


def test_workspace_sizes_per_color_set():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_geometry_workspace_bytes(1_000_000, ctypes.byref(n)) == 0
    per_gaussian = n.value / 1e6
    assert 60 <= per_gaussian <= 84, per_gaussian           # 60 B/Gaussian + 8 B ping-pong pair + sort/scan temp
    assert lib.sb_binning_workspace_bytes(2_500_000, 1200, 680, 1, ctypes.byref(n)) == 0
    assert 64 <= n.value / 2.5e6 <= 76                      # 48-B records + 16 B of sort arrays + 8 B ping-pong pair
    one_set = n.value
    assert lib.sb_binning_workspace_bytes(2_500_000, 1200, 680, 2, ctypes.byref(n)) == 0
    assert n.value >= one_set + 16 * 2_500_000               # the second colour set adds a 16-B record per instance
    assert lib.sb_image_workspace_bytes(1200, 680, ctypes.byref(n)) == 0
    assert n.value >= 8 * 1200 * 680
    assert lib.sb_backward_workspace_bytes(10, 1, ctypes.byref(n)) == 0 and n.value >= 480
    assert lib.sb_backward_workspace_bytes(1000, 1, ctypes.byref(n)) == 0
    one_set = n.value
    assert lib.sb_backward_workspace_bytes(1000, 2, ctypes.byref(n)) == 0 and n.value > one_set   # wider accumulator rows
    assert lib.sb_geometry_workspace_bytes(-1, ctypes.byref(n)) == 1      # SB_ERR_BAD_ARG
    assert lib.sb_image_workspace_bytes(0, 10, ctypes.byref(n)) == 1
    assert lib.sb_geometry_workspace_bytes(5, None) == 1
    assert lib.sb_binning_workspace_bytes(100, 64, 64, 3, ctypes.byref(n)) == 1    # color_sets must be 1 or 2
    assert lib.sb_backward_workspace_bytes(10, 0, ctypes.byref(n)) == 1


def test_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    R = ctypes.c_int(123)
    assert lib.sb_forward_geometry(None, 10, None, None, None, None, None, None, None, 0, ctypes.byref(R), None) == 1
    s = _lib.SbSettings(64, 64, 0.5, 0.5, 1, 1.0, 1, 1, 0, None, 0)   # non-null dummy pointers, never dereferenced
    assert lib.sb_forward_geometry(ctypes.byref(s), 10, None, None, None, None, None, None, None, 0,
                                   ctypes.byref(R), None) == 1
    assert lib.sb_forward_geometry(ctypes.byref(s), 0, None, None, None, None, None, None, None, 0,
                                   ctypes.byref(R), None) == 0 and R.value == 0    # P == 0 fast path
    assert lib.sb_mark_visible(-1, None, None, None, None, None) == 1
    # map-maintenance and training entry points: every argument check comes before the first CUDA call
    assert lib.sb_prune_mask(-1, None, None, 1, 0.5, 0.0, None, None) == 1
    assert lib.sb_prune_mask(4, 1, 1, 2, 0.5, 0.0, 1, None) == 1            # scale_dim must be 1 or 3
    assert lib.sb_prune_mask(0, None, None, 1, 0.5, 0.0, None, None) == 0   # empty map: nothing to do
    n = ctypes.c_int(7)
    assert lib.sb_compact_plan(-1, None, None, None, 0, ctypes.byref(n), None) == 1
    assert lib.sb_compact_plan(0, None, None, None, 0, ctypes.byref(n), None) == 0 and n.value == 0
    assert lib.sb_compact_plan(5, None, None, None, 0, ctypes.byref(n), None) == 1
    w = (ctypes.c_int * 2)(3, 0)
    assert lib.sb_compact_flat(4, 2, 1, 1, 2, w, 1, 1, None) == 1          # zero-width segment
    assert lib.sb_compact_flat(4, 5, 1, 1, 1, w, 1, 1, None) == 1          # P_new > P
    assert lib.sb_compact_flat(4, 2, 1, 1, 0, w, 1, 1, None) == 1          # no segments
    assert lib.sb_new_gaussian_mask(0, 8, 1, 1, 0.5, 1.0, 1, None) == 1
    assert lib.sb_depth_error(8, 8, None, 1, 1, None) == 1
    c2w = (ctypes.c_float * 16)()
    assert lib.sb_backproject(8, 8, 1, 1, 1.0, 1.0, 0.0, 0.0, c2w, 1, None, 1, 1, 1, 1, None, None) == 1   # mask without plan
    assert lib.sb_backproject(8, 8, 1, 1, 1.0, 1.0, 0.0, 0.0, c2w, None, None, 2, 1, 1, 1, None, None) == 1  # scale_dim
    lr = (ctypes.c_double * 1)(1e-3)
    end = (ctypes.c_uint32 * 1)(4)
    assert lib.sb_adam_step(1, 1, 1, 1, 4, end, lr, 1, 0, 0.9, 0.999, 1e-15, None) == 1                      # step counts from 1
    assert lib.sb_adam_step(1, 1, 1, 1, 4, end, lr, 17, 1, 0.9, 0.999, 1e-15, None) == 1                     # > 16 segments


def test_operator_argument_checks_match_reference():
    """Same two exceptions, same text, as the reference's GaussianRasterizer.forward (__init__.py:167-171)."""
    rs = S.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4)[None], torch.eye(4)[None],
                                         0, torch.zeros(3), False)
    assert rs._fields == ("image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
                          "projmatrix", "sh_degree", "campos", "prefiltered")
    r = S.GaussianRasterizer(rs)
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), scales=m, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), colors_precomp=m, scales=m)


def test_no_cpu_fallback():
    """CPU tensors must raise, never silently compute on the host."""
    rs = S.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4)[None], torch.eye(4)[None],
                                         0, torch.zeros(3), False)
    m = torch.zeros(4, 3)
    with pytest.raises(S.SplatamB200Error, match="no CPU fallback"):
        S.GaussianRasterizer(rs)(means3D=m, means2D=m, opacities=torch.zeros(4, 1), colors_precomp=m, scales=m,
                                 rotations=torch.zeros(4, 4))


def test_compat_alias_module():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "splatam_b200", "compat"))
    try:
        sys.modules.pop("diff_gaussian_rasterization", None)
        import diff_gaussian_rasterization as D
        assert D.GaussianRasterizer is S.GaussianRasterizer
        assert D.GaussianRasterizationSettings is S.GaussianRasterizationSettings
    finally:
        sys.path.pop(0)
        sys.modules.pop("diff_gaussian_rasterization", None)
