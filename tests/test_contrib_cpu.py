"""CPU suite for map compaction (splatam_b200/contrib.py, sb_blend_stats, tools/compact_record.py,
oracle/blend_stats_numpy.py): the entry point's argument checks, the counter guard, the keep rule, record handling
around the compaction kernels, the tool's arguments, and the oracle's statistics on hand-checkable stacks."""
import ctypes
import types

import numpy as np
import pytest
import torch

import scenes
from util import load
from splatam_b200 import _lib, contrib, formats


def test_blend_stats_is_exported():
    lib = _lib.load()
    assert "sb_blend_stats" in _lib.EXPORTED_SYMBOLS and hasattr(lib, "sb_blend_stats")
    assert lib.sb_abi_version() == 4


def test_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    s = _lib.SbSettings(64, 64, 0.5, 0.5, 1, 1.0, 1, 1, 0, None, 0)      # dummy pointers, never dereferenced
    n = ctypes.c_size_t(0)
    assert lib.sb_geometry_workspace_bytes(10, ctypes.byref(n)) == 0
    geom = n.value
    assert lib.sb_binning_workspace_bytes(100, 64, 64, 1, ctypes.byref(n)) == 0
    binning = n.value
    assert lib.sb_image_workspace_bytes(64, 64, ctypes.byref(n)) == 0
    image = n.value
    ok = lambda **kw: dict(dict(s=ctypes.byref(s), P=10, R=100, sf=0, g=1, gb=geom, b=1, bb=binning, i=1, ib=image,
                                bl=1, en=1, mw=1), **kw)
    call = lambda a: lib.sb_blend_stats(a["s"], a["P"], a["R"], a["sf"], a["g"], a["gb"], a["b"], a["bb"], a["i"],
                                        a["ib"], a["bl"], a["en"], a["mw"], None)
    assert call(ok(s=None)) == 1
    assert call(ok(P=-1)) == 1
    assert call(ok(R=-1)) == 1
    for k in ("g", "i", "b", "bl", "en", "mw"):            # null workspaces and statistic arrays
        assert call(ok(**{k: None})) == 1, k
    assert call(ok(gb=geom - 1)) == 2                       # SB_ERR_WORKSPACE
    assert call(ok(bb=binning - 1)) == 2
    assert call(ok(ib=image - 1)) == 2
    assert call(ok(P=0, g=None, b=None, i=None, bl=None, en=None, mw=None)) == 0      # empty map: nothing to do
    bad = _lib.SbSettings(0, 64, 0.5, 0.5, 1, 1.0, 1, 1, 0, None, 0)
    assert call(ok(s=ctypes.byref(bad))) == 1


def _fake_state(P, h=16, w=16):
    c = types.SimpleNamespace(image_height=h, image_width=w)
    return types.SimpleNamespace(P=P, settings=types.SimpleNamespace(c=c))


def test_counter_overflow_guard_raises():
    acc = contrib.BlendStats(4, "cpu")
    acc.reserve(5263, 680, 1200)                            # 4.29e9 pixels still fit in uint32
    with pytest.raises(ValueError, match="overflow"):
        acc.reserve(5264, 680, 1200)
    acc.pixels = contrib.COUNTER_MAX - 255
    with pytest.raises(ValueError, match="overflow"):       # one more 16x16 view could wrap: refused before any call
        acc.add(_fake_state(4))
    with pytest.raises(ValueError, match="statistics of 4"):
        contrib.BlendStats(4, "cpu").add(_fake_state(5))     # a render of another map
    with pytest.raises(ValueError):
        contrib.BlendStats(-1, "cpu")


def test_keep_rule_keeps_terminators_at_zero_weight():
    stats = dict(blended=torch.tensor([0, 3, 0, 0, 7]), ended=torch.tensor([0, 0, 2, 0, 1]),
                 max_weight=torch.tensor([0.0, 0.5, 0.0, 0.0, 0.01]))
    assert contrib.keep_mask(stats).tolist() == [False, True, True, False, True]      # ended-only Gaussian 2 stays
    assert contrib.keep_mask(stats, 0.01).tolist() == [False, True, False, False, True]
    assert contrib.keep_mask(stats, 0.02).tolist() == [False, True, False, False, False]
    with pytest.raises(ValueError):
        contrib.keep_mask(stats, -1.0)
    with pytest.raises(ValueError):
        contrib.keep_mask(stats, float("nan"))


def _synthetic_record(P=37, T=5, keyframes=True, seed=0):
    g = np.random.default_rng(seed)
    f = lambda *s: g.standard_normal(s).astype(np.float32)
    rec = dict(means3D=f(P, 3), rgb_colors=f(P, 3), unnorm_rotations=f(P, 4), logit_opacities=f(P, 1),
               log_scales=f(P, 1), cam_unnorm_rots=f(1, 4, T), cam_trans=f(1, 3, T),
               timestep=np.arange(P, dtype=np.float32), intrinsics=f(3, 3), w2c=f(4, 4),
               org_width=np.array(64, np.int64), org_height=np.array(48, np.int64), gt_w2c_all_frames=f(T, 4, 4))
    if keyframes:
        rec["keyframe_time_indices"] = np.array([0, 2, 4], np.int64)
    return rec


def _host_compaction(monkeypatch):
    """map_ops.compact_plan / compact_flat restated on the host, so the record handling runs without a GPU."""
    from splatam_b200 import map_ops

    def plan(mask):
        m = mask.to(torch.uint8)
        return m, torch.cumsum(m.to(torch.int64), 0).to(torch.int32) - m.to(torch.int32), int(m.sum())

    def flat(buf, P, widths, m8, dst, P_new):
        keep, out, off = m8.bool().numpy(), [], 0
        for w in widths:
            out.append(buf[off:off + w * P].reshape(P, w)[torch.from_numpy(keep)].reshape(-1))
            off += w * P
        assert sum(o.numel() for o in out) == sum(widths) * P_new
        return torch.cat(out)
    monkeypatch.setattr(map_ops, "compact_plan", plan)
    monkeypatch.setattr(map_ops, "compact_flat", flat)


@pytest.mark.parametrize("keyframes", [True, False], ids=["run-record", "offline-record"])
def test_record_compaction_copies_every_other_key(monkeypatch, keyframes):
    _host_compaction(monkeypatch)
    rec = _synthetic_record(keyframes=keyframes)
    keep = torch.from_numpy(np.random.default_rng(1).random(37) < 0.6)
    out = contrib.compact_arrays(rec, keep)
    assert list(out) == list(rec)
    k = keep.numpy()
    for key in rec:
        assert out[key].dtype == rec[key].dtype, key
        if key in contrib.PER_GAUSSIAN_KEYS:
            np.testing.assert_array_equal(out[key], rec[key][k])
        else:
            assert out[key].tobytes() == rec[key].tobytes() and out[key].shape == rec[key].shape, key
    none = contrib.compact_arrays(rec, torch.zeros(37, dtype=torch.bool))
    assert none["means3D"].shape == (0, 3) and none["timestep"].shape == (0,)
    with pytest.raises(ValueError):
        contrib.compact_arrays(rec, torch.ones(36, dtype=torch.bool))
    with pytest.raises(ValueError, match="float32"):
        contrib.compact_arrays(dict(rec, means3D=rec["means3D"].astype(np.float64)), keep)


def test_checkpoint_and_in_place_output_are_rejected(tmp_path):
    rec = _synthetic_record()
    ckpt = str(tmp_path / "params4.npz")
    np.savez(ckpt, **{k: rec[k] for k in formats.CHECKPOINT_KEYS})
    with pytest.raises(ValueError, match="timestep|intrinsics"):
        contrib.compact_record(ckpt, str(tmp_path / "out.npz"))
    full = str(tmp_path / "params.npz")
    np.savez(full, **rec)
    before = open(full, "rb").read()
    with pytest.raises(ValueError, match="differ"):
        contrib.compact_record(full, full)
    with pytest.raises(ValueError, match="differ"):
        contrib.compact_record(full, str(tmp_path / "." / "params.npz"))
    assert open(full, "rb").read() == before
    assert not (tmp_path / "out.npz").exists()


def test_tool_arguments(tmp_path):
    tool = load("tools/compact_record.py")
    rec = str(tmp_path / "params.npz")
    np.savez(rec, **_synthetic_record())
    a = tool.parse_args(["--record", rec, "--out", str(tmp_path / "c.npz")])
    assert (a.every, a.min_weight) == (1, 0.0)
    a = tool.parse_args(["--record", rec, "--out", str(tmp_path / "c.npz"), "--every", "5", "--min-weight", "0.02"])
    assert (a.every, a.min_weight) == (5, 0.02)
    for bad in (["--every", "0"], ["--min-weight", "-0.1"], ["--min-weight", "nan"]):
        with pytest.raises(SystemExit):
            tool.parse_args(["--record", rec, "--out", str(tmp_path / "c.npz")] + bad)
    with pytest.raises(SystemExit):
        tool.parse_args(["--record", rec, "--out", rec])
    with pytest.raises(SystemExit):
        tool.parse_args(["--record", str(tmp_path / "missing.npz"), "--out", str(tmp_path / "c.npz")])
    with pytest.raises(SystemExit):
        tool.parse_args(["--out", str(tmp_path / "c.npz")])


def _stack(opacities, w=16, h=16):
    """Gaussians of negligible 3D size on the camera axis, front to back, projected onto the centre of pixel (8, 8):
    the 0.3 px^2 screen-space dilation alone shapes them, so alpha = min(o, 0.99) at the centre, o exp(-5/3) at the
    4 edge neighbours, o exp(-10/3) at the 4 corners and < 1/255 further out."""
    n = len(opacities)
    z = torch.tensor([2.0 + 0.5 * i for i in range(n)])
    means = torch.stack([torch.zeros(n), torch.zeros(n), z], 1)
    return scenes.Scene("stack", w, h, 20.0, 20.0, 8.5, 8.5, means, torch.rand(n, 3, generator=torch.Generator().manual_seed(0)),
                        torch.tensor(opacities), torch.full((n, 3), 1e-4), torch.tensor([[1.0, 0, 0, 0]] * n))


def test_oracle_statistics_on_stacked_gaussians():
    from oracle import blend_stats_numpy as BS
    # two: the front one (alpha 0.99 at the centre) leaves T = 0.01, so the back one blends all 9 pixels
    st = BS.blend_stats(_stack([0.999, 0.5]).oracle())
    assert st["blended"].tolist() == [9, 9] and st["ended"].tolist() == [0, 0] and not st["flagged"].any()
    f32 = np.float32
    assert st["max_weight"][0] == f32(0.99)
    g = np.exp(-0.5 / 0.3)                                  # the edge neighbours, where the back one weighs most
    assert np.isclose(st["max_weight"][1], 0.5 * g * (1 - 0.999 * g), rtol=1e-4)
    # three: after 0.99 and 0.9 the centre has T = 1e-3, and the back one's 0.99 would leave 1e-5 < 1e-4: it ends that
    # walk and blends nothing there, but still blends its 8 neighbours, where T stays above 0.5
    st = BS.blend_stats(_stack([0.999, 0.9, 0.999]).oracle())
    assert st["blended"].tolist() == [9, 9, 8] and st["ended"].tolist() == [0, 0, 1] and not st["flagged"].any()
    # the oracle's walk agrees with the C oracle's render where both apply: a pixel is lit iff something blended
    o = _stack([0.999, 0.9, 0.999]).oracle()
    assert int((o.render()["n_contrib"] > 0).sum()) == 9
