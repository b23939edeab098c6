"""CPU suite of tools/extract_mesh.py's input frames and of the limits around mesh_record: --source input selects the
run's frames with run_slam_dataset.py's flags and refuses a selection whose length differs from the record's camera
count, RecordFusion refuses such a source before any device work, and volumes stay within what marching cubes can
count."""
import ctypes

import numpy as np
import pytest

from util import load
from splatam_b200 import _lib, formats
from splatam_b200.mesh import MC_MAX_SAMPLES, RecordFusion, TSDFVolume


def _record(tmp_path, T, width=64, height=48):
    P = 10
    g = np.random.default_rng(0)
    gauss = dict(means3D=g.normal(size=(P, 3)), rgb_colors=g.uniform(size=(P, 3)), unnorm_rotations=g.normal(size=(P, 4)),
                 logit_opacities=g.normal(size=(P, 1)), log_scales=g.normal(size=(P, 1)))
    rots = np.zeros((1, 4, T), np.float32)
    rots[0, 0] = 1
    K = np.array([[50.0, 0, 31.5], [0, 50.0, 23.5], [0, 0, 1]])
    return formats.save_run_record(str(tmp_path), gauss, rots, np.zeros((1, 3, T)), np.zeros(P), K, np.eye(4), width,
                                   height, [np.eye(4)] * T, [0])


class _FakeSequence:
    """Stands in for datasets.RGBDSequence: records its arguments and selects `n` frames."""
    made = []

    def __init__(self, dataset, basedir, sequence, config=None, **kw):
        self.args = dict(dataset=dataset, basedir=basedir, sequence=sequence, config=config, **kw)
        self.closed = False
        _FakeSequence.made.append(self)

    def __len__(self):
        return _FakeSequence.n

    def __getitem__(self, t):
        return dict(id=t)

    def close(self):
        self.closed = True


@pytest.fixture
def fake_sequence(monkeypatch):
    from splatam_b200 import datasets
    _FakeSequence.made = []
    monkeypatch.setattr(datasets, "RGBDSequence", _FakeSequence)
    monkeypatch.setattr(datasets, "load_config", lambda path: {"from": path})
    return _FakeSequence


def test_parser_takes_the_run_flags_and_keeps_them_to_input(tmp_path):
    tool = load("tools/extract_mesh.py")
    rec = _record(tmp_path, 4)
    a = tool.parse_args(["--record", rec, "--out", "m.ply", "--source", "input", "--dataset", "replica", "--basedir",
                         "d", "--sequence", "room0", "--config", "c.yaml", "--start", "100", "--end", "400",
                         "--stride", "2", "--frames", "50"])
    assert (a.config, a.start, a.end, a.stride, a.frames) == ("c.yaml", 100, 400, 2, 50)
    for extra in (["--stride", "2"], ["--start", "5"], ["--frames", "3"], ["--dataset", "replica"]):
        with pytest.raises(SystemExit):
            tool.parse_args(["--record", rec, "--out", "m.ply"] + extra)       # render: no input frames to select
    with pytest.raises(SystemExit):
        tool.parse_args(["--record", rec, "--out", "m.ply", "--source", "input", "--dataset", "replica"])


def _input_args(tool, rec, *extra):
    return tool.parse_args(["--record", rec, "--out", "m.ply", "--source", "input", "--dataset", "replica",
                            "--basedir", "d", "--sequence", "room0"] + list(extra))


def test_open_input_forwards_the_selection_at_the_record_size(tmp_path, fake_sequence):
    tool = load("tools/extract_mesh.py")
    rec = _record(tmp_path, 5, width=64, height=48)
    fake_sequence.n = 5
    seq, frames = tool.open_input(_input_args(tool, rec, "--config", "c.yaml", "--start", "100", "--end", "110",
                                              "--stride", "2"), rec, "cpu")
    assert seq.args == dict(dataset="replica", basedir="d", sequence="room0", config={"from": "c.yaml"}, start=100,
                            end=110, stride=2, desired_height=48, desired_width=64, device="cpu")
    assert len(frames) == 5 and frames[4] == dict(id=4) and not seq.closed
    fake_sequence.n = 12                                 # a --frames cap is the one case a longer sequence is allowed
    seq, frames = tool.open_input(_input_args(tool, rec, "--frames", "5"), rec, "cpu")
    assert len(frames) == 5 and seq.args["config"] is None and (seq.args["start"], seq.args["stride"]) == (0, 1)


@pytest.mark.parametrize("n, extra", [(12, []), (4, []), (4, ["--frames", "5"])])
def test_open_input_rejects_a_selection_of_another_length(tmp_path, fake_sequence, n, extra):
    tool = load("tools/extract_mesh.py")
    rec = _record(tmp_path, 5)
    fake_sequence.n = n
    with pytest.raises(ValueError, match="has 5 cameras but .* select %d frames" % min(n, 5 if extra else n)):
        tool.open_input(_input_args(tool, rec, *extra), rec, "cpu")
    assert fake_sequence.made[-1].closed


def test_record_fusion_rejects_a_source_of_another_length_before_device_work(tmp_path):
    rec = _record(tmp_path, 5)
    for n in (4, 6):
        with pytest.raises(ValueError, match="has 5 cameras but the source has %d frames" % n):
            RecordFusion(rec, device="cuda:0", source=[dict()] * n)


def test_volumes_stay_within_what_marching_cubes_can_count():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    side = int(round(MC_MAX_SAMPLES ** (1 / 3)))
    while side ** 3 > MC_MAX_SAMPLES:
        side -= 1
    assert lib.sb_mc_workspace_bytes(side, side, side, ctypes.byref(n)) == 0
    assert lib.sb_mc_workspace_bytes(side + 1, side + 1, side + 1, ctypes.byref(n)) == 1
    assert lib.sb_mc_workspace_bytes(1000, 1000, 1000, ctypes.byref(n)) == 1      # 5e9 triangles could wrap the scan
    with pytest.raises(ValueError, match="needs 1000000000 voxels .* max_voxels = %d" % MC_MAX_SAMPLES):
        TSDFVolume((0, 0, 0, 999, 999, 999), 1.0, device="cpu", max_voxels=2_000_000_000)
