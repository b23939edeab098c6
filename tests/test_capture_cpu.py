"""CPU: the NeRFCapture reader's host side and the live-capture host logic (splatam_b200/datasets.py, capture.py)
against the reference's own capture code run unmodified (tests/golden/capture/ref_capture.npz, written by
make_golden_capture.py); the uint8 / float32 / uint16 rules of oracle/capture_numpy.py against real cv2 and NumPy;
packet validation; argument checks of sb_ingest_capture and sb_capture_depth_u16; the DDS adapter against a stand-in
cyclonedds module (no socket is opened)."""
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from util import GOLDEN, bits_equal, load
from oracle import capture_numpy as N, ingest_numpy
from splatam_b200 import _lib, capture as C, datasets as D

FIX = os.path.join(GOLDEN, "capture", "ref_capture.npz")


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/capture/make_golden_capture.py")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIX))


def write_tree(fx, prefix, dst):
    for k, v in fx.items():
        if k.startswith(prefix + "/"):
            p = os.path.join(dst, k[len(prefix) + 1:])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(v.tobytes())


@pytest.fixture(scope="module")
def root(fx, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("captures"))
    write_tree(fx, "demo", os.path.join(d, "demo"))
    write_tree(fx, "script", os.path.join(d, "script"))
    return d


def frames_of(gen):
    return [C.sample_to_frame(s) for s in gen.make_packets()]


# ---- the numpy restatement against cv2 and NumPy ---------------------------------------------------------------------

@pytest.mark.parametrize("size", [(720, 960), (360, 480), (480, 640), (900, 1200), (500, 700), (721, 960), (257, 333),
                                  (719, 961), (1440, 1920), (1500, 2000), (1500, 1000)])
def test_uint8_linear_rule_matches_cv2_on_a_phone_frame(size):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(1).integers(0, 256, (1440, 1920, 3), dtype=np.uint8)
    H, W = size
    assert np.array_equal(N.resize_linear_u8(img, H, W), cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR))


@pytest.mark.parametrize("src,dst", [((45, 60), (22, 30)), ((45, 60), (11, 15)), ((23, 37), (11, 18)),
                                     ((23, 37), (27, 50)), ((3, 5), (40, 64)), ((1, 1), (3, 4)), ((7, 2), (20, 1)),
                                     ((1, 9), (5, 4)), ((55, 101), (40, 64)), ((6, 8), (3, 4))])
def test_uint8_linear_rule_matches_cv2_on_odd_sizes(src, dst):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(sum(src + dst)).integers(0, 256, src + (3,), dtype=np.uint8)
    H, W = dst
    assert np.array_equal(N.resize_linear_u8(img, H, W), cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR))


@pytest.mark.parametrize("size", [(720, 960), (360, 480), (1440, 1920), (7, 5)])
def test_float_nearest_and_saved_depth_match_cv2(gen, size):
    cv2 = pytest.importorskip("cv2")
    d = gen.special_depth(np.random.default_rng(3), 192, 256)
    H, W = size
    assert bits_equal(N.resize_nearest(d, H, W), cv2.resize(d, (W, H), interpolation=cv2.INTER_NEAREST))
    with np.errstate(invalid="ignore"):
        q = (d * 65535 / float(10.0)).astype(np.uint16)
    assert bits_equal(N.capture_depth_u16(d, 10.0, H, W), cv2.resize(q, (W, H), interpolation=cv2.INTER_NEAREST))


def test_quantisation_is_numpys_cast():
    d = np.array([10.5, -0.5, np.nan, np.inf, -np.inf, 0.0, 3.3e5, 2.0e5, -3.3e5, 1e9, 6.0, 9.99999], np.float32)
    got = N.quantise_u16(d, 10.0)
    assert got[:3].tolist() == [3275, 62260, 0] and got[3:6].tolist() == [0, 0, 0]
    with np.errstate(invalid="ignore"):
        assert bits_equal(got, (d * 65535 / float(10.0)).astype(np.uint16))
        assert bits_equal(N.quantise_u16(d, 3.0), (d * 65535 / float(3.0)).astype(np.uint16))


def test_full_size_digests_of_the_restatement(gen, fx):
    """The restatement on the seeded 1920x1440 packet hashes to cv2's outputs (stored as digests, not arrays)."""
    rgb, depth = gen.full_size_inputs(np.random.default_rng(int(fx["full_seed"])))
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    for H, W in gen.FULL_SIZES:
        assert sha(N.resize_linear_u8(rgb, H, W)) == str(fx["digest_color_%dx%d" % (H, W)])
        assert sha(N.resize_nearest(depth, H, W)) == str(fx["digest_depth_%dx%d" % (H, W)])
    assert sha(N.capture_depth_u16(depth, 10.0, 1440, 1920)) == str(fx["digest_depth_u16"])


def test_restatement_equals_the_demo_tensors(gen, fx):
    """oracle.ingest_capture on each kept packet equals iphone_demo.py's tracking- and densification-size tensors."""
    kept = [f for f in frames_of(gen) if f.has_depth]
    assert len(kept) == fx["demo_tracking_im"].shape[0] == 6
    for t, f in enumerate(kept):
        for kind, (H, W) in (("tracking", (22, 30)), ("densify", (11, 15))):
            c, d = N.ingest_capture(f.rgb(), f.depth(), H, W)
            assert bits_equal(c, fx["demo_%s_im" % kind][t]), (kind, t)
            assert bits_equal(d, fx["demo_%s_depth" % kind][t]), (kind, t)


def test_saved_depth_and_colour_files_equal_the_restatement(gen, fx, root):
    from PIL import Image
    kept = [f for f in frames_of(gen) if f.has_depth]
    for t, f in enumerate(kept):
        with Image.open(os.path.join(root, "demo", "depth", "%d.png" % t)) as im:
            saved = np.array(im).astype(np.uint16)
        assert bits_equal(saved, N.capture_depth_u16(f.depth(), 10.0, f.height, f.width)), t
        with Image.open(os.path.join(root, "demo", "rgb", "%d.png" % t)) as im:
            assert np.array_equal(np.array(im), f.rgb()), t


# ---- the manifest and the ARKit poses --------------------------------------------------------------------------------

def test_manifest_bytes_equal_the_references(gen, fx):
    import json
    kept = [f for f in frames_of(gen) if f.has_depth]
    m = C.manifest_header(kept[0], 10.0)
    m["frames"] = [C.manifest_entry(t, f) for t, f in enumerate(kept)]
    assert json.dumps(m, indent=4).encode() == fx["demo/transforms.json"].tobytes()


def test_gt_w2c_equals_the_demos(gen, fx):
    kept = [f for f in frames_of(gen) if f.has_depth]
    got = C.arkit_gt_w2c([f.x_wv() for f in kept])
    assert bits_equal(np.stack([g.numpy() for g in got]), fx["demo_gt_w2c"])
    assert bits_equal(np.stack([g.numpy() for g in got]), fx["demo_params_gt_w2c_all_frames"])


# ---- the reader ------------------------------------------------------------------------------------------------------

def test_reader_files_poses_and_intrinsics_equal_the_references(fx, root):
    f = D.SequenceFiles("nerfcapture", root, "demo", desired_height=22, desired_width=30)
    base = os.path.join(root, "demo")
    assert [os.path.relpath(p, base) for p in f.color_paths] == fx["reader_color_names"].tolist()
    assert [os.path.relpath(p, base) for p in f.depth_paths] == fx["reader_depth_names"].tolist()
    assert bits_equal(f.poses.numpy(), fx["reader_poses"])
    assert bits_equal(f.intrinsics.numpy(), fx["reader_intrinsics"])
    assert f.png_depth_scale == 6553.5


def test_reader_pixels_through_the_float64_restatement(fx, root):
    f = D.SequenceFiles("nerfcapture", root, "demo", desired_height=22, desired_width=30)
    for t in range(len(f)):
        c, d = ingest_numpy.ingest(D.decode_color(f.color_paths[t]), D.decode_depth(f.depth_paths[t]), 22, 30, 6553.5)
        assert bits_equal(c, fx["reader_color"][t]) and bits_equal(d, fx["reader_depth"][t]), t


def test_reader_natural_order_and_depth_name_rule(tmp_path, fx):
    import json
    seq = tmp_path / "rgb_scene"
    write_tree(fx, "demo", str(seq))
    for t in range(6, 11):                            # rgb/10.png must sort after rgb/9.png
        for sub in ("rgb", "depth"):
            (seq / sub / ("%d.png" % t)).write_bytes((seq / sub / "0.png").read_bytes())
    m = json.loads((seq / "transforms.json").read_text())
    m["frames"] += [dict(m["frames"][0], file_path="rgb/%d.png" % t) for t in range(6, 11)]
    (seq / "transforms.json").write_text(json.dumps(m))
    f = D.SequenceFiles("nerfcapture", str(tmp_path), "rgb_scene")
    assert [os.path.basename(p) for p in f.color_paths] == ["%d.png" % t for t in range(11)]
    # every 'rgb' in the relative name is replaced, not the directory's own
    assert f.depth_paths[0] == os.path.join(str(seq), "depth/0.png")
    assert (f.height, f.width) == (45, 60)


def test_reader_errors(tmp_path, fx):
    import json
    seq = tmp_path / "cap"
    write_tree(fx, "demo", str(seq))
    (seq / "rgb" / "99.png").write_bytes((seq / "rgb" / "0.png").read_bytes())
    with pytest.raises(ValueError, match="no entry in transforms.json"):
        D.SequenceFiles("nerfcapture", str(tmp_path), "cap")
    os.remove(seq / "rgb" / "99.png")
    m = json.loads((seq / "transforms.json").read_text())
    m["integer_depth_scale"] = 5.0 / 65535.0
    (seq / "transforms.json").write_text(json.dumps(m))
    with pytest.warns(UserWarning, match="integer_depth_scale"):
        f = D.SequenceFiles("nerfcapture", str(tmp_path), "cap")
    assert f.png_depth_scale == 6553.5
    with pytest.raises(ValueError, match="no shipped data config"):
        D.default_config("nerfcapture")


# ---- packets ---------------------------------------------------------------------------------------------------------

def test_packet_validation(gen):
    import dataclasses
    fr = frames_of(gen)
    first = fr[0]
    C.check_packet(first)
    C.check_packet(fr[NO := gen.NO_DEPTH], first)           # no depth: passes, the sequence drops it
    assert not fr[NO].has_depth
    bad = [dataclasses.replace(first, image=first.image[:-1]),
           dataclasses.replace(first, depth_image=first.depth_image + b"\0"),
           dataclasses.replace(first, width=0), dataclasses.replace(first, depth_height=-1),
           dataclasses.replace(first, transform_matrix=first.transform_matrix[:15]),
           dataclasses.replace(first, transform_matrix=(float("nan"),) * 16),
           dataclasses.replace(first, fl_x=0.0), dataclasses.replace(first, cy=float("inf"))]
    for b in bad:
        with pytest.raises(C.CaptureError):
            C.check_packet(b)
    for change in (dict(fl_x=first.fl_x + 1), dict(cx=first.cx + 0.5), dict(depth_width=4, depth_image=b"\0" * 96)):
        with pytest.raises(C.CaptureError, match="first packet"):
            C.check_packet(dataclasses.replace(first, **change), first)


def test_live_capture_drops_packets_without_depth_and_needs_cuda(gen):
    seq = C.LiveCapture(frames_of(gen), 6, 22, 30, 11, 15, device="cpu")
    assert len(seq) == 6
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        seq[0]
    with pytest.raises(ValueError):
        C.LiveCapture([], 0)


def test_kernel_wrappers_have_no_cpu_fallback():
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        C.ingest_capture(torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(2, 2), 2, 2)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        C.capture_depth_u16(torch.zeros(2, 2), 10.0, 4, 4)


def test_capture_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    f = lib.sb_ingest_capture
    assert f(None, 4, 4, 1, 2, 2, 2, 2, 1, 1, None) == 1                     # null pointers
    assert f(1, 4, 4, None, 2, 2, 2, 2, 1, 1, None) == 1
    assert f(1, 4, 4, 1, 2, 2, 2, 2, None, 1, None) == 1
    assert f(1, 4, 4, 1, 2, 2, 2, 2, 1, None, None) == 1
    assert f(1, 0, 4, 1, 2, 2, 2, 2, 1, 1, None) == 1                        # non-positive sizes
    assert f(1, 4, -4, 1, 2, 2, 2, 2, 1, 1, None) == 1
    assert f(1, 4, 4, 1, 0, 2, 2, 2, 1, 1, None) == 1
    assert f(1, 4, 4, 1, 2, 2, 2, 0, 1, 1, None) == 1
    assert f(1, 1 << 16, 1 << 16, 1, 2, 2, 2, 2, 1, 1, None) == 1            # 2^32 * 3 colour bytes overflow int
    assert f(1, 4, 4, 1, 2, 2, 1 << 16, 1 << 16, 1, 1, None) == 1            # output size overflows int
    g = lib.sb_capture_depth_u16
    assert g(None, 2, 2, 10.0, 4, 4, 1, None) == 1
    assert g(1, 2, 2, 10.0, 4, 4, None, None) == 1
    assert g(1, 0, 2, 10.0, 4, 4, 1, None) == 1
    assert g(1, 2, 2, 10.0, 4, -1, 1, None) == 1
    assert g(1, 2, 2, 0.0, 4, 4, 1, None) == 1                               # depth scale: finite and positive
    assert g(1, 2, 2, float("nan"), 4, 4, 1, None) == 1
    assert g(1, 2, 2, float("inf"), 4, 4, 1, None) == 1
    assert g(1, 1 << 16, 1 << 16, 10.0, 4, 4, 1, None) == 1


# ---- the DDS adapter -------------------------------------------------------------------------------------------------

def test_dds_adapter_against_a_stand_in(gen, monkeypatch):
    """dds_frames subscribes to topic "Frames" on the given domain with reliable QoS and maps each sample; the stand-in
    serves the golden packets with an empty read between them."""
    log = {}
    samples = gen.make_packets()
    queue = []
    for s in samples:
        queue += [None, s]
    names = ["cyclonedds", "cyclonedds.idl", "cyclonedds.idl.annotations", "cyclonedds.idl.types",
             "cyclonedds.domain", "cyclonedds.core", "cyclonedds.sub", "cyclonedds.topic", "cyclonedds.util"]
    mods = {n: types.ModuleType(n) for n in names}

    class IdlStruct:
        def __init_subclass__(cls, typename=None, **kw):
            log["typename"] = typename

    class Generic:
        def __class_getitem__(cls, item):
            return list
    mods["cyclonedds.idl"].IdlStruct = IdlStruct
    a = mods["cyclonedds.idl.annotations"]
    a.final, a.autoid, a.key = (lambda c: c), (lambda *x: (lambda c: c)), (lambda *x: None)
    t = mods["cyclonedds.idl.types"]
    t.uint8 = t.uint32 = int
    t.float32 = t.float64 = float
    t.array = t.sequence = Generic
    mods["cyclonedds.domain"].DomainParticipant = lambda d=0: log.setdefault("domain", d)
    mods["cyclonedds.util"].duration = lambda seconds: ("duration", seconds)
    mods["cyclonedds.core"].Policy = types.SimpleNamespace(
        Reliability=types.SimpleNamespace(Reliable=lambda max_blocking_time: ("reliable", max_blocking_time)))
    mods["cyclonedds.core"].Qos = lambda *p: ("qos",) + p

    def topic(participant, name, cls, qos=None):
        log.update(topic=name, cls=cls, qos=qos)
        return "topic"
    mods["cyclonedds.topic"].Topic = topic

    class Reader:
        def __init__(self, participant, tp):
            log["reader"] = tp

        def read_next(self):
            return queue.pop(0) if queue else None
    mods["cyclonedds.sub"].DataReader = Reader
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    monkeypatch.setattr(C.time, "sleep", lambda s: None)
    it = C.dds_frames(domain_id=3)
    got = [next(it) for _ in samples]
    assert log["domain"] == 3 and log["topic"] == "Frames" and log["reader"] == "topic"
    assert log["typename"] == "SplatCaptureData.SplatCaptureFrame"
    assert log["qos"] == ("qos", ("reliable", ("duration", 1)))
    assert [f for f, _ in C.DDS_FIELDS] == list(log["cls"].__annotations__)
    for s, f in zip(samples, got):
        assert isinstance(f, C.CaptureFrame)
        assert f.id == s.id and f.has_depth == s.has_depth and f.image == bytes(s.image)
        assert f.depth_image == bytes(s.depth_image) and f.transform_matrix == tuple(s.transform_matrix)
        assert (f.fl_x, f.fl_y, f.cx, f.cy, f.width, f.height) == (s.fl_x, s.fl_y, s.cx, s.cy, s.width, s.height)
    assert "cyclonedds" in sys.modules and queue == []
