"""GPU: the capture-ingest kernels (csrc/ingest.cu: sb_ingest_capture, sb_capture_depth_u16), LiveCapture and
CaptureWriter (splatam_b200/capture.py) and the NeRFCapture reader (datasets.py) against the reference's own capture
code (tests/golden/capture/ref_capture.npz) and cv2's digests on a full-size packet, bit for bit; and a short synthetic
online run whose capture the reader re-reads and whose params.npz formats and the viewer open."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

from util import GOLDEN, ROOT, bits_equal, load
from oracle import capture_numpy as N
from splatam_b200 import capture as C, datasets as D

pytestmark = pytest.mark.gpu

FIX = os.path.join(GOLDEN, "capture", "ref_capture.npz")


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/capture/make_golden_capture.py")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIX))


def test_full_size_packet_matches_cv2_digests(gen, fx, cuda_device):
    rgb, depth = gen.full_size_inputs(np.random.default_rng(int(fx["full_seed"])))
    assert np.isnan(depth).any() and np.isinf(depth).any() and (depth < 0).any() and (depth > 10).any()
    dr, dd = torch.from_numpy(rgb).to(cuda_device), torch.from_numpy(depth).to(cuda_device)
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    for H, W in gen.FULL_SIZES:
        c, d = C.ingest_capture(dr, dd, H, W)
        ref_c, ref_d = N.ingest_capture(rgb, depth, H, W)
        assert bits_equal(c.cpu().numpy(), ref_c) and bits_equal(d.cpu().numpy(), ref_d), (H, W)
        u8 = (c.cpu().numpy() * np.float32(255)).round().astype(np.uint8).transpose(1, 2, 0)
        assert sha(u8) == str(fx["digest_color_%dx%d" % (H, W)])
        assert sha(d[0].cpu().numpy()) == str(fx["digest_depth_%dx%d" % (H, W)])
    q = C.capture_depth_u16(dd, 10.0, 1440, 1920)
    assert sha(q.cpu().numpy()) == str(fx["digest_depth_u16"])


def test_kernels_match_the_restatement_on_random_sizes(gen, cuda_device):
    g = np.random.default_rng(9)
    cases = [((45, 60), (6, 8), 22, 30), ((45, 60), (6, 8), 11, 15), ((23, 37), (5, 3), 27, 50),
             ((3, 5), (3, 3), 40, 64), ((64, 48), (9, 7), 64, 48), ((100, 80), (3, 3), 50, 40), ((1, 1), (2, 4), 3, 4)]
    for (h, w), (hd, wd), H, W in cases:
        rgb = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        depth = gen.special_depth(g, hd, wd)
        c, d = C.ingest_capture(torch.from_numpy(rgb).to(cuda_device), torch.from_numpy(depth).to(cuda_device), H, W)
        ref_c, ref_d = N.ingest_capture(rgb, depth, H, W)
        assert bits_equal(c.cpu().numpy(), ref_c) and bits_equal(d.cpu().numpy(), ref_d), ((h, w), (H, W))
        for scale in (10.0, 3.0):
            q = C.capture_depth_u16(torch.from_numpy(depth).to(cuda_device), scale, H, W)
            assert bits_equal(q.cpu().numpy(), N.capture_depth_u16(depth, scale, H, W)), ((hd, wd), (H, W), scale)


def test_live_capture_equals_the_demos_tensors_and_files(gen, fx, tmp_path, cuda_device):
    packets = [C.sample_to_frame(s) for s in gen.make_packets()]
    out = str(tmp_path / "demo")
    w = C.CaptureWriter(out, 10.0)
    with C.LiveCapture(packets, 6, 22, 30, 11, 15, 2.0, 4.0, device=cuda_device, writer=w) as seq:
        frames = [seq[t] for t in range(len(seq))]
        assert seq.dropped == 1
        for t, fr in enumerate(frames):
            assert fr["id"] == t
            assert bits_equal(fr["im"].cpu().numpy(), fx["demo_tracking_im"][t]), t
            assert bits_equal(fr["depth"].cpu().numpy(), fx["demo_tracking_depth"][t]), t
            assert bits_equal(fr["gt_w2c"].cpu().numpy(), fx["demo_gt_w2c"][t]), t
        last = frames[-1]["densify"]                   # only the newest frame keeps its densification copy
        assert bits_equal(last["im"].cpu().numpy(), fx["demo_densify_im"][5])
        assert bits_equal(last["depth"].cpu().numpy(), fx["demo_densify_depth"][5])
        assert bits_equal(seq.intrinsics.cpu().numpy(), fx["demo_intrinsics"])
        assert bits_equal(seq.densify_intrinsics.cpu().numpy(), fx["demo_densify_intrinsics"])
        assert bits_equal(seq.intrinsics.cpu().numpy(), fx["demo_params_intrinsics"])
        assert torch.equal(seq.w2c.cpu(), torch.from_numpy(fx["demo_params_w2c"]))
    # every frame's densification copy, from a sequence read frame by frame
    with C.LiveCapture(packets, 6, 22, 30, 11, 15, 2.0, 4.0, device=cuda_device) as seq:
        for t in range(6):
            dn = seq[t]["densify"]
            assert bits_equal(dn["im"].cpu().numpy(), fx["demo_densify_im"][t]), t
            assert bits_equal(dn["depth"].cpu().numpy(), fx["demo_densify_depth"][t]), t
    from PIL import Image
    assert open(os.path.join(out, "transforms.json"), "rb").read() == fx["demo/transforms.json"].tobytes()
    for t in range(6):
        for sub in ("rgb", "depth"):
            name = "%s/%d.png" % (sub, t)
            with Image.open(os.path.join(out, name)) as a:
                got = np.array(a)
            import io
            with Image.open(io.BytesIO(fx["demo/" + name].tobytes())) as b:
                ref = np.array(b)
            assert np.array_equal(got, ref) and got.dtype.itemsize == ref.dtype.itemsize, name


def test_reader_frames_equal_the_references(fx, tmp_path, cuda_device):
    for k, v in fx.items():
        if k.startswith("demo/"):
            p = tmp_path / "demo" / k[len("demo/"):]
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(v.tobytes())
    for prefetch in (0, 2):
        with D.RGBDSequence("nerfcapture", str(tmp_path), "demo", desired_height=22, desired_width=30,
                            device=cuda_device, prefetch=prefetch) as seq:
            assert len(seq) == fx["reader_color"].shape[0]
            for t in range(len(seq)):
                fr = seq[t]
                assert bits_equal(fr["im"].cpu().numpy(), fx["reader_color"][t]), t
                assert bits_equal(fr["depth"].cpu().numpy(), fx["reader_depth"][t]), t
            assert bits_equal(seq.files.poses.numpy(), fx["reader_poses"])


def test_synthetic_online_run_writes_a_capture_the_reader_and_viewer_open(tmp_path, cuda_device):
    """The online demo on 6 rendered phone-size packets (short iterations): the capture it writes is read back by the
    NeRFCapture reader, the saved depth equals the packets' through the restatement, and params.npz opens."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import run_iphone_demo
    from splatam_b200 import formats, viewer
    out = str(tmp_path / "run")
    packets = list(C.synthetic_frames(6, cuda_device))
    res = run_iphone_demo.run(iter(packets), 6, out, device=cuda_device, tracking_iters=15, mapping_iters=10)
    assert np.isfinite(res["ate_m"]) and res["gaussians"] > 0 and res["dropped_packets"] == 0
    with D.RGBDSequence("nerfcapture", str(tmp_path), "run", desired_height=720, desired_width=960,
                        device=cuda_device, prefetch=0) as seq:
        assert len(seq) == 6
        fr = seq[3]
        assert fr["im"].shape == (3, 720, 960) and float(fr["depth"].max()) > 0
    from PIL import Image
    with Image.open(os.path.join(out, "depth", "3.png")) as im:
        saved = np.array(im).astype(np.uint16)
    assert bits_equal(saved, N.capture_depth_u16(packets[3].depth(), 10.0, 1440, 1920))
    rec = np.load(os.path.join(out, "params.npz"))
    assert set(rec.files) == set(formats.RECORD_KEYS)
    assert int(rec["org_width"]) == 960 and int(rec["org_height"]) == 720 and rec["gt_w2c_all_frames"].shape == (6, 4, 4)
    assert viewer.load_record(os.path.join(out, "params.npz"), cuda_device) is not None
    m = json.load(open(os.path.join(out, "transforms.json")))
    assert [f["file_path"] for f in m["frames"]] == ["rgb/%d.png" % t for t in range(6)]
