"""Live RGB-D frames from the NeRFCapture iOS app, as the reference's online demo consumes them
(R/scripts/iphone_demo.py) and its capture script records them (R/scripts/nerfcapture2dataset.py).

* `CaptureFrame`: one packet, with the fields of the app's DDS message (SplatCaptureData.SplatCaptureFrame).
  `check_packet` validates it, since it is input from outside the program.
* `LiveCapture`: a sequence of frame dicts, the shape `datasets.RGBDSequence` gives, over a stream of packets:
  `seq[t]` blocks until packet t has arrived, uploads it from a pinned staging slot on a side stream and turns it into
  the tracking-size and densification-size frames with two `sb_ingest_capture` launches (csrc/ingest.cu), exactly as
  the demo's four cv2.resize calls, `float() / 255` and `permute` compute them.  `slam.run_slam` consumes it unchanged.
* `CaptureWriter`: the capture directory the reference writes (rgb/N.png, depth/N.png from `sb_capture_depth_u16`,
  transforms.json), which `datasets.RGBDSequence("nerfcapture", ...)` reads back.  PNG encoding runs on
  `evaluate.HostWriter` threads.
* `synthetic_frames`: packets of the phone's shape rendered from a generating scene, for tests and runs without a
  phone; `dds_frames`: the packets of a live DDS topic (needs the cyclonedds package, imported only when called).

The reference keeps the first packet's camera for the whole run, so every packet must have the first one's sizes and
intrinsics; a packet without depth is dropped (and counted), as the demo skips it.  CUDA only: there is no CPU
fallback."""
import dataclasses
import json
import os
import time

import numpy as np
import torch

from . import _lib
from .datasets import _OPENGL_TO_OPENCV, NERFCAPTURE_DEPTH_SCALE, relative_poses, setup_camera


class CaptureError(ValueError):
    pass


@dataclasses.dataclass
class CaptureFrame:
    """One packet of the NeRFCapture app, field for field its DDS message: colour `image` is uint8 RGB [height, width,
    3] as bytes, `depth_image` float32 metres [depth_height, depth_width] as bytes, `transform_matrix` the 16 float32
    values of the ARKit camera-to-world matrix in column-major order (OpenGL camera axes).  `depth_scale` is carried
    and unused, as in the reference: the saved depth uses the writer's scale."""
    id: int
    timestamp: float
    fl_x: float
    fl_y: float
    cx: float
    cy: float
    transform_matrix: tuple
    width: int
    height: int
    image: bytes
    has_depth: bool
    depth_width: int
    depth_height: int
    depth_scale: float
    depth_image: bytes

    def camera(self):
        """What must stay equal to the first packet's: sizes and intrinsics."""
        return (self.width, self.height, self.depth_width, self.depth_height, self.fl_x, self.fl_y, self.cx, self.cy)

    def rgb(self):
        return np.frombuffer(self.image, dtype=np.uint8).reshape(self.height, self.width, 3)

    def depth(self):
        return np.frombuffer(self.depth_image, dtype=np.float32).reshape(self.depth_height, self.depth_width)

    def x_wv(self):
        """The ARKit camera-to-world matrix X_WV = transform_matrix.reshape(4, 4).T, float32."""
        return np.asarray(self.transform_matrix, dtype=np.float32).reshape(4, 4).T


def check_packet(fr, first=None):
    """Raises CaptureError unless `fr` is a well-formed packet whose camera equals the first packet's (`first`, a
    CaptureFrame or None).  A packet without depth passes: the caller drops it."""
    for name in ("width", "height"):
        v = getattr(fr, name)
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise CaptureError("packet %s: %s must be a positive integer, got %r" % (fr.id, name, v))
    if len(fr.image) != fr.width * fr.height * 3:
        raise CaptureError("packet %s: image has %d bytes, %dx%d RGB needs %d"
                           % (fr.id, len(fr.image), fr.width, fr.height, fr.width * fr.height * 3))
    if len(fr.transform_matrix) != 16 or not np.isfinite(np.asarray(fr.transform_matrix, np.float64)).all():
        raise CaptureError("packet %s: transform_matrix must be 16 finite values" % fr.id)
    if not all(np.isfinite(float(getattr(fr, k))) for k in ("fl_x", "fl_y", "cx", "cy")) or fr.fl_x <= 0 or fr.fl_y <= 0:
        raise CaptureError("packet %s: the intrinsics must be finite with positive focal lengths" % fr.id)
    if fr.has_depth:
        for name in ("depth_width", "depth_height"):
            v = getattr(fr, name)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
                raise CaptureError("packet %s: %s must be a positive integer, got %r" % (fr.id, name, v))
        if len(fr.depth_image) != fr.depth_width * fr.depth_height * 4:
            raise CaptureError("packet %s: depth_image has %d bytes, %dx%d float32 needs %d"
                               % (fr.id, len(fr.depth_image), fr.depth_width, fr.depth_height,
                                  fr.depth_width * fr.depth_height * 4))
    if first is not None and fr.has_depth and fr.camera() != first.camera():
        raise CaptureError("packet %s: camera %r differs from the first packet's %r; the run keeps the first "
                           "packet's camera" % (fr.id, fr.camera(), first.camera()))


# ---- the two capture kernels -----------------------------------------------------------------------------------------

def ingest_capture(rgb, depth, height, width, color_out=None, depth_out=None):
    """One `sb_ingest_capture` launch on the current stream: rgb uint8 [h, w, 3] and depth float32 [hd, wd] CUDA
    tensors -> (colour float32 [3, height, width] = cv2.resize(rgb, INTER_LINEAR) / 255, depth float32
    [1, height, width] = cv2.resize(depth, INTER_NEAREST)), bit for bit (oracle/capture_numpy.py: ingest_capture)."""
    _lib.need_cuda("ingest_capture", rgb, depth)
    if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3 or not rgb.is_contiguous():
        raise _lib.SplatamB200Error("ingest_capture expects contiguous uint8 [h, w, 3] colour, got %s %s"
                                    % (rgb.dtype, tuple(rgb.shape)))
    if depth.dtype != torch.float32 or depth.dim() != 2 or not depth.is_contiguous():
        raise _lib.SplatamB200Error("ingest_capture expects contiguous float32 [h, w] depth, got %s %s"
                                    % (depth.dtype, tuple(depth.shape)))
    dev = rgb.device
    if color_out is None:
        color_out = torch.empty(3, height, width, dtype=torch.float32, device=dev)
    if depth_out is None:
        depth_out = torch.empty(1, height, width, dtype=torch.float32, device=dev)
    _lib.call("sb_ingest_capture", rgb, rgb.shape[0], rgb.shape[1], depth, depth.shape[0], depth.shape[1], height,
              width, color_out, depth_out, device=dev)
    return color_out, depth_out


def capture_depth_u16(depth, depth_scale, height, width, out=None):
    """One `sb_capture_depth_u16` launch: float32 depth [hd, wd] (CUDA) -> the uint16 [height, width] image the
    capture writers save, cv2.resize((depth * 65535 / depth_scale).astype(uint16), INTER_NEAREST) bit for bit."""
    _lib.need_cuda("capture_depth_u16", depth)
    if depth.dtype != torch.float32 or depth.dim() != 2 or not depth.is_contiguous():
        raise _lib.SplatamB200Error("capture_depth_u16 expects contiguous float32 [h, w] depth, got %s %s"
                                    % (depth.dtype, tuple(depth.shape)))
    if out is None:
        out = torch.empty(height, width, dtype=torch.uint16, device=depth.device)
    _lib.call("sb_capture_depth_u16", depth, depth.shape[0], depth.shape[1], float(depth_scale), height, width, out,
              device=depth.device)
    return out


# ---- the capture directory -------------------------------------------------------------------------------------------

def manifest_header(fr, depth_scale):
    """transforms.json's top level from the first packet, in the reference's key order (`frames` is filled later)."""
    return {"fl_x": fr.fl_x, "fl_y": fr.fl_y, "cx": fr.cx, "cy": fr.cy, "w": fr.width, "h": fr.height, "frames": [],
            "integer_depth_scale": float(depth_scale) / 65535.0}


def manifest_entry(t, fr):
    """transforms.json's entry of frame t (packet `fr`), in the reference's key order."""
    return {"transform_matrix": fr.x_wv().tolist(), "file_path": "rgb/%d.png" % t, "fl_x": fr.fl_x, "fl_y": fr.fl_y,
            "cx": fr.cx, "cy": fr.cy, "w": fr.width, "h": fr.height, "depth_path": "depth/%d.png" % t}


class CaptureWriter:
    """Writes a capture as nerfcapture2dataset.py / iphone_demo.py do: rgb/N.png (the packet's pixels), depth/N.png
    (the uint16 image of `capture_depth_u16` at the colour's size) and, at `close`, transforms.json with the
    reference's keys in its order, as json.dumps(manifest, indent=4) text.  N counts the frames kept.  The PNGs are
    encoded on HostWriter threads; `close` waits for them and re-raises a writer error."""

    def __init__(self, out_dir, depth_scale=NERFCAPTURE_DEPTH_SCALE, threads=None):
        self.out_dir, self.depth_scale = out_dir, float(depth_scale)
        if os.path.exists(os.path.join(out_dir, "rgb")):
            raise FileExistsError("%s already holds a capture (rgb/)" % out_dir)
        self.manifest = None
        self.threads = threads
        self._color = self._depth = None
        self.closed = False

    def add(self, t, fr, rgb, depth):
        """Frame t from packet `fr`, whose pixels are uploaded as rgb uint8 [h, w, 3] and depth float32 [hd, wd] on
        the device; the writes are enqueued on the current stream."""
        from PIL import Image
        from .evaluate import HostWriter
        if self.manifest is None:
            os.makedirs(os.path.join(self.out_dir, "rgb"))
            os.makedirs(os.path.join(self.out_dir, "depth"), exist_ok=True)
            self.manifest = manifest_header(fr, self.depth_scale)
            self._color = HostWriter((fr.height, fr.width, 3), rgb.device, self.threads, name="capture-rgb")
            self._depth = HostWriter((fr.height, fr.width * 2), rgb.device, self.threads, name="capture-depth")
        rgb_path = os.path.join(self.out_dir, "rgb", "%d.png" % t)
        depth_path = os.path.join(self.out_dir, "depth", "%d.png" % t)
        self._color.put(lambda st: st.copy_(rgb), lambda px: Image.fromarray(px).save(rgb_path))
        self._depth.put(lambda st: capture_depth_u16(depth, self.depth_scale, fr.height, fr.width,
                                                     out=st.view(torch.uint16)),
                        lambda px: Image.fromarray(px.view(np.uint16)).save(depth_path))
        self.manifest["frames"].append(manifest_entry(t, fr))

    def manifest_text(self):
        return json.dumps(self.manifest, indent=4)

    def close(self):
        """Waits for every PNG and writes transforms.json (once frames were added)."""
        if self.closed:
            return
        self.closed = True
        for w in (self._color, self._depth):
            if w is not None:
                w.close()
        if self.manifest is not None:
            with open(os.path.join(self.out_dir, "transforms.json"), "w") as f:
                f.write(self.manifest_text())


# ---- live frames -----------------------------------------------------------------------------------------------------

def arkit_gt_w2c(x_wv_list):
    """gt_w2c of each frame as iphone_demo.py computes it on the host: inv(relative(P @ X_WV @ P^T)), float32, with
    the pose relative to the first frame's."""
    P = torch.tensor(_OPENGL_TO_OPENCV).float()
    poses = [P @ torch.from_numpy(np.ascontiguousarray(x)).float() @ P.T for x in x_wv_list]
    return [torch.linalg.inv(relative_poses(torch.stack([poses[0], p]))[1]) for p in poses]


class _PinnedSlot:
    def __init__(self):
        self.rgb = self.depth = None
        self.copied = None

    def arrays(self, rgb_shape, depth_shape):
        if self.copied is not None:
            self.copied.synchronize()                 # refilled only once its previous upload has completed
        if self.rgb is None or tuple(self.rgb.shape) != rgb_shape:
            self.rgb = torch.empty(rgb_shape, dtype=torch.uint8, pin_memory=True)
        if self.depth is None or tuple(self.depth.shape) != depth_shape:
            self.depth = torch.empty(depth_shape, dtype=torch.float32, pin_memory=True)
        return self.rgb, self.depth


class LiveCapture:
    """`num_frames` frames from an iterable of CaptureFrame packets, as a sequence: ``len(seq)`` and ``seq[t]``.

    ``seq[t]`` reads packets until frame t has arrived (frames are the packets with depth, in arrival order) and returns
    dict(id=t, cam, w2c, im [3,H,W], depth [1,H,W], intrinsics [3,3], gt_w2c [4,4], densify=dict(id, cam, w2c, im,
    depth, intrinsics)) on `device`, what iphone_demo.py builds: `intrinsics` = K / downscale_factor with [2,2] = 1
    (K of the first packet), the densification intrinsics likewise with densify_downscale_factor, `w2c` the identity,
    `cam` / `densify` cam at the two sizes, `gt_w2c` = `arkit_gt_w2c`.  A live stream cannot be read twice, so every
    frame is kept (the densification copy only until the next frame arrives); `gt_w2c` lists every frame's so far.

    Each packet is copied into one of `slots` pinned staging pairs, uploaded on a side stream and converted there by
    two `sb_ingest_capture` launches; the caller's stream waits on the result.  `writer` (a CaptureWriter) also saves
    every frame; it is closed after the last one.  `dropped` counts packets without depth, `load_wait_s` the host time
    spent in seq[t] for new frames."""

    def __init__(self, packets, num_frames, height=720, width=960, densify_height=360, densify_width=480,
                 downscale_factor=2.0, densify_downscale_factor=4.0, device="cuda", writer=None, slots=2):
        if num_frames < 1:
            raise ValueError("num_frames must be positive, got %r" % (num_frames,))
        self.packets = iter(packets)
        self.num_frames = int(num_frames)
        self.height, self.width = int(height), int(width)
        self.densify_height, self.densify_width = int(densify_height), int(densify_width)
        self.downscale_factor, self.densify_downscale_factor = float(downscale_factor), float(densify_downscale_factor)
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.writer = writer
        self.first = None
        self.frames, self.x_wv, self.gt_w2c = [], [], []
        self.dropped = 0
        self.load_wait_s = 0.0
        self._slots = [_PinnedSlot() for _ in range(max(int(slots), 1))]
        self._side = None
        self.intrinsics = self.cam = self.densify_intrinsics = self.densify_cam = None
        self.w2c = torch.eye(4, device=self.device)

    def __len__(self):
        return self.num_frames

    def _next_packet(self):
        for fr in self.packets:
            check_packet(fr, self.first)
            if not fr.has_depth:
                self.dropped += 1
                continue
            return fr
        raise CaptureError("the packet stream ended after %d of %d frames" % (len(self.frames), self.num_frames))

    def _setup(self, fr):
        """The cameras of the first packet (iphone_demo.py:227-248)."""
        self.first = fr
        K = torch.tensor([[fr.fl_x, 0, fr.cx], [0, fr.fl_y, fr.cy], [0, 0, 1]]).float()
        Ki = K / self.downscale_factor
        Ki[2, 2] = 1.0
        Kd = K / self.densify_downscale_factor
        Kd[2, 2] = 1.0
        eye = np.eye(4, dtype=np.float32)
        self.intrinsics, self.densify_intrinsics = Ki.to(self.device), Kd.to(self.device)
        self.cam = setup_camera(self.width, self.height, Ki.numpy(), eye, self.device)
        self.densify_cam = setup_camera(self.densify_width, self.densify_height, Kd.numpy(), eye, self.device)
        self._side = torch.cuda.Stream(self.device)

    def _ingest(self, fr, t):
        if self.device.type != "cuda":
            raise _lib.SplatamB200Error("LiveCapture needs a CUDA device (there is no CPU fallback)")
        if self.first is None:
            self._setup(fr)
        slot = self._slots[t % len(self._slots)]
        pr, pd = slot.arrays((fr.height, fr.width, 3), (fr.depth_height, fr.depth_width))
        pr.numpy()[...] = fr.rgb()
        pd.numpy()[...] = fr.depth()
        consumer = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device), torch.cuda.stream(self._side):
            dr = pr.to(self.device, non_blocking=True)
            dd = pd.to(self.device, non_blocking=True)
            slot.copied = torch.cuda.Event()
            slot.copied.record(self._side)
            color, depth = ingest_capture(dr, dd, self.height, self.width)
            dcolor, ddepth = ingest_capture(dr, dd, self.densify_height, self.densify_width)
            if self.writer is not None:
                self.writer.add(t, fr, dr, dd)
        consumer.wait_stream(self._side)
        for x in (dr, dd, color, depth, dcolor, ddepth):
            x.record_stream(consumer)                 # allocated on the side stream, used and freed on the consumer's
        return color, depth, dcolor, ddepth

    def _arrive(self):
        t = len(self.frames)
        fr = self._next_packet()
        color, depth, dcolor, ddepth = self._ingest(fr, t)
        self.x_wv.append(fr.x_wv())
        gt = arkit_gt_w2c([self.x_wv[0], self.x_wv[-1]])[1]
        self.gt_w2c.append(gt.to(self.device))
        if self.frames:
            self.frames[-1].pop("densify", None)
        self.frames.append(dict(id=t, cam=self.cam, w2c=self.w2c, im=color, depth=depth, intrinsics=self.intrinsics,
                                gt_w2c=self.gt_w2c[-1],
                                densify=dict(id=t, cam=self.densify_cam, w2c=self.w2c, im=dcolor, depth=ddepth,
                                             intrinsics=self.densify_intrinsics)))
        if t == self.num_frames - 1 and self.writer is not None:
            self.writer.close()

    def __getitem__(self, t):
        if isinstance(t, slice):
            return [self[i] for i in range(*t.indices(len(self)))]
        t = int(t)
        if t < 0:
            t += len(self)
        if not 0 <= t < len(self):
            raise IndexError("frame %d out of range for a capture of %d" % (t, len(self)))
        t0 = time.perf_counter()
        while len(self.frames) <= t:
            self._arrive()
        if len(self.frames) == t + 1:
            self.load_wait_s += time.perf_counter() - t0
        return self.frames[t]

    def close(self):
        if self.writer is not None:
            self.writer.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


# ---- packet sources --------------------------------------------------------------------------------------------------

PHONE_CAMERA = dict(width=1920, height=1440, depth_width=256, depth_height=192, fl_x=1450.0, fl_y=1450.0, cx=959.5,
                    cy=719.5)


def arkit_transform(w2c):
    """The 16 column-major values of the ARKit camera-to-world matrix of an OpenCV-axes w2c: X_WV = P inv(w2c) P."""
    P = np.array(_OPENGL_TO_OPENCV, dtype=np.float64)
    x_wv = (P @ np.linalg.inv(np.asarray(w2c, np.float64)) @ P).astype(np.float32)
    return tuple(float(v) for v in x_wv.T.reshape(-1))


def synthetic_frames(num_frames, device, seed=14, camera=None, depth_scale=NERFCAPTURE_DEPTH_SCALE):
    """Packets of the phone's shape (1920x1440 colour, 256x192 depth by default; `camera` overrides PHONE_CAMERA's
    keys) rendered on `device` from a view-filling generating scene along `slam.look_trajectory`, with ARKit's pose
    convention.  Depth is 0 where the silhouette is below 0.9, as a sensor reports it.  A generator: each packet is
    rendered when it is asked for."""
    import scenes
    from . import mapping as M, slam
    c = dict(PHONE_CAMERA, **(camera or {}))
    W, H, Wd, Hd = c["width"], c["height"], c["depth_width"], c["depth_height"]
    gen_cam = dict(w=W // 4, h=H // 4, fx=c["fl_x"] / 4, fy=c["fl_y"] / 4, cx=(c["cx"] + 0.5) / 4 - 0.5,
                   cy=(c["cy"] + 0.5) / 4 - 0.5)
    gen = scenes.view_filling(seed=seed, cam=gen_cam, margin=48, opacity=(0.85, 0.95))
    gt = dict(means3D=gen.means3D, rgb_colors=gen.colors, unnorm_rotations=gen.rotations,
              logit_opacities=torch.logit(gen.opacities.clamp(0.02, 0.98)), log_scales=torch.log(gen.scales[:, :1]))
    gt = {k: v.to(device).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(num_frames, device)
    eye = np.eye(4, dtype=np.float32)
    K = np.array([[c["fl_x"], 0, c["cx"]], [0, c["fl_y"], c["cy"]], [0, 0, 1]], dtype=np.float32)
    sx, sy = Wd / W, Hd / H
    Kd = np.array([[c["fl_x"] * sx, 0, (c["cx"] + 0.5) * sx - 0.5], [0, c["fl_y"] * sy, (c["cy"] + 0.5) * sy - 0.5],
                   [0, 0, 1]], dtype=np.float32)
    cam = setup_camera(W, H, K, eye, device)
    dcam = setup_camera(Wd, Hd, Kd, eye, device)
    for t in range(num_frames):
        f = slam.render_frame(gt, rots, trans, t, cam)
        d = slam.render_frame(gt, rots, trans, t, dcam)
        depth = torch.where(d["sil"] > 0.9, d["depth"] / d["sil"].clamp(min=1e-6), torch.zeros_like(d["depth"]))
        rgb = (f["im"].clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).contiguous().cpu().numpy()
        w2c = M.camera_w2c(rots[..., t], trans[..., t])[0].detach().double().cpu().numpy()
        yield CaptureFrame(id=t, timestamp=t / 30.0, fl_x=float(np.float32(c["fl_x"])), fl_y=float(np.float32(c["fl_y"])),
                           cx=float(np.float32(c["cx"])), cy=float(np.float32(c["cy"])),
                           transform_matrix=arkit_transform(w2c), width=W, height=H, image=rgb.tobytes(),
                           has_depth=True, depth_width=Wd, depth_height=Hd, depth_scale=float(depth_scale),
                           depth_image=depth[0].float().contiguous().cpu().numpy().tobytes())


# The DDS message of the NeRFCapture app (topic "Frames", type SplatCaptureData.SplatCaptureFrame), in field order:
# the wire contract the adapter below reads.
DDS_FIELDS = (("id", "uint32"), ("timestamp", "float64"), ("fl_x", "float32"), ("fl_y", "float32"),
              ("cx", "float32"), ("cy", "float32"), ("transform_matrix", "float32[16]"), ("width", "uint32"),
              ("height", "uint32"), ("image", "sequence<uint8>"), ("has_depth", "bool"), ("depth_width", "uint32"),
              ("depth_height", "uint32"), ("depth_scale", "float32"), ("depth_image", "sequence<uint8>"))


def _dds_message_type():
    from dataclasses import dataclass
    import cyclonedds.idl as idl
    import cyclonedds.idl.annotations as annotate
    import cyclonedds.idl.types as types

    @dataclass
    @annotate.final
    @annotate.autoid("sequential")
    class SplatCaptureFrame(idl.IdlStruct, typename="SplatCaptureData.SplatCaptureFrame"):
        id: types.uint32
        annotate.key("id")
        timestamp: types.float64
        fl_x: types.float32
        fl_y: types.float32
        cx: types.float32
        cy: types.float32
        transform_matrix: types.array[types.float32, 16]
        width: types.uint32
        height: types.uint32
        image: types.sequence[types.uint8]
        has_depth: bool
        depth_width: types.uint32
        depth_height: types.uint32
        depth_scale: types.float32
        depth_image: types.sequence[types.uint8]
    return SplatCaptureFrame


def sample_to_frame(s):
    """A CaptureFrame from one DDS sample (any object with the DDS_FIELDS attributes)."""
    return CaptureFrame(
        id=int(s.id), timestamp=float(s.timestamp), fl_x=float(s.fl_x), fl_y=float(s.fl_y), cx=float(s.cx),
        cy=float(s.cy), transform_matrix=tuple(float(v) for v in s.transform_matrix), width=int(s.width),
        height=int(s.height), image=bytes(s.image), has_depth=bool(s.has_depth), depth_width=int(s.depth_width),
        depth_height=int(s.depth_height), depth_scale=float(s.depth_scale), depth_image=bytes(s.depth_image))


def dds_frames(domain_id=0, poll_s=0.001):
    """Packets from the NeRFCapture app over DDS: joins `domain_id`, subscribes to topic "Frames" with reliable QoS
    (1 s maximum blocking time) and yields a CaptureFrame per sample, polling every `poll_s` seconds while none is
    waiting.  Needs the cyclonedds package, which is imported here only."""
    from cyclonedds.core import Policy, Qos
    from cyclonedds.domain import DomainParticipant
    from cyclonedds.sub import DataReader
    from cyclonedds.topic import Topic
    from cyclonedds.util import duration
    participant = DomainParticipant(domain_id)
    qos = Qos(Policy.Reliability.Reliable(max_blocking_time=duration(seconds=1)))
    reader = DataReader(participant, Topic(participant, "Frames", _dds_message_type(), qos=qos))
    while True:
        s = reader.read_next()
        if s:
            yield sample_to_frame(s)
        else:
            time.sleep(poll_s)
