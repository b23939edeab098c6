"""SplaTAM's final evaluation (R/utils/eval_helpers.py:408-623, `eval`) on the GPU: per-frame PSNR, MS-SSIM, depth
errors and the ATE of the estimated trajectory, with the metric kernels of csrc/eval_metrics.cu.

The reference renders every evaluated frame twice, computes PSNR and the depth errors in PyTorch and copies both
weighted images to the host for pytorch_msssim on the CPU.  Here the renders go through the same front end as
mapping and tracking (`mapping._render_pair`), one kernel pass per frame writes the masked images and the PSNR /
depth sums, MS-SSIM runs on the device, and the per-frame metrics stay on the device until one read at the end.
`evaluate_nvs` is the reference's novel-view evaluation (eval_helpers.py:626-841, `eval_nvs`) over a test split: the
same metrics on held-out views rendered at their ground-truth poses, averaged over the views the map covers.
LPIPS (AlexNet, v0.1, csrc/lpips.cu) is opt-in: pass ``lpips=LpipsAlex.load(alexnet_path, lin_path, device)`` with the
two weight files already on disk (nothing is downloaded); without it the result carries ``lpips: None``.
``save_frames=True`` also writes the reference's four PNGs per evaluated frame (rendered and ground-truth colour and
depth, csrc/eval_frames.cu), encoded by writer threads while the evaluation goes on.  CUDA only; no CPU fallback."""
import os
import queue
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib
from . import mapping as M

# columns of the per-frame metric rows: the five that sb_frame_metrics writes, then MS-SSIM and LPIPS
_PSNR, _RMSE, _L1, _NVALID, _NMASK, _SSIM, _LPIPS = range(7)

# cv2.COLORMAP_JET as 256 RGB entries, the table the reference's saved depth images go through:
#   cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_JET)[:, 0, ::-1].tobytes().hex()
# No closed form was found that reproduces it: the usual clip(1.5 - |4x - c|, 0, 1) is one off at some entries, and
# the integer ramps that match the rest give 2 where cv2 has 1 (blue, entry 159).
JET_RGB = np.frombuffer(bytes.fromhex(
    "00008000008400008800008c00009000009400009800009c0000a00000a40000a80000ac0000b00000b40000b80000bc"
    "0000c00000c40000c80000cc0000d00000d40000d80000dc0000e00000e40000e80000ec0000f00000f40000f80000fc"
    "0000ff0004ff0008ff000cff0010ff0014ff0018ff001cff0020ff0024ff0028ff002cff0030ff0034ff0038ff003cff"
    "0040ff0044ff0048ff004cff0050ff0054ff0058ff005cff0060ff0064ff0068ff006cff0070ff0074ff0078ff007cff"
    "0080ff0084ff0088ff008cff0090ff0094ff0098ff009cff00a0ff00a4ff00a8ff00acff00b0ff00b4ff00b8ff00bcff"
    "00c0ff00c4ff00c8ff00ccff00d0ff00d4ff00d8ff00dcff00e0ff00e4ff00e8ff00ecff00f0ff00f4ff00f8ff00fcff"
    "02fffe06fffa0afff60efff212ffee16ffea1affe61effe222ffde26ffda2affd62effd232ffce36ffca3affc63effc2"
    "42ffbe46ffba4affb64effb252ffae56ffaa5affa65effa262ff9e66ff9a6aff966eff9272ff8e76ff8a7aff867eff82"
    "82ff7e86ff7a8aff768eff7292ff6e96ff6a9aff669eff62a2ff5ea6ff5aaaff56aeff52b2ff4eb6ff4abaff46beff42"
    "c2ff3ec6ff3acaff36ceff32d2ff2ed6ff2adaff26deff22e2ff1ee6ff1aeaff16eeff12f2ff0ef6ff0afaff06feff01"
    "fffc00fff800fff400fff000ffec00ffe800ffe400ffe000ffdc00ffd800ffd400ffd000ffcc00ffc800ffc400ffc000"
    "ffbc00ffb800ffb400ffb000ffac00ffa800ffa400ffa000ff9c00ff9800ff9400ff9000ff8c00ff8800ff8400ff8000"
    "ff7c00ff7800ff7400ff7000ff6c00ff6800ff6400ff6000ff5c00ff5800ff5400ff5000ff4c00ff4800ff4400ff4000"
    "ff3c00ff3800ff3400ff3000ff2c00ff2800ff2400ff2000ff1c00ff1800ff1400ff1000ff0c00ff0800ff0400ff0000"
    "fc0000f80000f40000f00000ec0000e80000e40000e00000dc0000d80000d40000d00000cc0000c80000c40000c00000"
    "bc0000b80000b40000b00000ac0000a80000a40000a000009c00009800009400009000008c0000880000840000800000"),
    dtype=np.uint8).reshape(256, 3)

# the reference's frame directories, in the order of sb_eval_frames_u8's four images
FRAME_DIRS = ("rendered_rgb", "rendered_depth", "rgb", "depth")
# threads that encode the saved frames; the evaluation loop waits only when all FRAME_WRITER_THREADS + 2 pinned host
# slots hold frames not yet written.  Saving is bound by PNG encoding on the host, which scales with the threads
# (tools/time_eval_frames.py: 3.3, 6.3, 13.1 and 25.4 frames/s at 1, 2, 4 and 8 threads, 1200x680, one H100 80GB HBM3
# at 700 W with 16 host CPUs)
FRAME_WRITER_THREADS = min(8, os.cpu_count() or 1)
# zlib level of the saved PNGs: the contract is the decoded pixels, not the file bytes, so the fastest level is used
PNG_COMPRESS_LEVEL = 1


def _ms_ssim_into(x, y, data_range, per_channel, mean, ws=None):
    """Enqueues sb_ms_ssim on contiguous float32 [N,C,H,W] CUDA tensors; `per_channel` / `mean`: float64 device
    tensors or None."""
    N, C, H, W = x.shape
    if ws is None:
        ws = torch.empty(_lib.nbytes("sb_ms_ssim_workspace_bytes", N, C, H, W), dtype=torch.uint8, device=x.device)
    _lib.call("sb_ms_ssim", x, y, N, C, H, W, float(data_range), ws, ws.numel(), per_channel, mean, device=x.device)


def ms_ssim(x, y, data_range=1.0, size_average=True):
    """MS-SSIM of two [N,C,H,W] CUDA images as pytorch_msssim.ms_ssim defines it (11-tap sigma-1.5 Gaussian window,
    valid filtering, 5 levels with weights 0.0448, 0.2856, 0.3001, 0.2363, 0.1333), computed in double on the device.
    size_average=True returns the mean (a float64 0-d tensor); otherwise the float64 [N,C] values (pytorch_msssim
    averages those over channels).  The smaller image side must exceed 160."""
    _lib.need_cuda("ms_ssim", x, y)
    if x.dim() != 4 or x.shape != y.shape:
        raise _lib.SplatamB200Error("ms_ssim expects two [N,C,H,W] images of the same shape, got %s and %s"
                                    % (tuple(x.shape), tuple(y.shape)))
    if min(x.shape[-2:]) <= 160:
        raise _lib.SplatamB200Error("ms_ssim needs a smaller image side > 160, got %s" % (tuple(x.shape),))
    x, y = x.detach().float().contiguous(), y.detach().float().contiguous()
    N, C = x.shape[:2]
    if size_average:
        mean = torch.empty((), dtype=torch.float64, device=x.device)
        _ms_ssim_into(x, y, data_range, None, mean)
        return mean
    out = torch.empty(N, C, dtype=torch.float64, device=x.device)
    _ms_ssim_into(x, y, data_range, out, None)
    return out


# (features index, Cin, Cout, kernel) of torchvision's five AlexNet convolutions, in sb_lpips' packing order
_ALEX_CONVS = ((0, 3, 64, 11), (3, 64, 192, 5), (6, 192, 384, 3), (8, 384, 256, 3), (10, 256, 256, 3))


class LpipsAlex:
    """The weights of LPIPS v0.1 with the AlexNet backbone (torchmetrics' net_type='alex'), packed on one device in
    the layout sb_lpips reads (include/splatam_b200.h): `weights`, a float32 device tensor."""

    def __init__(self, weights):
        self.weights = weights

    @classmethod
    def load(cls, alexnet_path, lin_path, device):
        """Reads torchvision's ImageNet AlexNet state dict (alexnet-owt-7be5be79.pth; features.{0,3,6,8,10}.{weight,
        bias}, classifier keys ignored) and LPIPS v0.1's alex.pth (lin{0..4}.model.1.weight, [1,C,1,1]) with
        torch.load(weights_only=True).  Nothing is downloaded; a missing key or a wrong shape raises
        SplatamB200Error naming the key."""
        load = lambda p: torch.load(p, map_location="cpu", weights_only=True)
        return cls.from_state_dicts(load(alexnet_path), load(lin_path), device)

    @classmethod
    def from_state_dicts(cls, alexnet, lin, device):
        """As `load`, from the two state dicts already in memory."""
        def get(sd, key, shape):
            if key not in sd:
                raise _lib.SplatamB200Error("LPIPS weights: missing key %r" % key)
            t = sd[key]
            if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape:
                raise _lib.SplatamB200Error("LPIPS weights: %r has shape %s, expected %s"
                                            % (key, tuple(getattr(t, "shape", ())), shape))
            return t.detach().to("cpu", torch.float32)
        parts = []
        for idx, cin, cout, k in _ALEX_CONVS:
            w = get(alexnet, "features.%d.weight" % idx, (cout, cin, k, k))
            parts += [w.reshape(cout, -1).t().reshape(-1), get(alexnet, "features.%d.bias" % idx, (cout,))]
        for l, (_, _, cout, _) in enumerate(_ALEX_CONVS):
            parts.append(get(lin, "lin%d.model.1.weight" % l, (1, cout, 1, 1)).reshape(-1))
        packed = torch.cat(parts)
        n = _lib.nbytes("sb_lpips_weights_floats")
        if packed.numel() != n:
            raise _lib.SplatamB200Error("LPIPS weights: packed %d floats, sb_lpips reads %d" % (packed.numel(), n))
        return cls(packed.to(device))


def _lpips_into(x, y, net, per_image, mean, ws=None):
    """Enqueues sb_lpips on contiguous float32 [N,3,H,W] CUDA tensors; `per_image` / `mean`: float64 device tensors or
    None."""
    N, _, H, W = x.shape
    if ws is None:
        ws = torch.empty(_lib.nbytes("sb_lpips_workspace_bytes", N, H, W), dtype=torch.uint8, device=x.device)
    _lib.call("sb_lpips", x, y, N, H, W, net.weights, ws, ws.numel(), per_image, mean, device=x.device)


def _check_lpips_net(net, device):
    if not isinstance(net, LpipsAlex):
        raise _lib.SplatamB200Error("lpips expects an evaluate.LpipsAlex, got %s" % type(net).__name__)
    if net.weights.device != device:
        raise _lib.SplatamB200Error("LPIPS weights are on %s, the images on %s" % (net.weights.device, device))


def lpips(x, y, net, size_average=True):
    """LPIPS (AlexNet, v0.1) of two [N,3,H,W] CUDA images as torchmetrics' LearnedPerceptualImagePatchSimilarity(
    net_type='alex', normalize=True) defines it, on clamp(x, 0, 1) and clamp(y, 0, 1); `net`: an LpipsAlex on the
    images' device.  FP32 convolutions, deterministic.  size_average=True returns the mean (a float64 0-d tensor);
    otherwise the float64 [N] values.  H and W must be >= 31."""
    _lib.need_cuda("lpips", x, y)
    if x.dim() != 4 or x.shape[1] != 3 or x.shape != y.shape:
        raise _lib.SplatamB200Error("lpips expects two [N,3,H,W] images of the same shape, got %s and %s"
                                    % (tuple(x.shape), tuple(y.shape)))
    if min(x.shape[-2:]) < 31:
        raise _lib.SplatamB200Error("lpips needs H and W >= 31, got %s" % (tuple(x.shape),))
    _check_lpips_net(net, x.device)
    x, y = x.detach().float().contiguous(), y.detach().float().contiguous()
    if size_average:
        mean = torch.empty((), dtype=torch.float64, device=x.device)
        _lpips_into(x, y, net, None, mean)
        return mean
    out = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
    _lpips_into(x, y, net, out, None)
    return out


def jet_lut(device):
    """JET_RGB as a contiguous uint8 [256, 3] tensor on `device`, the colormap sb_eval_frames_u8 reads."""
    return torch.from_numpy(JET_RGB.copy()).to(device)


def eval_frames_u8(im, depth_sil, gt_im, gt_depth, lut=None, out=None):
    """The four images the reference saves for an evaluated frame (eval_helpers.py:509-528), as uint8 HWC RGB in one
    [4, H, W, 3] CUDA tensor: the rendered colour `im` [3,H,W] and ground-truth colour `gt_im` [3,H,W] as
    round_half_even(clamp(x, 0, 1) * 255) (NaN -> 0), the rendered depth (channel 0 of `depth_sil` [3,H,W], unmasked)
    and `gt_depth` [1,H,W] through `lut` (default: JET_RGB) at trunc(clip(d / 6, 0, 1) * 255) (NaN -> 0), all in
    float32 as numpy and cv2 compute them.  `out`: a contiguous uint8 [4,H,W,3] tensor to write into.  One launch on
    the current stream, no synchronisation."""
    _lib.need_cuda("eval_frames_u8", im, depth_sil, gt_im, gt_depth)
    H, W = im.shape[-2:]
    if im.shape != (3, H, W) or depth_sil.shape != (3, H, W) or gt_im.shape != (3, H, W) or \
            gt_depth.shape != (1, H, W):
        raise _lib.SplatamB200Error("eval_frames_u8 expects im, depth_sil, gt_im [3,H,W] and gt_depth [1,H,W], got "
                                    "%s" % ([tuple(t.shape) for t in (im, depth_sil, gt_im, gt_depth)],))
    dev = im.device
    lut = jet_lut(dev) if lut is None else lut
    if out is None:
        out = torch.empty(4, H, W, 3, dtype=torch.uint8, device=dev)
    if lut.dtype != torch.uint8 or lut.shape != (256, 3) or not lut.is_contiguous() or \
            out.dtype != torch.uint8 or out.shape != (4, H, W, 3) or not out.is_contiguous():
        raise _lib.SplatamB200Error("eval_frames_u8 needs a contiguous uint8 [256,3] lut and [4,H,W,3] out")
    c = lambda t: t.detach().float().contiguous()
    _lib.call("sb_eval_frames_u8", c(im), c(depth_sil), c(gt_im), c(gt_depth), H, W, lut, out, device=dev)
    return out


class _FrameWriter:
    """Saves the four images of each evaluated frame under out_dir/{FRAME_DIRS} without holding up the evaluation:
    sb_eval_frames_u8 writes one device staging buffer, an async copy moves it to a free pinned host slot, and a writer
    thread waits for that copy's event, encodes the four PNGs with Pillow and frees the slot.  The next frame's kernel
    may reuse the staging buffer at once, since it runs after the copy on the same stream.  `put` blocks only when every
    host slot is busy.  `close` waits for every file and re-raises the first writer error; no thread outlives it.
    File names: <render_prefix>_{i:04d}.png for the renders and gt_{i:04d}.png for the ground truth, with
    i = t + index_offset for frame t."""

    def __init__(self, out_dir, render_prefix, index_offset, H, W, device, threads=None):
        threads = FRAME_WRITER_THREADS if threads is None else threads
        self.dirs = [os.path.join(out_dir, d) for d in FRAME_DIRS]
        for d in self.dirs:
            os.makedirs(d, exist_ok=True)
        self.prefixes = (render_prefix, render_prefix, "gt", "gt")
        self.offset, self.H, self.W, self.device = index_offset, H, W, device
        self.lut = jet_lut(device)
        self.staging = torch.empty(4, H, W, 3, dtype=torch.uint8, device=device)
        n = threads + 2
        self.host = [torch.empty(4, H, W, 3, dtype=torch.uint8).pin_memory() for _ in range(n)]
        self.events = [torch.cuda.Event() for _ in range(n)]
        self.free = queue.SimpleQueue()
        for s in range(n):
            self.free.put(s)
        self.pool = ThreadPoolExecutor(threads, thread_name_prefix="eval-frames")
        self.jobs = []

    def put(self, t, im, depth_sil, gt_im, gt_depth):
        """Enqueues frame t's four images on the current stream (im, depth_sil, gt_im, gt_depth: contiguous float32)."""
        s = self.free.get()
        _lib.call("sb_eval_frames_u8", im, depth_sil, gt_im, gt_depth, self.H, self.W, self.lut, self.staging,
                  device=self.device)
        self.host[s].copy_(self.staging, non_blocking=True)
        self.events[s].record()
        i = t + self.offset
        paths = [os.path.join(d, "%s_%04d.png" % (p, i)) for d, p in zip(self.dirs, self.prefixes)]
        self.jobs.append(self.pool.submit(self._write, s, paths))

    def _write(self, s, paths):
        from PIL import Image
        try:
            self.events[s].synchronize()
            px = self.host[s].numpy()
            for k, path in enumerate(paths):
                Image.fromarray(px[k]).save(path, compress_level=PNG_COMPRESS_LEVEL)
        finally:
            self.free.put(s)

    def close(self):
        self.pool.shutdown(wait=True)
        for job in self.jobs:
            job.result()


def _check_save_frames(name, save_frames, out_dir):
    if save_frames and out_dir is None:
        raise ValueError("%s: save_frames=True needs out_dir" % name)


def select_frames(num_frames, eval_every=1):
    """Indices the reference evaluates: frame 0, then every frame with (t + 1) % eval_every == 0
    (eval_helpers.py:447-448)."""
    return [t for t in range(num_frames) if t == 0 or (t + 1) % eval_every == 0]


def trajectory_ate(params, first_w2c, gt_w2c):
    """ATE of the estimated trajectory (eval_helpers.py:545-575): estimate 0 is the first frame's w2c, estimate t the
    w2c of the normalised camera quaternion and translation of frame t; frames t >= 1 whose ground-truth w2c contains
    NaN are skipped; slam.ate_horn aligns and averages.  Host code over the pose tensors."""
    from .slam import ate_horn
    rots, trans = params["cam_unnorm_rots"].detach(), params["cam_trans"].detach()
    gt = [torch.as_tensor(m) for m in gt_w2c]
    est, ref = [first_w2c], [gt[0]]
    for t in range(1, rots.shape[-1]):
        if torch.isnan(gt[t]).any():
            continue
        est.append(M.camera_w2c(rots[..., t], trans[..., t])[0])
        ref.append(gt[t])
    return ate_horn(ref, est)


def _check_inputs(name, params, frames, lpips):
    _lib.need_cuda(name, params["means3D"], frames[0]["im"])
    H, W = frames[0]["im"].shape[-2:]
    if min(H, W) <= 160:
        raise _lib.SplatamB200Error("%s: MS-SSIM needs a smaller image side > 160, got %dx%d" % (name, W, H))
    if lpips is not None:
        _check_lpips_net(lpips, params["means3D"].device)
    return H, W


def _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused, at_gt_pose=False,
                  count_holes=False, lpips=None, writer=None):
    """Renders frames[t] for t in `ids` and scores each with sb_frame_metrics and MS-SSIM, and with sb_lpips on the
    same weighted images when `lpips` (an LpipsAlex) is given: float64 device rows [len(ids), 7] (columns _PSNR ..
    _LPIPS; _LPIPS stays 0 without `lpips`).  at_gt_pose: render at the frame's gt_w2c instead of its estimated pose.
    count_holes: also returns [len(ids), 7] rows of a presence-masked sb_frame_metrics call into scratch images, whose
    _NVALID - _NMASK is the number of valid-depth pixels the silhouette leaves uncovered (None otherwise).
    writer: a _FrameWriter that is handed each frame's unmasked renders and ground truth."""
    render = M.default_render if render is None else render
    if fused is None:
        fused = render is M.default_render
    dev = params["means3D"].device
    H, W = frames[0]["im"].shape[-2:]
    metrics = torch.zeros(len(ids), 7, dtype=torch.float64, device=dev)
    presence = torch.zeros_like(metrics) if count_holes else None
    w_im = torch.empty(3, H, W, dtype=torch.float32, device=dev)
    w_gt = torch.empty_like(w_im)
    ws_frame = torch.empty(_lib.nbytes("sb_frame_metrics_workspace_bytes", H, W), dtype=torch.uint8, device=dev)
    ws_ssim = torch.empty(_lib.nbytes("sb_ms_ssim_workspace_bytes", 1, 3, H, W), dtype=torch.uint8, device=dev)
    if lpips is not None:
        ws_lpips = torch.empty(_lib.nbytes("sb_lpips_workspace_bytes", 1, H, W), dtype=torch.uint8, device=dev)
    with torch.no_grad(), torch.cuda.device(dev):
        for k, t in enumerate(ids):
            fr = dict(frames[t], cam=cam)
            if at_gt_pose:
                fr["pose"] = M.gt_pose(fr["gt_w2c"].to(dev).float())
            im, depth_sil, _, _ = M._render_pair(params, fr, render, fused, camera_grad=False)
            im, depth_sil = im.float().contiguous(), depth_sil.float().contiguous()
            gt_im, gt_d = fr["im"].float().contiguous(), fr["depth"].float().contiguous()
            _lib.call("sb_frame_metrics", im, depth_sil, gt_im, gt_d, H, W, float(sil_thres), use_presence, w_im, w_gt,
                      ws_frame, ws_frame.numel(), metrics[k], device=dev)
            _ms_ssim_into(w_im[None], w_gt[None], 1.0, None, metrics[k, _SSIM], ws_ssim)
            if writer is not None:
                writer.put(t, im, depth_sil, gt_im, gt_d)
            if lpips is not None:                # sb_lpips clamps the weighted images to [0, 1] as it loads them
                _lpips_into(w_im[None], w_gt[None], lpips, None, metrics[k, _LPIPS], ws_lpips)
            if count_holes:
                if use_presence:
                    presence[k].copy_(metrics[k])
                else:
                    _lib.call("sb_frame_metrics", im, depth_sil, gt_im, gt_d, H, W, float(sil_thres), 1, w_im, w_gt,
                              ws_frame, ws_frame.numel(), presence[k], device=dev)
    return metrics, presence


def _per_frame(m, lpips):
    out = dict(psnr_per_frame=m[:, _PSNR], ms_ssim_per_frame=m[:, _SSIM], depth_rmse_per_frame=m[:, _RMSE],
               depth_l1_per_frame=m[:, _L1], valid_pixels=m[:, _NVALID].astype(np.int64),
               mask_pixels=m[:, _NMASK].astype(np.int64))
    if lpips is not None:
        out["lpips_per_frame"] = m[:, _LPIPS]
    return out


def _write_lists(out_dir, out):
    os.makedirs(out_dir, exist_ok=True)
    for name, key in (("psnr", "psnr_per_frame"), ("rmse", "depth_rmse_per_frame"), ("l1", "depth_l1_per_frame"),
                      ("ssim", "ms_ssim_per_frame"), ("lpips", "lpips_per_frame")):
        if key in out:
            np.savetxt(os.path.join(out_dir, name + ".txt"), out[key])


def evaluate(params, frames, cam, sil_thres, mapping_iters, add_new_gaussians, eval_every=1, gt_w2c=None, fused=None,
             render=None, out_dir=None, lpips=None, at_gt_pose=False, save_frames=False):
    """The reference's final `eval` over this repo's frame dicts (id, im [3,H,W] in [0,1], depth [1,H,W], w2c = the
    first frame's w2c, as slam.render_frame builds them).  `params`: the final Gaussians plus cam_unnorm_rots /
    cam_trans [.., T]; `cam`: the raster settings; frames are evaluated as `select_frames` picks them.

    Masks as in the reference: valid = gt depth > 0; when mapping_iters == 0 and not add_new_gaussians the images and
    the depth error are also masked by silhouette > sil_thres.  Rendered images are not clamped.
      psnr        mean over the three channels of the per-channel PSNR of the weighted images, each MSE taken over
                  all H*W pixels (calc_psnr)
      ms_ssim     MS-SSIM of the weighted images (`ms_ssim`)
      depth_rmse  sum(sqrt(e^2) * valid) / sum(valid): the reference takes sqrt(x^2) element-wise, so this is a
                  masked mean absolute error; it is reported as the reference defines it
      depth_l1    sum(|e| * valid) / sum(valid)
      ate         `trajectory_ate` against gt_w2c (a list of T ground-truth w2c matrices), None without it
      lpips       with `lpips` (an LpipsAlex on the map's device, `LpipsAlex.load`): LPIPS of the weighted images clamped
                  to [0, 1] (`lpips`), else None
    Returns those averages plus frame_ids and the per-frame arrays psnr_per_frame, ms_ssim_per_frame,
    depth_rmse_per_frame, depth_l1_per_frame, valid_pixels, mask_pixels and, with `lpips`, lpips_per_frame.
    `out_dir`: also writes psnr.txt, rmse.txt, l1.txt, ssim.txt and, with `lpips`, lpips.txt as the reference does
    (np.savetxt, one value per evaluated frame).
    fused / render: as for mapping (`mapping._render_pair`); fused defaults to the fast path on CUDA.
    at_gt_pose: render every frame at its `gt_w2c` instead of its estimated pose, as the offline drivers' `eval` does
    (R/utils/gs_helpers.py:463-510); `params` then needs no camera tensors.
    save_frames: also writes, for each evaluated frame t (its position in `frames`), the reference's four PNGs
    (`eval_frames_u8` of the unmasked renders): out_dir/rendered_rgb/gs_{t:04d}.png, rendered_depth/gs_{t:04d}.png,
    rgb/gt_{t:04d}.png and depth/gt_{t:04d}.png.  Needs `out_dir` (ValueError otherwise); returns once every file is
    written and re-raises a writer's error."""
    _check_save_frames("evaluate", save_frames, out_dir)
    H, W = _check_inputs("evaluate", params, frames, lpips)
    ids = select_frames(len(frames), eval_every)
    use_presence = int(mapping_iters == 0 and not add_new_gaussians)
    writer = _FrameWriter(out_dir, "gs", 0, H, W, params["means3D"].device) if save_frames else None
    try:
        metrics, _ = _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused,
                                   at_gt_pose=at_gt_pose, lpips=lpips, writer=writer)
    finally:
        if writer is not None:
            writer.close()
    m = metrics.cpu().numpy()                    # the one device-to-host read
    out = dict(frame_ids=[int(frames[t]["id"]) for t in ids], **_per_frame(m, lpips))
    out.update(psnr=float(m[:, _PSNR].mean()), ms_ssim=float(m[:, _SSIM].mean()),
               depth_rmse=float(m[:, _RMSE].mean()), depth_l1=float(m[:, _L1].mean()),
               lpips=None if lpips is None else float(m[:, _LPIPS].mean()),
               ate=None if gt_w2c is None else trajectory_ate(params, frames[0]["w2c"], gt_w2c))
    if out_dir is not None:
        _write_lists(out_dir, out)
    return out


def select_nvs_frames(num_frames, eval_every=1):
    """Indices the reference's eval_nvs evaluates in a test split: frame 0 (the first train frame) never; frame t >= 1
    (test view k = t - 1) when k == 0 or (k + 1) % eval_every == 0 (eval_helpers.py:666-669)."""
    return [t for t in range(1, num_frames) if t == 1 or t % eval_every == 0]


def evaluate_nvs(params, frames, cam, sil_thres, mapping_iters, add_new_gaussians, eval_every=1, fused=None,
                 render=None, out_dir=None, lpips=None, save_frames=False):
    """The reference's novel-view evaluation `eval_nvs` over a test split (datasets.RGBDSequence(..., split="test"):
    frame 0 is the first train frame, frames 1.. the held-out views, each with its ground-truth `gt_w2c`).  Frames are
    picked by `select_nvs_frames` and rendered at gt_w2c -- the means transformed by it, anisotropic rotations
    composed with its normalised quaternion -- not at an estimated pose; `params` needs no camera tensors.

    Masks and per-frame metrics are those of `evaluate`.  A view is valid unless its holes -- pixels with gt depth > 0
    and silhouette <= sil_thres -- exceed 0.1 % of the image (holes * 1000 > H * W; the reference's float32 percentage
    test agrees at the datasets' image sizes).  Returns the averages psnr, ms_ssim, depth_rmse and depth_l1 over the
    valid views (NaN when none is valid), lpips (the same average with `lpips`, an LpipsAlex, else None), frame_ids
    (indices into `frames`), the per-frame arrays of `evaluate` over every evaluated view, hole_pixels and
    valid_nvs_frames (bool).  `out_dir`: also writes psnr.txt, rmse.txt, l1.txt, ssim.txt (and lpips.txt with `lpips`)
    over every evaluated view and valid_nvs_frames.npy, as the reference does.
    save_frames: the four PNGs of `evaluate` for every evaluated view, valid or not, named by the test-view index
    k = t - 1: rendered_rgb/splatam_{k:04d}.png, rendered_depth/splatam_{k:04d}.png, rgb/gt_{k:04d}.png and
    depth/gt_{k:04d}.png.  Needs `out_dir` (ValueError otherwise)."""
    _check_save_frames("evaluate_nvs", save_frames, out_dir)
    H, W = _check_inputs("evaluate_nvs", params, frames, lpips)
    ids = select_nvs_frames(len(frames), eval_every)
    use_presence = int(mapping_iters == 0 and not add_new_gaussians)
    writer = _FrameWriter(out_dir, "splatam", -1, H, W, params["means3D"].device) if save_frames else None
    try:
        metrics, presence = _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused,
                                          at_gt_pose=True, count_holes=True, lpips=lpips, writer=writer)
    finally:
        if writer is not None:
            writer.close()
    m, p = torch.stack([metrics, presence]).cpu().numpy()          # the one device-to-host read
    holes = (p[:, _NVALID] - p[:, _NMASK]).astype(np.int64)
    valid = holes * 1000 <= H * W
    out = dict(frame_ids=[int(frames[t]["id"]) for t in ids], hole_pixels=holes, valid_nvs_frames=valid,
               **_per_frame(m, lpips))
    avg = lambda c: float(m[valid, c].mean()) if valid.any() else float("nan")
    out.update(psnr=avg(_PSNR), ms_ssim=avg(_SSIM), depth_rmse=avg(_RMSE), depth_l1=avg(_L1),
               lpips=None if lpips is None else avg(_LPIPS))
    if out_dir is not None:
        _write_lists(out_dir, out)
        np.save(os.path.join(out_dir, "valid_nvs_frames.npy"), valid)
    return out
