"""Host-side wrappers of the fused training ops in libsplatam_b200.so (csrc/train_ops.cu):
``FusedAdam`` over a flat parameter buffer and ``image_loss`` = 0.8*L1 + 0.2*(1-SSIM) with a fused
backward.  CUDA only; no CPU fallback."""
import ctypes

import torch

from . import _lib


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class FusedAdam:
    """torch.optim.Adam semantics (betas, eps, per-segment lr; no amsgrad / weight decay) over ONE flat
    fp32 buffer and its flat gradient; one kernel launch per step."""

    def __init__(self, flat, flat_grad, seg_sizes, seg_lrs, betas=(0.9, 0.999), eps=1e-15, exp_avg=None,
                 exp_avg_sq=None, step=0):
        if not flat.is_cuda:
            raise _lib.SplatamB200Error("FusedAdam needs CUDA tensors (there is no CPU fallback)")
        self.flat, self.flat_grad = flat, flat_grad
        self.m = torch.zeros_like(flat) if exp_avg is None else exp_avg
        self.v = torch.zeros_like(flat) if exp_avg_sq is None else exp_avg_sq
        assert self.m.numel() == flat.numel() and self.v.numel() == flat.numel()
        ends, acc = [], 0
        for n in seg_sizes:
            acc += int(n)
            ends.append(acc)
        assert acc == flat.numel() and len(ends) == len(seg_lrs) <= 16
        self.n = len(ends)
        self.seg_end = (ctypes.c_uint32 * self.n)(*ends)
        self.seg_lr = (ctypes.c_double * self.n)(*[float(x) for x in seg_lrs])
        self.betas, self.eps, self.t = betas, eps, int(step)
        self.clock = None           # device-side step clock of the guarded mode (created on first use)

    def _clock(self):
        if self.clock is None:
            lib = _lib.load()
            nints = (int(lib.sb_adam_clock_bytes()) + 3) // 4
            self.clock = torch.zeros(nints, dtype=torch.int32, device=self.flat.device)
            self.clock[0] = self.t
        return self.clock

    def step_guarded(self, skip_if_nonzero=None):
        """One Adam step whose step count lives on the device; a no-op (count unchanged) when the device float
        `skip_if_nonzero[0]` is non-zero.  Never synchronises.  `applied_steps()` reads the clock back."""
        lib = _lib.load()
        clk = self._clock()
        with torch.cuda.device(self.flat.device):
            _lib.check(lib.sb_adam_step_guarded(
                self.flat.data_ptr(), self.flat_grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.flat.numel(),
                self.seg_end, self.seg_lr, self.n, clk.data_ptr(),
                None if skip_if_nonzero is None else skip_if_nonzero.data_ptr(), self.betas[0], self.betas[1], self.eps,
                _stream(self.flat.device)), "sb_adam_step_guarded")

    def applied_steps(self):
        """(steps applied, steps skipped) of the guarded mode; synchronises."""
        if self.clock is None:
            return self.t, 0
        c = self.clock[:2].tolist()
        self.t = int(c[0])
        return int(c[0]), int(c[1])

    def step(self):
        if self.clock is not None:      # once guarded, the device clock is the step count
            return self.step_guarded(None)
        self.t += 1
        lib = _lib.load()
        with torch.cuda.device(self.flat.device):
            _lib.check(lib.sb_adam_step(self.flat.data_ptr(), self.flat_grad.data_ptr(), self.m.data_ptr(),
                                        self.v.data_ptr(), self.flat.numel(), self.seg_end, self.seg_lr, self.n, self.t,
                                        self.betas[0], self.betas[1], self.eps, _stream(self.flat.device)), "sb_adam_step")


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, w_l1, w_ssim):
        lib = _lib.load()
        x, y = x.contiguous().float(), y.contiguous().float()
        C, H, W = x.shape
        dev = x.device
        work = torch.empty(lib.sb_image_loss_workspace_floats(C, H, W), dtype=torch.float32, device=dev)
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.sb_image_loss_forward(x.data_ptr(), y.data_ptr(), C, H, W, work.data_ptr(), sums.data_ptr(),
                                                 _stream(dev)), "sb_image_loss_forward")
        n = float(C * H * W)
        ctx.save_for_backward(x, y, work)
        ctx.w = (float(w_l1), float(w_ssim))
        return (w_l1 * sums[1] / n + w_ssim * (1.0 - sums[0] / n)).float()

    @staticmethod
    def backward(ctx, grad_out):
        lib = _lib.load()
        x, y, work = ctx.saved_tensors
        C, H, W = x.shape
        gx = torch.empty_like(x)
        go = grad_out.contiguous().float().reshape(1)
        with torch.cuda.device(x.device):
            _lib.check(lib.sb_image_loss_backward(x.data_ptr(), y.data_ptr(), C, H, W, work.data_ptr(), go.data_ptr(),
                                                  ctx.w[1], ctx.w[0], gx.data_ptr(), _stream(x.device)),
                       "sb_image_loss_backward")
        return gx, None, None, None


def image_loss(im, gt, w_l1=0.8, w_ssim=0.2):
    """0.8 * mean|im-gt| + 0.2 * (1 - SSIM(im, gt)) -- SplaTAM's mapping RGB loss (R/scripts/splatam.py:290)."""
    if not im.is_cuda:
        raise _lib.SplatamB200Error("image_loss needs CUDA tensors (there is no CPU fallback)")
    return _ImageLoss.apply(im, gt, w_l1, w_ssim)


class _MaskedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_sil, gt_depth, im, gt_im, sil_thres, use_sil, depth_mean):
        lib = _lib.load()
        dev = depth_sil.device
        depth_sil, gt_depth = depth_sil.contiguous().float(), gt_depth.contiguous().float()
        _, H, W = depth_sil.shape
        have_im = im is not None
        if have_im:
            im, gt_im = im.contiguous().float(), gt_im.contiguous().float()
        sums = torch.empty(3, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.sb_masked_l1_forward(depth_sil.data_ptr(), gt_depth.data_ptr(),
                                                im.data_ptr() if have_im else None, gt_im.data_ptr() if have_im else None,
                                                H, W, float(sil_thres), int(use_sil), sums.data_ptr(), _stream(dev)),
                       "sb_masked_l1_forward")
        ctx.save_for_backward(depth_sil, gt_depth, sums, *([im, gt_im] if have_im else []))
        ctx.cfg = (float(sil_thres), int(use_sil), int(depth_mean), have_im)
        l_depth = (sums[0] / sums[1] if depth_mean else sums[0]).float()
        return l_depth, sums[2].float()

    @staticmethod
    def backward(ctx, g_depth, g_im):
        lib = _lib.load()
        sil_thres, use_sil, depth_mean, have_im = ctx.cfg
        depth_sil, gt_depth, sums, *rest = ctx.saved_tensors
        dev = depth_sil.device
        _, H, W = depth_sil.shape
        grad_ds = torch.empty_like(depth_sil)
        grad_im = torch.empty_like(rest[0]) if have_im else None
        gd = g_depth.contiguous().float().reshape(1)
        gi = g_im.contiguous().float().reshape(1) if have_im else None
        with torch.cuda.device(dev):
            _lib.check(lib.sb_masked_l1_backward(
                depth_sil.data_ptr(), gt_depth.data_ptr(), rest[0].data_ptr() if have_im else None,
                rest[1].data_ptr() if have_im else None, H, W, sil_thres, use_sil, depth_mean, sums.data_ptr(),
                gd.data_ptr(), gi.data_ptr() if have_im else None, grad_ds.data_ptr(),
                grad_im.data_ptr() if have_im else None, _stream(dev)), "sb_masked_l1_backward")
        return grad_ds, None, grad_im, None, None, None, None


def masked_l1(depth_sil, gt_depth, im=None, gt_im=None, sil_thres=0.99, use_sil=False, depth_mean=True):
    """(loss_depth, loss_im) of SplaTAM's get_loss: validity (and optionally silhouette) masked L1 over the depth
    channel of the [3,H,W] depth/silhouette/depth^2 render and, if `im` is given, over the RGB image (sum)."""
    if not depth_sil.is_cuda:
        raise _lib.SplatamB200Error("masked_l1 needs CUDA tensors (there is no CPU fallback)")
    return _MaskedL1.apply(depth_sil, gt_depth, im, gt_im, sil_thres, use_sil, depth_mean)
