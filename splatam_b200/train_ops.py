"""Host-side wrappers of the fused training ops in libsplatam_b200.so (csrc/train_ops.cu):
``FusedAdam`` over a flat parameter buffer and ``image_loss`` = 0.8*L1 + 0.2*(1-SSIM) with a fused
backward.  CUDA only; no CPU fallback."""
import ctypes

import torch

from . import _lib


class FusedAdam:
    """torch.optim.Adam semantics (betas, eps, per-segment lr; no amsgrad / weight decay) over ONE flat
    fp32 buffer and its flat gradient; one kernel launch per step."""

    def __init__(self, flat, flat_grad, seg_sizes, seg_lrs, betas=(0.9, 0.999), eps=1e-15, exp_avg=None,
                 exp_avg_sq=None, step=0):
        _lib.need_cuda("FusedAdam", flat)
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

    def set_lr(self, segment, lr):
        """Learning rate of segment `segment` from the next step on: a host-side write into the array each launch
        reads (no reallocation, no synchronisation)."""
        if not 0 <= int(segment) < self.n:
            raise IndexError("segment %d out of range for %d segments" % (segment, self.n))
        self.seg_lr[int(segment)] = float(lr)

    def _clock(self):
        if self.clock is None:
            nints = (int(_lib.load().sb_adam_clock_bytes()) + 3) // 4
            self.clock = torch.zeros(nints, dtype=torch.int32, device=self.flat.device)
            self.clock[0] = self.t
        return self.clock

    def step_guarded(self, skip_if_nonzero=None):
        """One Adam step whose step count lives on the device; a no-op (count unchanged) when the device float
        `skip_if_nonzero[0]` is non-zero.  Never synchronises.  `applied_steps()` reads the clock back."""
        _lib.call("sb_adam_step_guarded", self.flat, self.flat_grad, self.m, self.v, self.flat.numel(), self.seg_end,
                  self.seg_lr, self.n, self._clock(), skip_if_nonzero, self.betas[0], self.betas[1], self.eps,
                  device=self.flat.device)

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
        _lib.call("sb_adam_step", self.flat, self.flat_grad, self.m, self.v, self.flat.numel(), self.seg_end,
                  self.seg_lr, self.n, self.t, self.betas[0], self.betas[1], self.eps, device=self.flat.device)


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, w_l1, w_ssim):
        x, y = x.contiguous().float(), y.contiguous().float()
        C, H, W = x.shape
        dev = x.device
        work = torch.empty(_lib.load().sb_image_loss_workspace_floats(C, H, W), dtype=torch.float32, device=dev)
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        _lib.call("sb_image_loss_forward", x, y, C, H, W, work, sums, device=dev)
        n = float(C * H * W)
        ctx.save_for_backward(x, y, work)
        ctx.w = (float(w_l1), float(w_ssim))
        return (w_l1 * sums[1] / n + w_ssim * (1.0 - sums[0] / n)).float()

    @staticmethod
    def backward(ctx, grad_out):
        x, y, work = ctx.saved_tensors
        C, H, W = x.shape
        gx = torch.empty_like(x)
        go = grad_out.contiguous().float().reshape(1)
        _lib.call("sb_image_loss_backward", x, y, C, H, W, work, go, ctx.w[1], ctx.w[0], gx, device=x.device)
        return gx, None, None, None


def image_loss(im, gt, w_l1=0.8, w_ssim=0.2):
    """0.8 * mean|im-gt| + 0.2 * (1 - SSIM(im, gt)) -- SplaTAM's mapping RGB loss (R/scripts/splatam.py:290)."""
    _lib.need_cuda("image_loss", im)
    return _ImageLoss.apply(im, gt, w_l1, w_ssim)


class _MaskedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_sil, gt_depth, im, gt_im, sil_thres, use_sil, depth_mean):
        dev = depth_sil.device
        depth_sil, gt_depth = depth_sil.contiguous().float(), gt_depth.contiguous().float()
        _, H, W = depth_sil.shape
        have_im = im is not None
        if have_im:
            im, gt_im = im.contiguous().float(), gt_im.contiguous().float()
        sums = torch.empty(3, dtype=torch.float64, device=dev)
        _lib.call("sb_masked_l1_forward", depth_sil, gt_depth, im, gt_im, H, W, float(sil_thres), int(use_sil), sums,
                  device=dev)
        ctx.save_for_backward(depth_sil, gt_depth, sums, *([im, gt_im] if have_im else []))
        ctx.cfg = (float(sil_thres), int(use_sil), int(depth_mean), have_im)
        l_depth = (sums[0] / sums[1] if depth_mean else sums[0]).float()
        return l_depth, sums[2].float()

    @staticmethod
    def backward(ctx, g_depth, g_im):
        sil_thres, use_sil, depth_mean, have_im = ctx.cfg
        depth_sil, gt_depth, sums, *rest = ctx.saved_tensors
        im, gt_im = rest if have_im else (None, None)
        _, H, W = depth_sil.shape
        grad_ds = torch.empty_like(depth_sil)
        grad_im = torch.empty_like(im) if have_im else None
        gd = g_depth.contiguous().float().reshape(1)
        gi = g_im.contiguous().float().reshape(1) if have_im else None
        _lib.call("sb_masked_l1_backward", depth_sil, gt_depth, im, gt_im, H, W, sil_thres, use_sil, depth_mean, sums,
                  gd, gi, grad_ds, grad_im, device=depth_sil.device)
        return grad_ds, None, grad_im, None, None, None, None


def masked_l1(depth_sil, gt_depth, im=None, gt_im=None, sil_thres=0.99, use_sil=False, depth_mean=True):
    """(loss_depth, loss_im) of SplaTAM's get_loss: validity (and optionally silhouette) masked L1 over the depth
    channel of the [3,H,W] depth/silhouette/depth^2 render and, if `im` is given, over the RGB image (sum)."""
    _lib.need_cuda("masked_l1", depth_sil)
    return _MaskedL1.apply(depth_sil, gt_depth, im, gt_im, sil_thres, use_sil, depth_mean)
