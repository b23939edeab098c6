"""``prepare_gaussians``: SplaTAM's per-iteration parameter glue as ONE forward and ONE backward kernel
(csrc/prepare.cu).  Returns the tensors the two raster calls consume:

    means_cam, rotations, opacities, scales3, depth_sil_colors =
        prepare_gaussians(means3D, unnorm_rotations, logit_opacities, log_scales, rel_w2c, cam_rot, w2c0)

equal (to float rounding) to transform_to_frame + transformed_params2rendervar +
transformed_params2depthplussilhouette of R/utils/slam_helpers.py.  CUDA only."""
import torch

from . import _lib


class _Prepare(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, unnorm, logit, log_scales, rel_w2c, cam_rot, w2c0):
        dev = means3D.device
        P, sd = means3D.shape[0], log_scales.shape[1]
        c = lambda t: t.detach().contiguous().float()
        means3D, unnorm, logit, log_scales = c(means3D), c(unnorm), c(logit), c(log_scales)
        rel, cr, w0 = c(rel_w2c), c(cam_rot).reshape(4), c(w2c0)
        e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        means_cam, rot, opac, sc3, dcols = e(P, 3), e(P, 4), e(P, 1), e(P, 3), e(P, 3)
        _lib.call("sb_prepare_forward", P, sd, means3D, unnorm, logit, log_scales, rel, cr, w0, means_cam, rot, opac,
                  sc3, dcols, device=dev)
        ctx.save_for_backward(means3D, unnorm, rel, cr, w0, means_cam, opac, sc3)
        ctx.sd = sd
        ctx.want_pose = bool(ctx.needs_input_grad[4] or ctx.needs_input_grad[5])
        ctx.shapes = (logit.shape, log_scales.shape, rel_w2c.shape, cam_rot.shape)
        return means_cam, rot, opac, sc3, dcols

    @staticmethod
    def backward(ctx, g_means_cam, g_rot, g_opac, g_sc3, g_dcols):
        means3D, unnorm, rel, cr, w0, means_cam, opac, sc3 = ctx.saved_tensors
        dev = means3D.device
        P = means3D.shape[0]
        keep = [None if t is None else t.contiguous().float() for t in (g_means_cam, g_rot, g_opac, g_sc3, g_dcols)]
        e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        g_means, g_unnorm, g_logit, g_ls = e(P, 3), e(P, 4), e(*ctx.shapes[0]), e(*ctx.shapes[1])
        pose = torch.empty(16, dtype=torch.float64, device=dev) if ctx.want_pose else None     # zeroed by the call
        _lib.call("sb_prepare_backward", P, ctx.sd, int(ctx.want_pose), means3D, unnorm, rel, cr, w0, means_cam, opac,
                  sc3, *keep, g_means, g_unnorm, g_logit, g_ls, pose, device=dev)
        g_rel = g_cr = None
        if ctx.want_pose:
            g_rel = torch.zeros(4, 4, dtype=torch.float32, device=dev)
            g_rel[:3, :] = pose[:12].view(3, 4)
            g_rel = g_rel.reshape(ctx.shapes[2])
            g_cr = pose[12:].float().reshape(ctx.shapes[3])
        return g_means, g_unnorm, g_logit, g_ls, g_rel, g_cr, None


def prepare_gaussians(means3D, unnorm_rotations, logit_opacities, log_scales, rel_w2c, cam_rot, w2c0):
    _lib.need_cuda("prepare_gaussians", means3D)
    return _Prepare.apply(means3D, unnorm_rotations, logit_opacities, log_scales, rel_w2c, cam_rot, w2c0)
