"""Keyframe-sharded mapping step (SURVEY.md section 8e) -- NEW functionality; the reference mapping
loop is single-GPU and renders ONE keyframe per Adam step (R/scripts/splatam.py:828-885).

One process per GPU.  Every rank holds the full Gaussian parameter set; in a K-rank step rank r
renders keyframe ``perm[step*K + r]`` of the selected window (2 raster calls, RGB and
depth/silhouette, exactly SplaTAM's ``get_loss(mapping=True)``: R/scripts/splatam.py:214-347), the
per-Gaussian gradients of all ranks are summed with ONE all-reduce over a flat, packed gradient
bucket (NCCL over NVLink on the box, gloo in the CPU tests), and every rank applies the same Adam
update so the replicas stay bit-identical without any parameter broadcast.  Tracking stays
single-GPU.  A K-rank step is a K-keyframe minibatch: gradients equal a 1-process accumulation over
the same K keyframes up to float summation order (tests/test_mapping_gloo.py).

The PyTorch glue below restates R/utils/slam_helpers.py:124-139,196-304 and
R/utils/slam_external.py:25-97 (transform_to_frame, rendervars, L1, SSIM); it is host-side plumbing
around the operator, not part of the rasterizer hot path.
"""
import math

import torch
import torch.nn.functional as F

from .formats import GAUSSIAN_KEYS
from .rasterizer import GaussianRasterizer


def build_rotation(q):
    """Unit-quaternion (w,x,y,z) rows -> rotation matrices (R/utils/slam_external.py:25-42)."""
    q = q / torch.sqrt((q * q).sum(-1, keepdim=True))
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def quat_mult(q1, q2):
    """Hamilton product, (w,x,y,z) convention (R/utils/slam_helpers.py:24-31)."""
    w1, x1, y1, z1 = q1.T
    w2, x2, y2, z2 = q2.T
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2]).T


def matrix_to_quaternion(R):
    """Quaternion (w,x,y,z) of a 3x3 rotation matrix, up to sign, without a host synchronisation.

    For a unit quaternion, 1 + R00 + R11 + R22 = 4w^2, 1 + R00 - R11 - R22 = 4x^2, 1 - R00 + R11 - R22 = 4y^2 and
    1 - R00 - R11 + R22 = 4z^2, and the off-diagonal sums and differences are 4wx = R21 - R12, 4wy = R02 - R20,
    4wz = R10 - R01, 4xy = R10 + R01, 4xz = R02 + R20, 4yz = R12 + R21.  Row k of `cand` is 4 q_k q / (4 |q_k|) = +-q;
    the row of the largest |q_k| (at least 1/2) is the well-conditioned one."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = R.reshape(9).unbind()
    four_sq = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22])
    cand = torch.stack([torch.stack([four_sq[0], m21 - m12, m02 - m20, m10 - m01]),
                        torch.stack([m21 - m12, four_sq[1], m10 + m01, m02 + m20]),
                        torch.stack([m02 - m20, m10 + m01, four_sq[2], m12 + m21]),
                        torch.stack([m10 - m01, m02 + m20, m12 + m21, four_sq[3]])])
    cand = cand / (2 * torch.sqrt(four_sq.clamp(min=0)))[:, None]
    return cand.index_select(0, four_sq.argmax().reshape(1))[0]


def gt_pose(w2c):
    """(w2c, normalised quaternion of its rotation [1,4]): the pose argument of a render at a given w2c matrix (the
    frames' "pose" key), as the reference's eval_nvs transforms the Gaussians by a ground-truth w2c."""
    return w2c, F.normalize(matrix_to_quaternion(w2c[:3, :3]).unsqueeze(0))


def camera_w2c(rot, tran):
    """(rel_w2c [4,4], normalised camera quaternion [1,4]) of an unnormalised camera quaternion [1,4] and a
    translation [1,3] (R/utils/slam_helpers.py:266-275)."""
    cam_rot = F.normalize(rot)
    rel_w2c = torch.eye(4, device=rot.device, dtype=torch.float32)
    rel_w2c[:3, :3] = build_rotation(cam_rot)
    rel_w2c[:3, 3] = tran
    return rel_w2c, cam_rot


def pose_matrices(params, time_idx, camera_grad=False):
    """camera_w2c of frame `time_idx`; the pose gets gradient only if `camera_grad`."""
    rot, tran = params["cam_unnorm_rots"][..., time_idx], params["cam_trans"][..., time_idx]
    if not camera_grad:
        rot, tran = rot.detach(), tran.detach()
    return camera_w2c(rot, tran)


def transform_to_frame(params, time_idx, gaussians_grad, camera_grad, pose=None):
    """World -> camera-frame Gaussians for frame `time_idx` (R/utils/slam_helpers.py:252-304), or for the given
    `pose` = (w2c [4,4], normalised quaternion [1,4]) instead of the frame's estimated one."""
    rel_w2c, cam_rot = pose_matrices(params, time_idx, camera_grad) if pose is None else pose
    dev = params["means3D"].device
    pts, unnorm = params["means3D"], params["unnorm_rotations"]
    if not gaussians_grad:
        pts, unnorm = pts.detach(), unnorm.detach()
    pts4 = torch.cat((pts, torch.ones(pts.shape[0], 1, device=dev)), dim=1)
    out = {"means3D": (rel_w2c @ pts4.T).T[:, :3]}
    if params["log_scales"].shape[1] == 1:            # isotropic: rotations irrelevant
        out["unnorm_rotations"] = unnorm
    else:
        out["unnorm_rotations"] = quat_mult(cam_rot, F.normalize(unnorm))
    return out


def _scales(params):
    ls = params["log_scales"]
    return torch.exp(torch.tile(ls, (1, 3)) if ls.shape[1] == 1 else ls)


def rgb_rendervar(params, tg):
    """R/utils/slam_helpers.py:124-139."""
    return dict(means3D=tg["means3D"], colors_precomp=params["rgb_colors"],
                rotations=F.normalize(tg["unnorm_rotations"]), opacities=torch.sigmoid(params["logit_opacities"]),
                scales=_scales(params), means2D=torch.zeros_like(params["means3D"], requires_grad=True) + 0)


def depth_sil_rendervar(params, w2c, tg):
    """colours = [z, 1, z^2] in the camera frame (R/utils/slam_helpers.py:196-249)."""
    pts = tg["means3D"]
    pts4 = torch.cat((pts, torch.ones_like(pts[:, :1])), dim=-1)
    z = (w2c @ pts4.T).T[:, 2:3]
    col = torch.cat((z, torch.ones_like(z), z * z), dim=1)
    return dict(means3D=pts, colors_precomp=col, rotations=F.normalize(tg["unnorm_rotations"]),
                opacities=torch.sigmoid(params["logit_opacities"]), scales=_scales(params),
                means2D=torch.zeros_like(params["means3D"], requires_grad=True) + 0)


_POSE_CACHE = {}


def _pose_cache_get(rots_all, trans_all, time_idx):
    """Cache of (rel_w2c, cam_rot) per (pose tensors, their versions, frame).  Keys use id(): every entry holds weak
    references to the two tensors and is only honoured while both are the very same live objects, so a recycled
    id can never return another tensor's pose."""
    key = (id(rots_all), id(trans_all), rots_all._version, trans_all._version, int(time_idx))
    hit = _POSE_CACHE.get(key)
    if hit is not None and hit[0]() is rots_all and hit[1]() is trans_all:
        return key, hit[2]
    return key, None


def _pose_cache_put(key, rots_all, trans_all, value):
    import weakref
    if len(_POSE_CACHE) > 256:
        _POSE_CACHE.clear()
    _POSE_CACHE[key] = (weakref.ref(rots_all), weakref.ref(trans_all), value)


def fused_pose_cached(params, time_idx):
    """Cached (rel_w2c, cam_rot) of a frame whose pose is not being optimised."""
    rots_all, trans_all = params["cam_unnorm_rots"], params["cam_trans"]
    key, hit = _pose_cache_get(rots_all, trans_all, time_idx)
    if hit is None:
        hit = pose_matrices(params, time_idx)
        _pose_cache_put(key, rots_all, trans_all, hit)
    return hit


def fused_rendervars(params, time_idx, w2c0, camera_grad, pose=None):
    """Both rendervars of one frame from ONE fused kernel (splatam_b200/prepare.py); equals
    transform_to_frame + rgb_rendervar + depth_sil_rendervar above to float rounding.  `pose` = precomputed
    (rel_w2c, cam_rot) tensors (the CUDA-graph path keeps them in static buffers)."""
    from .prepare import prepare_gaussians
    if pose is not None:
        rel_w2c, cam_rot = pose
    elif not camera_grad:     # poses are constants of the mapping loop: build each frame's matrix once
        rel_w2c, cam_rot = fused_pose_cached(params, time_idx)
    else:
        rel_w2c, cam_rot = pose_matrices(params, time_idx, camera_grad)
    means_cam, rots, opac, sc3, dcols = prepare_gaussians(params["means3D"], params["unnorm_rotations"],
                                                          params["logit_opacities"], params["log_scales"], rel_w2c,
                                                          cam_rot, w2c0)
    z2 = lambda: torch.zeros_like(params["means3D"], requires_grad=True) + 0
    rgb = dict(means3D=means_cam, colors_precomp=params["rgb_colors"], rotations=rots, opacities=opac, scales=sc3,
               means2D=z2())
    dep = dict(means3D=means_cam, colors_precomp=dcols, rotations=rots, opacities=opac, scales=sc3, means2D=z2())
    return rgb, dep


def _ssim_window(channel, device, size=11, sigma=1.5):
    g = torch.tensor([math.exp(-(x - size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(size)])
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).float()[None, None].expand(channel, 1, size, size).contiguous().to(device)


def calc_ssim(img1, img2, window_size=11):
    """R/utils/slam_external.py:66-97 (mean SSIM, 11x11 Gaussian window, sigma 1.5)."""
    return ssim_map(img1, img2, window_size).mean()


def ssim_map(img1, img2, window_size=11):
    """The per-pixel, per-channel SSIM of `calc_ssim`."""
    ch = img1.size(-3)
    w = _ssim_window(ch, img1.device, window_size).type_as(img1)
    pad = window_size // 2
    conv = lambda t: F.conv2d(t, w, padding=pad, groups=ch)
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(img1 * img1) - mu1_sq, conv(img2 * img2) - mu2_sq, conv(img1 * img2) - mu12
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    return ((2 * mu12 + c1) * (2 * s12 + c2)) / ((mu1_sq + mu2_sq + c1) * (s1 + s2 + c2))


def _render_pair(params, frame, render, fused, camera_grad, max_rendered=None, gaussians_grad=None):
    """The RGB and depth/silhouette renders of `frame` -> (image, depth_sil, radii, means2D of the RGB render).  The
    camera pose gets gradient iff `camera_grad`.  `gaussians_grad` (default: not `camera_grad`) decides whether the
    Gaussians get gradient on the torch glue path (transform_to_frame's flag); both together give both gradients
    from one backward (the reference's do_ba=True).  The fused path's kernel (csrc/prepare.cu) gives gradient to
    whichever Gaussian tensors require it, so a caller that wants only the pose passes detached Gaussian tensors, as
    tracking does.  fused: one kernel builds both rendervars
    (csrc/prepare.cu), and the product rasterizer blends both colour sets in one pass (N1), with a fixed instance
    capacity if `max_rendered`; otherwise the PyTorch glue and two `render` calls.  Both render at frame["pose"]
    (w2c, normalised quaternion) if given, else at the frame's pose in params.  The RGB render is corrected by the
    frame's exposure (`frame_exposure`) when it has one: train_ops.exposure when fused, its torch statement otherwise."""
    if fused:
        rv_rgb, rv_depth = fused_rendervars(params, frame["id"], frame["w2c"], camera_grad, pose=frame.get("pose"))
    else:
        gaussians_grad = (not camera_grad) if gaussians_grad is None else gaussians_grad
        tg = transform_to_frame(params, frame["id"], gaussians_grad=gaussians_grad, camera_grad=camera_grad,
                                pose=frame.get("pose"))
        rv_rgb, rv_depth = rgb_rendervar(params, tg), depth_sil_rendervar(params, frame["w2c"], tg)
    if fused and render is default_render:
        im, depth_sil, radius, _ = GaussianRasterizer(raster_settings=frame["cam"], max_rendered=max_rendered).forward_fused(
            means3D=rv_rgb["means3D"], means2D=rv_rgb["means2D"], opacities=rv_rgb["opacities"],
            colors_precomp=rv_rgb["colors_precomp"], colors_extra=rv_depth["colors_precomp"],
            scales=rv_rgb["scales"], rotations=rv_rgb["rotations"])
    else:
        im, radius, _ = render(frame["cam"], **rv_rgb)
        depth_sil, _, _ = render(frame["cam"], **rv_depth)
    ab = frame_exposure(params, frame)
    if ab is not None:
        from .train_ops import exposure, exposure_torch
        im = exposure(im, ab) if fused else exposure_torch(im, ab)
    return im, depth_sil, radius, rv_rgb["means2D"]


def frame_exposure(params, frame):
    """The colour correction ab [6] (log-gains, biases; train_ops.exposure) of `frame`'s RGB render: frame["exposure"]
    when given, else column frame["id"] of params["cam_exposure"] [1,6,T] when the params hold one, else None (no
    correction)."""
    ab = frame.get("exposure")
    if ab is None and "cam_exposure" in params:
        ab = params["cam_exposure"][0, :, frame["id"]]
    return ab


def mapping_loss(params, frame, render, loss_weights=(0.5, 1.0), ignore_outlier_depth_loss=False, fused_loss=False,
                 max_rendered=None, keep=None, camera_grad=False):
    """SplaTAM get_loss(mapping=True): the Gaussians get gradient, and with `camera_grad` the keyframe's pose too
    (R/scripts/splatam.py:214-347 with tracking=False, mapping=True, do_ba=camera_grad, use_l1=True).
    frame: dict(im [3,H,W], depth [1,H,W], cam settings, w2c [4,4] first-frame w2c, id time index).
    render(settings, **rendervar) -> (image, radii, depth).  frame["dynamic"] (bool [H,W], run_slam's motion mask),
    when given, takes its pixels out of both terms."""
    dyn = frame.get("dynamic")
    kept = None if dyn is None else ~dyn
    im, depth_sil, radius, means2D = _render_pair(params, frame, render, fused_loss, camera_grad=camera_grad,
                                                  max_rendered=max_rendered, gaussians_grad=True)
    if keep is not None:       # the caller wants d loss / d means2D of the RGB render (densification statistic)
        means2D.retain_grad()
        keep["means2D"] = means2D
    if fused_loss and not ignore_outlier_depth_loss:
        from .train_ops import masked_l1        # validity-masked mean |gt - depth| in one kernel (+ one backward)
        l_depth, _ = masked_l1(depth_sil, frame["depth"], depth_mean=True, keep=kept)
    else:
        depth = depth_sil[0:1]
        uncertainty = (depth_sil[2:3] - depth ** 2).detach()
        mask = (frame["depth"] > 0) & (~torch.isnan(depth)) & (~torch.isnan(uncertainty))
        if ignore_outlier_depth_loss:
            err = torch.abs(frame["depth"] - depth) * (frame["depth"] > 0)
            mask = mask & (err < 10 * err.median())
        if kept is not None:
            mask = mask & kept
        mask = mask.detach()
        l_depth = torch.abs(frame["depth"] - depth)[mask].mean()
        if kept is not None:
            l_depth = torch.nan_to_num(l_depth, nan=0.0)
    if fused_loss:      # one forward + one backward kernel instead of 5 depthwise convs + autograd (train_ops.cu)
        from .train_ops import image_loss
        l_im = image_loss(im, frame["im"], 0.8, 0.2, keep=kept)
    elif kept is None:
        l_im = 0.8 * torch.abs(im - frame["im"]).mean() + 0.2 * (1.0 - calc_ssim(im, frame["im"]))
    else:             # boolean indexing: with every pixel kept, the same elements in the same order as the means above
        k3 = kept.expand_as(im)
        l_im = 0.8 * torch.abs(im - frame["im"])[k3].mean() + 0.2 * (1.0 - ssim_map(im, frame["im"])[k3].mean())
        l_im = torch.nan_to_num(l_im, nan=0.0)        # every pixel masked: the mean of nothing counts as zero
    return loss_weights[0] * l_im + loss_weights[1] * l_depth, radius


def tracking_loss(params, frame, render, sil_thres=0.99, loss_weights=(0.5, 1.0), fused=False, max_rendered=None,
                  keep=None, motion=None):
    """SplaTAM get_loss(tracking=True, use_sil_for_loss=True, use_l1=True): only the camera pose of frame
    `frame["id"]` gets gradient; L1 sums over pixels with silhouette > sil_thres and valid depth
    (R/scripts/splatam.py:220-224,254-288; weights R/configs/replica/splatam.py:65-68).  `keep`: a dict that receives
    the unweighted depth L1 sum as "depth" (the reference's losses['depth']).
    motion: None, or dict(cfg (dynamic.config), exclude (bool [H,W] buffer), refresh (bool, or a device bool [1])):
    where `refresh` holds, `exclude` is first replaced by dynamic | inconsistent of this render's motion masks
    (dynamic.masks); the loss then leaves out the `exclude` pixels."""
    im, depth_sil, radius, _ = _render_pair(params, frame, render, fused, camera_grad=True, max_rendered=max_rendered)
    kept = None
    if motion is not None:
        from . import dynamic
        refresh = motion["refresh"]
        if isinstance(refresh, torch.Tensor) or refresh:
            dyn, inc, _ = dynamic.masks(depth_sil.detach(), frame["depth"], motion["cfg"], sil_thres, fused)
            new = dyn | inc
            motion["exclude"].copy_(torch.where(refresh, new, motion["exclude"]) if isinstance(refresh, torch.Tensor)
                                    else new)
        kept = ~motion["exclude"]
    if fused:
        from .train_ops import masked_l1
        l_depth, l_im = masked_l1(depth_sil, frame["depth"], im, frame["im"], sil_thres=sil_thres, use_sil=True,
                                  depth_mean=False, keep=kept)
    else:
        depth, sil = depth_sil[0:1], depth_sil[1]
        uncertainty = (depth_sil[2:3] - depth ** 2).detach()
        mask = (frame["depth"] > 0) & (~torch.isnan(depth)) & (~torch.isnan(uncertainty)) & (sil > sil_thres)
        if kept is not None:
            mask = mask & kept
        mask = mask.detach()
        # boolean indexing, as the reference: a NaN depth under a cleared mask bit must not reach the sum
        l_depth = torch.abs(frame["depth"] - depth)[mask].sum()
        l_im = torch.abs(frame["im"] - im)[torch.tile(mask, (3, 1, 1))].sum()
    if keep is not None:
        keep["depth"] = l_depth
    return loss_weights[0] * l_im + loss_weights[1] * l_depth, radius


def track_frame(params, frame, render=None, num_iters=40, lr_rot=0.0004, lr_trans=0.002, fused=None, graph=None,
                depth_loss_thres=None, lr_exposure=None, dynamic=None):
    """SplaTAM's tracking inner loop for one frame (R/scripts/splatam.py:676-744): Adam on the frame's camera
    quaternion and translation only, keeping the best-loss pose.  `params` holds detached Gaussian tensors and
    cam_unnorm_rots [1,4,T] / cam_trans [1,3,T] leaf tensors.  Returns the list of per-iteration losses.
    depth_loss_thres: the reference's use_depth_loss_thres rule (splatam.py:727-738): when the unweighted depth L1 sum
    of iteration `num_iters` (evaluated before its Adam step) is not below it, `num_iters` more iterations run once,
    with the same Adam state and best-pose record; the list then has 2 * num_iters entries.
    graph: the iteration -- loss forward + backward over the sync-free rasterizer, the Adam step and the best-pose
    bookkeeping, all on the device -- is captured once and replayed, so a frame costs one host synchronisation instead of
    one per iteration (`_TrackingGraph`); None = re-use a cached graph, build one only for loops of >= 100 iterations.
    lr_exposure: None, or (lr_log_gain, lr_bias): column t of params["cam_exposure"] [1,6,T] (the frame's colour
    correction, `frame_exposure`) is optimised with the pose, its log-gains and biases as two more Adam groups of these
    rates, and the best-loss record keeps it together with the pose.
    dynamic: None, or a dynamic.config dict: at iterations i % refresh_every == 0 the frame's motion mask is recomputed
    from that iteration's render, and the loss leaves out its pixels (tracking_loss's `motion`)."""
    render = default_render if render is None else render
    if fused is None:
        fused = params["means3D"].is_cuda and render is default_render
    can_graph = bool(fused) and params["means3D"].is_cuda and render is default_render
    if can_graph and graph is not False:
        # default policy: always re-use a cached graph; BUILD one only where it pays -- long loops (TUM: 200 iterations
        # per frame) or on request (graph=True: tracking-only runs over a map that stays put).  Building costs about as
        # much as ~40 eager iterations (capacity probe, warm-up, capture into a fresh memory pool).
        out = _track_frame_graphed(params, frame, num_iters, lr_rot, lr_trans, build=(graph is True or num_iters >= 100),
                                   depth_loss_thres=depth_loss_thres, lr_exposure=lr_exposure, dynamic=dynamic)
        if out is not None:
            return out              # None: no graph, or the instance capacity overflowed mid-frame -> run eagerly
    rots, trans = params["cam_unnorm_rots"], params["cam_trans"]
    rots.requires_grad_(True); trans.requires_grad_(True)
    groups = [{"params": [rots], "lr": lr_rot}, {"params": [trans], "lr": lr_trans}]
    t = frame["id"]
    if lr_exposure is not None:         # the column as two [1,3] leaves: log-gains and biases step at their own rates
        col = params["cam_exposure"][..., t].detach()
        gain, bias = col[:, :3].clone().requires_grad_(True), col[:, 3:].clone().requires_grad_(True)
        groups += [{"params": [gain], "lr": lr_exposure[0]}, {"params": [bias], "lr": lr_exposure[1]}]
    opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    best, best_rot, best_tran, best_ab, losses = None, None, None, None, []
    keep = None if depth_loss_thres is None else {}
    motion = None
    if dynamic is not None:
        motion = dict(cfg=dynamic, exclude=torch.zeros(frame["depth"].shape[-2:], dtype=torch.bool,
                                                        device=frame["depth"].device))
    total = num_iters
    while len(losses) < total:
        opt.zero_grad(set_to_none=True)
        fr = frame if lr_exposure is None else dict(frame, exposure=torch.cat([gain, bias], 1).reshape(6))
        if motion is not None:
            motion["refresh"] = len(losses) % dynamic["refresh_every"] == 0
        loss, _ = tracking_loss(params, fr, render, fused=fused, keep=keep, motion=motion)
        loss.backward()
        opt.step()
        with torch.no_grad():
            # as the reference (splatam.py:703-712): the candidate is the pose AFTER the step, ranked by the loss that
            # was evaluated before it
            lv = float(loss)
            if best is None or lv < best:
                best, best_rot, best_tran = lv, rots[..., t].detach().clone(), trans[..., t].detach().clone()
                if lr_exposure is not None:
                    best_ab = torch.cat([gain, bias], 1).detach().clone()
        losses.append(lv)
        if keep is not None and len(losses) == num_iters and not float(keep["depth"].detach()) < depth_loss_thres:
            total = 2 * num_iters
    with torch.no_grad():
        rots[..., t] = best_rot
        trans[..., t] = best_tran
        if lr_exposure is not None:
            params["cam_exposure"][..., t] = best_ab
    return losses


class _CapturedStep:
    """One step over the sync-free rasterizer, captured into a CUDA graph on a side stream and replayed: its instance
    capacity `cap`, the static frame buffers it renders (`frame`: id, cam, w2c, im, depth; `load` refills them) and
    the overflow flag of its render.  `cap` is `capacity`, or slack x the largest instance count of the `probe`
    frames at their poses in `params`, plus 4096."""

    def __init__(self, params, frame, probe, slack, capacity=None):
        self.dev = params["means3D"].device
        if capacity is None:
            worst = 0
            for fr in probe:
                with torch.no_grad():
                    rgb, _ = fused_rendervars(params, fr["id"], fr["w2c"], camera_grad=False)
                worst = max(worst, GaussianRasterizer(fr["cam"]).num_rendered(rgb["means3D"], rgb["opacities"],
                                                                              rgb["scales"], rgb["rotations"]))
            capacity = int(worst * slack) + 4096
        self.cap = int(capacity)
        self.frame = dict(id=frame["id"], cam=frame["cam"], w2c=frame["w2c"].clone(), im=frame["im"].clone(),
                          depth=frame["depth"].clone())
        if frame.get("dynamic") is not None:      # the keyframes' motion masks (run_slam's `dynamic`)
            self.frame["dynamic"] = frame["dynamic"].clone()
        self.side = torch.cuda.Stream(self.dev)
        self.side.wait_stream(torch.cuda.current_stream(self.dev))      # for state a caller creates on it before capture

    def load(self, frame):
        for k in ("im", "depth", "w2c", "dynamic"):
            if k in self.frame:
                self.frame[k].copy_(frame[k], non_blocking=True)

    def overflow(self):
        """int32 [1] device view of the overflow flag of the latest sync-free render: inside the step, its own."""
        return GaussianRasterizer.last_state(self.dev).header()[2:3]

    def capture(self, body):
        """Runs body() three times (warm-up: kernels load, lazily created state such as capturable Adam's exists),
        then captures it into `graph`, all on the side stream after the work enqueued so far on the current one.
        capture_begin / capture_end directly: the torch.cuda.graph context manager also runs gc.collect() and
        torch.cuda.empty_cache(), which costs tens of milliseconds and throws the allocator's cached blocks away."""
        self.side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.side):
            for _ in range(3):
                body()
            self.graph = torch.cuda.CUDAGraph()
            self.graph.capture_begin()
            try:
                body()
            finally:
                self.graph.capture_end()
        torch.cuda.current_stream(self.dev).wait_stream(self.side)


class _TrackingGraph:
    """One captured tracking iteration (loss forward + backward over the sync-free rasterizer, capturable Adam step,
    best-pose bookkeeping, all on the device) bound to ONE map (the Gaussian tensors' storage), camera and iteration
    count -- not to a pose column: the pose travels through two small leaf tensors.  Re-used frame after frame while
    the map tensors stay the same objects (tracking-only runs; SLAM phases without map growth): a frame then costs two
    small image copies, `num_iters` graph launches and one host synchronisation.

    With `depth_loss_thres` the graph records the depth L1 sum too and a frame replays 2 * num_iters iterations; the
    decision of track_frame's rule is taken on the device after iteration num_iters, and when the frame stops there
    the remaining replays run gated: they record no loss, update no best pose and raise no overflow.  The frame
    still costs one host synchronisation; the gated replays cost GPU time.

    With `lr_exposure` the frame's colour correction travels the same way, as two [1,3] leaves (log-gains, biases)
    with two more capturable Adam groups and a best-loss record of their own."""

    def __init__(self, params, frame, num_iters, lr_rot, lr_trans, depth_loss_thres=None, lr_exposure=None,
                 dynamic=None):
        t = frame["id"]
        rots, trans = params["cam_unnorm_rots"], params["cam_trans"]
        self.gp = gp = {k: params[k].detach() for k in GAUSSIAN_KEYS}        # keeps the storage the graph reads alive
        self.rule = rule = depth_loss_thres is not None
        self.replays = 2 * num_iters if rule else num_iters
        self.step = step = _CapturedStep(params, frame, [frame], slack=1.5)     # sized at the starting pose
        dev = step.dev
        with torch.cuda.stream(step.side):
            self.q = rots[..., t].detach().clone().requires_grad_(True)      # [1,4], [1,3]: leaves born on the capture stream
            self.tr = trans[..., t].detach().clone().requires_grad_(True)
            q, tr = self.q, self.tr
            q.grad, tr.grad = torch.zeros_like(q), torch.zeros_like(tr)
            leaves, groups = [q, tr], [{"params": [q], "lr": lr_rot}, {"params": [tr], "lr": lr_trans}]
            self.expo = expo = lr_exposure is not None
            if expo:
                col = params["cam_exposure"][..., t].detach()
                self.gain = col[:, :3].clone().requires_grad_(True)
                self.bias = col[:, 3:].clone().requires_grad_(True)
                self.gain.grad, self.bias.grad = torch.zeros_like(self.gain), torch.zeros_like(self.bias)
                leaves += [self.gain, self.bias]
                groups += [{"params": [self.gain], "lr": lr_exposure[0]}, {"params": [self.bias], "lr": lr_exposure[1]}]
                self.best_ab = col.clone()
            self.opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15, capturable=True)
            self.best_loss = torch.full((), float("inf"), device=dev)
            self.best_q, self.best_tr = q.detach().clone(), tr.detach().clone()
            self.hist = torch.zeros(self.replays, device=dev)
            self.it = torch.zeros(1, dtype=torch.long, device=dev)
            self.bad_any = torch.zeros(1, device=dev)
            self.live = torch.ones(1, dtype=torch.bool, device=dev)   # rule only: this replay is a real iteration
            self.motion = None
            if dynamic is not None:       # the mask is computed every replay and kept where it % refresh_every == 0
                self.motion = dict(cfg=dynamic, exclude=torch.zeros(frame["depth"].shape[-2:], dtype=torch.bool,
                                                                    device=dev))

        def body():
            for leaf in leaves:
                leaf.grad.zero_()
            keep = {} if rule else None
            fr = dict(step.frame, pose=camera_w2c(q, tr))
            if expo:
                fr["exposure"] = torch.cat([self.gain, self.bias], 1).reshape(6)
            if self.motion is not None:
                self.motion["refresh"] = self.it % self.motion["cfg"]["refresh_every"] == 0
            loss, _ = tracking_loss(gp, fr, default_render, fused=True, max_rendered=step.cap, keep=keep,
                                    motion=self.motion)
            loss.backward()
            lossd = loss.detach().reshape(1)
            bad = (step.overflow() != 0) | ~torch.isfinite(lossd)
            for leaf in leaves:
                leaf.grad.copy_(torch.where(bad, torch.zeros_like(leaf.grad), leaf.grad))
            self.bad_any.add_((bad & self.live).float() if rule else bad.float())
            self.opt.step()
            # the reference's rule (splatam.py:703-712): candidate = pose AFTER the step, ranked by the loss evaluated
            # before it; the first strictly smaller loss wins
            better = (lossd < self.best_loss) & ~bad
            if rule:
                better = better & self.live
            self.best_loss.copy_(torch.where(better, lossd, self.best_loss.reshape(1)).reshape(()))
            self.best_q.copy_(torch.where(better, q.detach(), self.best_q))
            self.best_tr.copy_(torch.where(better, tr.detach(), self.best_tr))
            if expo:
                self.best_ab.copy_(torch.where(better, torch.cat([self.gain, self.bias], 1).detach(), self.best_ab))
            self.hist.scatter_(0, self.it, lossd)
            if rule:
                # a gated replay overwrites slot `it` (the first unused one, num_iters) and does not advance `it`
                self.it.add_(self.live.long())
                # after the num_iters-th real iteration: continue only if its depth sum is not below the threshold
                stop = self.live & (self.it == num_iters) & (keep["depth"].detach().reshape(1) < depth_loss_thres)
                self.live.copy_(self.live & ~stop)
            else:
                self.it.add_(1)
        step.capture(body)              # the warm-up's optimizer steps and records are undone by reset()

    def reset(self, params, frame):
        """Loads a frame: images, starting pose, fresh optimizer state (the reference builds a new Adam per frame,
        splatam.py:680), empty best-pose record."""
        t = frame["id"]
        with torch.no_grad():
            self.step.load(frame)
            self.q.copy_(params["cam_unnorm_rots"][..., t]); self.tr.copy_(params["cam_trans"][..., t])
            if self.expo:
                col = params["cam_exposure"][..., t]
                self.gain.copy_(col[:, :3]); self.bias.copy_(col[:, 3:]); self.best_ab.copy_(col)
            for st in self.opt.state.values():
                st["exp_avg"].zero_(); st["exp_avg_sq"].zero_(); st["step"].zero_()
            self.best_loss.fill_(float("inf")); self.best_q.copy_(self.q); self.best_tr.copy_(self.tr)
            self.hist.zero_(); self.it.zero_(); self.bad_any.zero_(); self.live.fill_(True)

    def run(self, params, frame):
        side, cur = self.step.side, torch.cuda.current_stream(self.step.dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self.reset(params, frame)
            for _ in range(self.replays):
                self.step.graph.replay()
        cur.wait_stream(side)
        if float(self.bad_any) != 0.0:                                   # the one host synchronisation of the frame
            return None
        with torch.no_grad():
            params["cam_unnorm_rots"][..., frame["id"]] = self.best_q
            params["cam_trans"][..., frame["id"]] = self.best_tr
            if self.expo:
                params["cam_exposure"][..., frame["id"]] = self.best_ab
        hist = self.hist.tolist()
        return hist[:int(self.it)] if self.rule else hist


_TRACK_GRAPHS = {}


def _tracking_key(params, frame, num_iters, lr_rot, lr_trans, depth_loss_thres, lr_exposure=None, dynamic=None):
    """What a captured tracking iteration is bound to: the storage (pointer and shape) of each Gaussian tensor it
    reads, the camera, the image shape, the iteration count, the learning rates (the exposure rates included), the
    depth-loss rule and the motion-mask options."""
    return (tuple((params[k].data_ptr(), tuple(params[k].shape)) for k in GAUSSIAN_KEYS), id(frame["cam"]),
            tuple(frame["im"].shape), num_iters, lr_rot, lr_trans, depth_loss_thres,
            None if lr_exposure is None else tuple(float(r) for r in lr_exposure),
            None if dynamic is None else tuple(sorted(dynamic.items())))


def _track_frame_graphed(params, frame, num_iters, lr_rot, lr_trans, build=True, depth_loss_thres=None,
                         lr_exposure=None, dynamic=None):
    """Graph-replayed tracking of one frame, or None when no graph is available / an iteration overflowed the instance
    capacity (the caller then runs the frame eagerly).  Graphs are cached per `_tracking_key`; `build` creates one on
    a miss (worth it for long loops or when the map stays put)."""
    key = _tracking_key(params, frame, num_iters, lr_rot, lr_trans, depth_loss_thres, lr_exposure, dynamic)
    tg = _TRACK_GRAPHS.get(key)
    if tg is None:
        if not build:
            return None
        if len(_TRACK_GRAPHS) >= 2:
            _TRACK_GRAPHS.clear()
        tg = _TRACK_GRAPHS[key] = _TrackingGraph(params, frame, num_iters, lr_rot, lr_trans,
                                                 depth_loss_thres=depth_loss_thres, lr_exposure=lr_exposure,
                                                 dynamic=dynamic)
    return tg.run(params, frame)


class FlatGaussians:
    """The five Gaussian parameter tensors as views into ONE flat fp32 buffer, their gradients as
    views into ONE flat gradient bucket of the same layout -- the packed send buffer of the
    all-reduce (48-56 B per Gaussian).  `pose_numel` > 0 appends the pose-gradient table of keyframe-pose refinement
    ([7, T]: the 4 quaternion rows, then the 3 translation rows) to the bucket."""

    def __init__(self, tensors, pose_numel=0):
        self.shapes = {k: tuple(tensors[k].shape) for k in GAUSSIAN_KEYS}
        n = sum(math.prod(s) for s in self.shapes.values())
        dev = tensors["means3D"].device
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        # ONE all-reduce bucket: [per-Gaussian gradients (n) | per-Gaussian "seen" flags as 0/1 floats (P) | loss (1) |
        # capacity-overflow flag of the sync-free rasterizer (1): non-zero on ANY rank => every rank skips the update |
        # pose-gradient table (pose_numel, refinement only)]
        P_ = tensors["means3D"].shape[0]
        self.bucket = torch.zeros(n + P_ + 2 + pose_numel, dtype=torch.float32, device=dev)
        self.flat_grad = self.bucket[:n]
        self.seen_f = self.bucket[n:n + P_]
        self.loss_slot = self.bucket[n + P_:n + P_ + 1]
        self.overflow_slot = self.bucket[n + P_ + 1:n + P_ + 2]
        self.pose_grad = self.bucket[n + P_ + 2:]
        self.params, grads = self.views(self.flat), self.views(self.flat_grad)
        for k, p in self.params.items():
            p.copy_(tensors[k].detach().reshape(self.shapes[k]))
            p.requires_grad_(True)
            p.grad = grads[k]                   # autograd accumulates in place

    def views(self, buf):
        """{key: view of the key's segment of `buf`}, for any flat buffer of this layout (parameters, gradients, Adam
        moments)."""
        out, off = {}, 0
        for k in GAUSSIAN_KEYS:
            m = math.prod(self.shapes[k])
            out[k] = buf[off:off + m].view(self.shapes[k])
            off += m
        return out

    def zero_grad(self):
        self.bucket.zero_()


def densify_due(iter, densify_dict):
    """Whether `densify` edits the map at iteration `iter` (R/utils/slam_external.py:205): it then replaces every
    Gaussian tensor, so in the reference's loops the optimizer step that follows finds no gradient."""
    return (densify_dict["start_after"] <= iter <= densify_dict["stop_after"]
            and iter % densify_dict["densify_every"] == 0)


def default_render(settings, **rendervar):
    return GaussianRasterizer(raster_settings=settings)(**rendervar)


CAM_KEYS = ("cam_unnorm_rots", "cam_trans")


class ShardedMapper:
    """Data-parallel mapping over keyframes.  `lrs` follow R/configs/replica/splatam.py:92-100.

    Keyframe-pose refinement (the reference's get_loss(mapping=True, do_ba=True)) is on iff the `lrs` of
    cam_unnorm_rots or cam_trans is non-zero.  The mapper then owns the cameras: `cam` holds two views of one flat
    [4T | 3T] buffer, and camera tensors a caller puts into `cam` (tracking, `sync_camera`) are copied into it before
    the next step.  Each step's render gives gradient to the Gaussians and to its keyframe's pose; the [7, T] pose
    gradient (zero outside the keyframe's column) travels in the all-reduce bucket, and an Adam over the whole two
    tensors (torch.optim.Adam on the torch path, FusedAdam on the fused one) steps them on every step.  Its moments
    reset with `reset_optimizer` and survive map edits.  At zero camera rates nothing of this exists.

    `cam` may also hold `cam_exposure` [1,6,T], each frame's colour correction (train_ops.exposure): every step's RGB
    render is corrected by its keyframe's column (which mapping does not step), and `add_new_gaussians` takes the
    frame's colours mapped back to frame 0's appearance.  Without it nothing of this runs."""

    DEFAULT_LRS = dict(means3D=0.0001, rgb_colors=0.0025, unnorm_rotations=0.001, logit_opacities=0.05,
                       log_scales=0.001)

    def __init__(self, gaussians, cam_unnorm_rots, cam_trans, lrs=None, render=default_render, group=None, seed=0,
                 fused=None, track_means2D=False, timestep=None, cam_exposure=None):
        """track_means2D: keep d loss / d means2D of every eager step's RGB render and which Gaussians it saw (the
        statistic of `densify`).  timestep: the frame that created each Gaussian ([P], e.g. from a checkpoint); default
        zeros, as the reference starts its initial map (R/scripts/splatam.py:155)."""
        import torch.distributed as dist
        self.dist = dist if (dist.is_available() and dist.is_initialized()) else None
        self.group = group
        self.rank = self.dist.get_rank(group) if self.dist else 0
        self.world = self.dist.get_world_size(group) if self.dist else 1
        lrs = dict(self.DEFAULT_LRS, **(lrs or {}))
        self.lrs = lrs
        self.refine_poses = any(float(lrs.get(k, 0.0)) != 0.0 for k in CAM_KEYS)
        T = cam_trans.shape[-1]
        self.g = FlatGaussians(gaussians, pose_numel=7 * T if self.refine_poses else 0)
        P, dev = self.g.shapes["means3D"][0], self.g.flat.device
        # per-Gaussian creation frame: kept beside the flat buffer, outside the gradient / Adam / all-reduce layout, and
        # edited with the same masks as the parameters, so every replica holds the same one
        if timestep is None:
            self.timestep = torch.zeros(P, dtype=torch.float32, device=dev)
        else:
            self.timestep = torch.as_tensor(timestep).detach().to(dev, torch.float32).reshape(-1).clone()
            if self.timestep.shape[0] != P:
                raise ValueError("timestep has %d entries for a map of %d Gaussians" % (self.timestep.shape[0], P))
        self.cam = dict(cam_unnorm_rots=cam_unnorm_rots.detach(), cam_trans=cam_trans.detach())
        if cam_exposure is not None:
            self.cam["cam_exposure"] = cam_exposure.detach()
        # fused = hand-written Adam over the flat buffer + fused L1/SSIM loss (CUDA only); the torch path is
        # the reference formulation (R/scripts/splatam.py:160-166) and the one the CPU/gloo test exercises
        self.fused = self.g.flat.is_cuda if fused is None else bool(fused)
        self._make_optimizer()
        if self.refine_poses:
            self._cam_flat = torch.zeros(7 * T, dtype=torch.float32, device=dev)
            self._cam_views = {"cam_unnorm_rots": self._cam_flat[:4 * T].view(1, 4, T),
                               "cam_trans": self._cam_flat[4 * T:].view(1, 3, T)}
            for v in self._cam_views.values():
                v.requires_grad_(True)
            self._bind_pose_grad()
            self._bind_cameras()
            self._make_cam_optimizer()
        self.render = render
        self.gen = torch.Generator().manual_seed(seed)   # shared seed -> identical schedule on every rank
        self.step_idx = 0
        self.track_means2D = bool(track_means2D)
        self.last_means2D_grad = self.last_seen_local = None
        self._dens = None                   # densification statistic: dict(accum, denom) per Gaussian
        self._dev_gen = None                # shared-seed device generator of the split samples (world > 1)
        self._graph = None                  # CUDA-graph mode: the captured step (enable_graph)
        self.overflow_events = 0

    def params(self):
        return dict(self.g.params, **self.cam)

    # ---- what stays single-GPU (SURVEY.md 8(e)): rank `src` does it, the result is broadcast ---------------------
    def sync_camera(self, src=0):
        """Tracking runs on one rank (its backward uses float atomics, so two ranks would not end bit-identical);
        the estimated poses are broadcast so every replica maps with the same cameras."""
        if self.dist and self.world > 1:
            for k in [k for k in CAM_KEYS + ("cam_exposure",) if k in self.cam]:
                t = self.cam[k].detach().clone().contiguous()
                self.dist.broadcast(t, src=src, group=self.group)
                self.cam[k] = t
        return self.cam

    def broadcast_frame(self, frame, src=0):
        """A keyframe's images are loaded by one rank and broadcast once when the keyframe is created (13 MB at
        1200x680); `frame` must hold tensors of the right shape on every rank (contents are overwritten)."""
        if self.dist and self.world > 1:
            for k in ("im", "depth", "w2c"):
                t = frame[k].contiguous()
                self.dist.broadcast(t, src=src, group=self.group)
                frame[k] = t
        return frame

    # ---- map maintenance (prune / grow); every rank applies the same deterministic edit --------------------------
    def _make_optimizer(self, m=None, v=None, t=0):
        """Adam over the current map whose two moments live in flat buffers of the parameter layout (zero by default)
        and which has taken `t` steps."""
        self.exp_avg = torch.zeros_like(self.g.flat) if m is None else m
        self.exp_avg_sq = torch.zeros_like(self.g.flat) if v is None else v
        if self.fused:
            from .train_ops import FusedAdam
            sizes = [math.prod(self.g.shapes[k]) for k in GAUSSIAN_KEYS]
            self.opt = FusedAdam(self.g.flat, self.g.flat_grad, sizes, [self.lrs[k] for k in GAUSSIAN_KEYS], eps=1e-15,
                                 exp_avg=self.exp_avg, exp_avg_sq=self.exp_avg_sq, step=t)
        else:
            self.opt = torch.optim.Adam([{"params": [self.g.params[k]], "name": k, "lr": self.lrs[k]}
                                         for k in GAUSSIAN_KEYS], lr=0.0, eps=1e-15)
            for k, (mk, vk) in self.moments().items():    # the state torch.optim.Adam would create, on our buffers
                self.opt.state[self.g.params[k]] = dict(step=torch.tensor(float(t)), exp_avg=mk, exp_avg_sq=vk)

    def moments(self):
        """{key: (exp_avg, exp_avg_sq)}: the Adam moments of each parameter tensor, for either optimizer."""
        m, v = self.g.views(self.exp_avg), self.g.views(self.exp_avg_sq)
        return {k: (m[k], v[k]) for k in GAUSSIAN_KEYS}

    def _adam_steps(self):
        if self.fused:
            return self.opt.applied_steps()[0]
        return int(self.opt.state[self.g.params["means3D"]]["step"])

    # ---- keyframe-pose refinement ---------------------------------------------------------------------------------
    def _bind_pose_grad(self):
        """The camera views' gradients are the bucket's pose table (autograd accumulates into it in place)."""
        T = self._cam_flat.numel() // 7
        self._cam_views["cam_unnorm_rots"].grad = self.g.pose_grad[:4 * T].view(1, 4, T)
        self._cam_views["cam_trans"].grad = self.g.pose_grad[4 * T:].view(1, 3, T)

    def _bind_cameras(self):
        """Copies camera tensors a caller put into `cam` into the mapper's buffer, whose views `cam` holds again."""
        if all(self.cam[k] is self._cam_views[k] for k in CAM_KEYS):
            return
        T = self._cam_flat.numel() // 7
        with torch.no_grad():
            self._cam_flat[:4 * T].copy_(self.cam["cam_unnorm_rots"].reshape(-1))
            self._cam_flat[4 * T:].copy_(self.cam["cam_trans"].reshape(-1))
        self.cam = dict(self.cam, **self._cam_views)

    def _make_cam_optimizer(self):
        """Fresh Adam over the two whole camera tensors (initialize_optimizer(tracking=False), R/scripts/splatam.py:
        160-166): the fused path steps the flat buffer with FusedAdam, the torch path uses torch.optim.Adam groups."""
        lr = [self.lrs.get(k, 0.0) for k in CAM_KEYS]
        if self.fused:
            from .train_ops import FusedAdam
            T = self._cam_flat.numel() // 7
            self.cam_opt = FusedAdam(self._cam_flat, self.g.pose_grad, [4 * T, 3 * T], lr, eps=1e-15)
        else:
            self.cam_opt = torch.optim.Adam([{"params": [self._cam_views[k]], "name": k, "lr": r}
                                             for k, r in zip(CAM_KEYS, lr)], lr=0.0, eps=1e-15)

    def _cam_step(self, guard=None):
        """Adam step of the cameras; `guard`: the overflow slot of a graph step (a no-op when it is non-zero)."""
        if self.fused:
            self.cam_opt.flat_grad = self.g.pose_grad
            if guard is None:
                self.cam_opt.step()
            else:
                self.cam_opt.step_guarded(guard)
            # the kernel writes through a raw pointer: bump the version the pose cache (fused_pose_cached) keys on
            torch.autograd.graph.increment_version(self._cam_flat)
        else:
            self.cam_opt.step()

    def set_lr(self, key, lr):
        """Learning rate of parameter tensor `key` from the next Adam step on, and for the optimizers a map edit
        rebuilds (update_learning_rate, R/utils/gs_external.py:260-266).  A camera key needs a mapper built with
        refinement on (a non-zero camera rate), or a zero rate."""
        if key in CAM_KEYS:
            if not self.refine_poses:
                if float(lr) != 0.0:
                    raise ValueError("keyframe-pose refinement is off: build the mapper with a non-zero %s rate" % key)
                return
            self.lrs[key] = float(lr)
            i = CAM_KEYS.index(key)
            if self.fused:
                self.cam_opt.set_lr(i, lr)
            else:
                self.cam_opt.param_groups[i]["lr"] = float(lr)
            return
        self.lrs[key] = float(lr)
        i = GAUSSIAN_KEYS.index(key)
        if self.fused:
            self.opt.set_lr(i, lr)
        else:
            self.opt.param_groups[i]["lr"] = float(lr)

    def reset_optimizer(self):
        """Fresh Adam state, as the reference re-creates its optimizer at the start of every frame's mapping
        phase (R/scripts/splatam.py:822), the cameras' included."""
        self._make_optimizer()
        if self.refine_poses:
            self._make_cam_optimizer()

    def _widths(self):
        return [self.g.shapes[k][1] if len(self.g.shapes[k]) > 1 else 1 for k in GAUSSIAN_KEYS]

    def _rebuild(self, flat, P_new, m, v, t):
        """The map becomes `P_new` rows: parameters `flat` and Adam moments `m`, `v` (flat buffers of the packed layout)
        after `t` Adam steps."""
        tensors, off = {}, 0
        for k, w in zip(GAUSSIAN_KEYS, self._widths()):
            tensors[k] = flat[off:off + w * P_new].view(P_new, w)
            off += w * P_new
        old_pose_grad = self.g.pose_grad
        self.g = FlatGaussians(tensors, pose_numel=old_pose_grad.numel())
        if self.refine_poses:       # map edits leave the cameras alone (R/utils/slam_external.py:141): keep the gradient
            self.g.pose_grad.copy_(old_pose_grad)
            self._bind_pose_grad()
        self._make_optimizer(m, v, t)
        self._graph = None                      # shapes changed: a captured graph is stale

    def remove_points(self, to_remove):
        """Drop the rows where `to_remove` is set from the parameters, both Adam moments and `timestep`
        (remove_points, R/utils/slam_external.py:144-167).  Returns the number of Gaussians kept."""
        P = self.g.shapes["means3D"][0]
        keep = ~to_remove.reshape(-1).bool()
        if self.fused:              # stream compaction kernels (csrc/map_ops.cu)
            from . import map_ops
            m8, dst, P_new = map_ops.compact_plan(keep)
            compact = lambda buf: map_ops.compact_flat(buf, P, self._widths(), m8, dst, P_new)
            compact_ts = lambda ts: map_ops.compact_flat(ts, P, [1], m8, dst, P_new)
        else:
            P_new = int(keep.sum())
            compact = lambda buf: torch.cat([x[keep].reshape(-1) for x in self.g.views(buf).values()])
            compact_ts = lambda ts: ts[keep]
        if P_new == P:
            return P
        self._rebuild(compact(self.g.flat), P_new, compact(self.exp_avg), compact(self.exp_avg_sq), self._adam_steps())
        self.timestep = compact_ts(self.timestep.contiguous())
        return P_new

    def _reset_opacities(self):
        """Every opacity to 0.01 (inverse_sigmoid(0.01)), its Adam moments to zero (R/utils/slam_external.py:184-186)."""
        with torch.no_grad():
            self.g.params["logit_opacities"].fill_(math.log(0.01 / 0.99))
        for mom in self.moments()["logit_opacities"]:
            mom.zero_()

    def prune_gaussians(self, iter, prune_dict, scene_radius):
        """prune_gaussians of the reference (R/utils/slam_external.py:170-197): same schedule keys
        (start_after, stop_after, prune_every, removal_opacity_threshold, final_removal_opacity_threshold,
        remove_big_after, reset_opacities, reset_opacities_every).  Returns the Gaussian count afterwards."""
        P = self.g.shapes["means3D"][0]
        if iter > prune_dict["stop_after"]:
            return P
        if iter >= prune_dict["start_after"] and iter % prune_dict["prune_every"] == 0:
            thr = (prune_dict["final_removal_opacity_threshold"] if iter == prune_dict["stop_after"]
                   else prune_dict["removal_opacity_threshold"])
            big = 0.1 * float(scene_radius) if iter >= prune_dict["remove_big_after"] else None
            lo, ls = self.g.params["logit_opacities"].detach(), self.g.params["log_scales"].detach()
            if self.fused:
                from . import map_ops
                keep = map_ops.prune_mask(lo, ls, thr, big)
            else:
                remove = (torch.sigmoid(lo) < thr).squeeze(-1)
                if big is not None:
                    remove = remove | (torch.exp(ls).max(dim=1).values > big)
                keep = ~remove
            P = self.remove_points(~keep)
        if iter > 0 and iter % prune_dict["reset_opacities_every"] == 0 and prune_dict["reset_opacities"]:
            self._reset_opacities()
        return P

    def add_gaussians(self, new, timestep=0):
        """Append rows (dict of the five tensors) to the map; Adam moments of the new rows start at zero
        (cat_params_to_optimizer, R/utils/slam_external.py:121-141).  `timestep`: the new rows' creation frame, one
        value for all of them or one per row.  Returns the new Gaussian count."""
        P, n_new = self.g.shapes["means3D"][0], new["means3D"].shape[0]
        if n_new == 0:
            return P
        dev = self.g.flat.device
        ts = torch.as_tensor(timestep).detach().to(dev, torch.float32)
        ts = ts.expand(n_new) if ts.dim() == 0 else ts.reshape(-1)
        if ts.shape[0] != n_new:
            raise ValueError("timestep has %d entries for %d new Gaussians" % (ts.shape[0], n_new))

        def grown(buf, rows):
            return torch.cat([torch.cat([x, rows[k]], 0).reshape(-1) for k, x in self.g.views(buf).items()])
        zeros = {k: torch.zeros(n_new, w, device=dev) for k, w in zip(GAUSSIAN_KEYS, self._widths())}
        flat = grown(self.g.flat, {k: new[k].to(dev).float().reshape(n_new, -1) for k in GAUSSIAN_KEYS})
        self._rebuild(flat, P + n_new, grown(self.exp_avg, zeros), grown(self.exp_avg_sq, zeros), self._adam_steps())
        self.timestep = torch.cat([self.timestep, ts])
        return P + n_new

    def deform(self, table, flag):
        """Loop closure's map deformation (loop.deform_gaussians): every Gaussian's mean and quaternion move, in place
        in the flat buffer, by the correction table [T,12] row of its `timestep`; nothing moves if the device int32
        `flag` is 0.  The storage stays, so a captured mapping step and a cached tracking graph read the moved map at
        their next replay."""
        from . import loop
        p = self.g.params
        with torch.no_grad():
            loop.deform_gaussians(p["means3D"], p["unnorm_rotations"], self.timestep.contiguous(), table, flag)

    def add_new_gaussians(self, frame, time_idx, intrinsics, sil_thres, exclude=None):
        """add_new_gaussians of the reference (R/scripts/splatam.py:378-420): one depth/silhouette render of the
        current map at the frame's estimated pose, non-presence mask, back-projection of the selected pixels,
        append with `timestep` = time_idx (splatam.py:417-418).  CUDA only.  Returns the number of Gaussians added.
        exclude: a bool mask (the frame's motion mask, max-pooled to the frame's size when that differs) whose pixels
        grow nothing."""
        from . import map_ops
        p = self.params()
        with torch.no_grad():
            tg = transform_to_frame(p, time_idx, gaussians_grad=False, camera_grad=False)
            depth_sil, _, _ = self.render(frame["cam"], **depth_sil_rendervar(p, frame["w2c"], tg))
            curr_w2c, _ = pose_matrices(p, time_idx)
            if "cam_exposure" in p:         # the new Gaussians take the frame's colour in frame 0's appearance
                from .train_ops import exposure
                frame = dict(frame, im=exposure(frame["im"], p["cam_exposure"][0, :, time_idx], inverse=True))
        if exclude is not None:
            from .dynamic import footprint
            exclude = footprint(exclude, frame["depth"].shape[-2:])
        new, n = map_ops.new_gaussians_from_frame(depth_sil, frame, intrinsics, curr_w2c, sil_thres,
                                                  scale_dim=self._widths()[4], exclude=exclude)
        if n:
            self.add_gaussians(new, timestep=time_idx)
        return n

    # ---- CUDA-graph mode -----------------------------------------------------------------------------------
    def enable_graph(self, window, slack=1.3, capacity=None):
        """Capture loss forward + backward of one keyframe into a CUDA graph (sync-free rasterizer with a fixed
        instance capacity = slack x the largest num_rendered over `window`, or `capacity`).  Afterwards `step`
        copies the chosen keyframe into static buffers and replays the graph: ~6 launches per step instead of ~60,
        and no host synchronisation, so the step no longer depends on host speed.  Frames must share one camera.

        Safety: if the map moves or grows until a render needs more instances than the capacity, the rasterizer
        raises its device-side overflow flag and writes NaN images; the flag travels in the all-reduce bucket, the
        guarded Adam step (device-side step clock) is a no-op on every rank for that step, and `step` -- which
        polls the flag with a one-step lag, never blocking on the step in flight -- re-captures with a larger
        capacity.  An overflowed step therefore costs time, never correctness."""
        assert self.fused and self.g.flat.is_cuda and self.render is default_render
        # a geometry pass per probed frame sizes the capacity (an overflow later is safe: it skips the step and
        # re-captures, see the docstring)
        probe = window if len(window) <= 3 else [window[0], window[len(window) // 2], window[-1]]
        if self.refine_poses:
            self._bind_cameras()
        step = _CapturedStep(self.params(), window[0], probe, slack, capacity)
        step.frame["pose"] = tuple(t.clone() for t in fused_pose_cached(self.params(), window[0]["id"]))
        if "cam_exposure" in self.cam:        # static [6]: `step` loads the keyframe's column as it loads its pose
            step.frame["exposure"] = self.cam["cam_exposure"][0, :, window[0]["id"]].detach().clone()
        self._slack = slack
        self._polls = []                 # (event, pinned copy of the overflow slot) of steps in flight
        self._pin = [torch.empty(1, dtype=torch.float32, pin_memory=True) for _ in range(8)]
        refine = self.refine_poses
        if refine:
            # the keyframe's pose as two static leaves [1,4], [1,3] loaded from its column before each replay; the
            # backward leaves their gradient in static .grad buffers, scattered into column `col` of the pose table
            T = self._cam_flat.numel() // 7
            t0 = window[0]["id"]
            with torch.cuda.stream(step.side):
                q = self.cam["cam_unnorm_rots"][..., t0].detach().clone().requires_grad_(True)
                tr = self.cam["cam_trans"][..., t0].detach().clone().requires_grad_(True)
                q.grad, tr.grad = torch.zeros_like(q), torch.zeros_like(tr)
                col = torch.full((1,), int(t0), dtype=torch.long, device=step.dev)
            step.pose_leaves = (q, tr, col)

        def body():
            self.g.bucket.zero_()
            frame = step.frame
            if refine:
                q.grad.zero_(); tr.grad.zero_()
                frame = dict(step.frame, pose=camera_w2c(q, tr))
            loss, radius = mapping_loss(self.params(), frame, self.render, fused_loss=True, max_rendered=step.cap)
            loss.backward()
            if refine:
                self.g.pose_grad.view(7, T).index_copy_(1, col, torch.cat([q.grad, tr.grad], 1).reshape(7, 1))
            self.g.seen_f.copy_(radius > 0)
            self.g.loss_slot.copy_(loss.detach().reshape(1))
            self.g.overflow_slot.copy_(step.overflow())     # int32 0/1 -> float
        step.capture(body)
        self._graph = step
        return step.cap

    def check_capacity(self):
        """(num_rendered, overflowed) of the last graph replay; synchronises."""
        return GaussianRasterizer.last_counts(self.g.flat.device)

    def effective_steps(self):
        """(Adam steps applied, steps skipped because a render overflowed the instance capacity); synchronises."""
        return self.opt.applied_steps() if self.fused else (self.step_idx, 0)

    def poll_overflow(self, window, block=False):
        """Graph mode: looks at the overflow flags of COMPLETED earlier steps (one-step lag: never waits for the step in
        flight unless `block`); on overflow grows the capacity from the measured instance count and re-captures.
        Returns whether a step overflowed; False without a captured graph."""
        if self._graph is None:
            return False
        hit = False
        while self._polls and (block or len(self._polls) > 1 or self._polls[0][0].query()):
            ev, host = self._polls.pop(0)
            ev.synchronize()
            hit = hit or float(host[0]) != 0.0
        if hit:
            torch.cuda.synchronize(self.g.flat.device)
            self._polls = []
            n_r, _ = self.check_capacity()
            self.overflow_events += 1
            self.enable_graph(window, slack=self._slack, capacity=max(int(n_r * self._slack), int(self._graph.cap * 1.5)) + 4096)
        return hit

    def timing_breakdown(self, window, reps=10):
        """Device time (CUDA events, ms) of the step's collective alone -- the all-reduce of the packed bucket -- measured
        outside any timed benchmark region; {} on a single rank."""
        if not (self.dist and self.world > 1):
            return {}
        dev = self.g.flat.device
        buf = torch.zeros_like(self.g.bucket)
        for _ in range(3):
            self.dist.all_reduce(buf, op=self.dist.ReduceOp.SUM, group=self.group)
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            self.dist.all_reduce(buf, op=self.dist.ReduceOp.SUM, group=self.group)
        e1.record()
        torch.cuda.synchronize(dev)
        ms = torch.tensor([e0.elapsed_time(e1) / reps], device=dev)
        self.dist.all_reduce(ms, op=self.dist.ReduceOp.MAX, group=self.group)
        return {"allreduce_ms": float(ms.item()), "allreduce_algbw_gbs": buf.numel() * 4 / (float(ms.item()) * 1e-3) / 1e9}

    def schedule(self, window_size):
        """Keyframe index (into the window) rendered by each rank this step: a shared-seed permutation
        dealt round-robin, so ranks draw distinct keyframes whenever the window holds >= world frames."""
        perm = torch.randperm(window_size, generator=self.gen).tolist()
        return [perm[r % window_size] for r in range(self.world)]

    def accumulate(self, frame):
        """Local backward of one keyframe into the flat gradient bucket (no communication)."""
        keep = {} if self.track_means2D else None
        if self.refine_poses:
            self._bind_cameras()
        loss, radius = mapping_loss(self.params(), frame, self.render, fused_loss=self.fused, keep=keep,
                                    camera_grad=self.refine_poses)
        loss.backward()
        if keep is not None:      # gradient of the RGB render's 2D means: the densification statistic (splatam.py:250)
            self.last_means2D_grad = keep["means2D"].grad
            self.last_seen_local = (radius > 0)
        return loss.detach(), radius

    # ---- gradient-based densification (3DGS-style; off in every shipped SLAM config) -----------------------------
    def densify(self, iter, densify_dict, scene_radius, means2D_grad=None, seen=None, generator=None):
        """densify of the reference (R/utils/slam_external.py:191-243), same schedule keys (start_after, stop_after,
        densify_every, grad_thresh, num_to_split_into, removal_opacity_threshold, final_removal_opacity_threshold,
        remove_big_after, reset_opacities, reset_opacities_every): accumulates |d loss / d means2D| of the seen
        Gaussians, clones the small high-gradient ones, splits the large ones into num_to_split_into samples of
        their own distribution, drops transparent / oversized ones and optionally resets opacities.  Parameters and both
        Adam moments follow (new rows start with zero moments).  Clones and split samples inherit their parent's
        `timestep`, as R/utils/gs_external.py:202-222 does: the SLAM densify of slam_external.py does not grow it at all
        (DESIGN.md section 9).  Every rank must call it with the same all-reduced
        statistics; `generator` (default: the mapper's shared-seed generator when distributed, else torch's global
        RNG, as the reference) draws the split samples.  Returns the Gaussian count afterwards."""
        P = self.g.shapes["means3D"][0]
        dev = self.g.flat.device
        if self._dens is None or self._dens["accum"].shape[0] != P:
            self._dens = dict(accum=torch.zeros(P, device=dev), denom=torch.zeros(P, device=dev))
        if iter > densify_dict["stop_after"]:
            return P
        means2D_grad = self.last_means2D_grad if means2D_grad is None else means2D_grad
        if seen is None:       # the Gaussians THIS rank's render saw (the bucket's seen flags are already summed over ranks)
            seen = self.last_seen_local if self.last_seen_local is not None else (self.g.seen_f > 0)
        if self.dist and self.world > 1:
            # K ranks rendered K keyframes this step: the statistic of the step is the sum over the keyframes, exactly
            # what K sequential single-keyframe steps of the reference would have accumulated; summing it over the ranks
            # also keeps the replicas' clone / split decisions identical
            st = torch.stack([torch.norm(means2D_grad[:, :2], dim=-1) * seen, seen.to(torch.float32)])
            self.dist.all_reduce(st, op=self.dist.ReduceOp.SUM, group=self.group)
            self._dens["accum"] += st[0]
            self._dens["denom"] += st[1]
        elif self.fused:            # one launch, no nonzero() synchronisation (csrc/map_ops.cu)
            from . import map_ops
            map_ops.densify_accumulate(means2D_grad, seen, self._dens["accum"], self._dens["denom"])
        else:
            self._dens["accum"][seen] += torch.norm(means2D_grad[seen, :2], dim=-1)      # accumulate_mean2d_gradient
            self._dens["denom"][seen] += 1
        if not densify_due(iter, densify_dict):
            return P
        grads = self._dens["accum"] / self._dens["denom"]
        grads[grads.isnan()] = 0.0
        thr = densify_dict["grad_thresh"]
        cur = lambda: {k: self.g.params[k].detach() for k in GAUSSIAN_KEYS}
        big = lambda: torch.max(torch.exp(self.g.params["log_scales"].detach()), dim=1).values
        to_clone = torch.logical_and(grads >= thr, big() <= 0.01 * scene_radius)
        self.add_gaussians({k: v[to_clone] for k, v in cur().items()}, timestep=self.timestep[to_clone])
        num = self.g.shapes["means3D"][0]
        padded = torch.zeros(num, device=dev)
        padded[:grads.shape[0]] = grads
        to_split = torch.logical_and(padded >= thr, big() > 0.01 * scene_radius)
        n = int(densify_dict["num_to_split_into"])
        p = cur()
        new = {k: v[to_split].repeat(n, 1) for k, v in p.items()}
        stds = torch.exp(p["log_scales"])[to_split].repeat(n, 3)
        if generator is None and self.world > 1:
            generator = self._device_generator()
        samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds, generator=generator)
        rots = build_rotation(p["unnorm_rotations"][to_split]).repeat(n, 1, 1)
        new["means3D"] = new["means3D"] + torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1)
        new["log_scales"] = torch.log(torch.exp(new["log_scales"]) / (0.8 * n))
        self.add_gaussians(new, timestep=self.timestep[to_split].repeat(n))
        self.remove_points(torch.cat((to_split, torch.zeros(n * int(to_split.sum()), dtype=torch.bool, device=dev))))
        rthr = (densify_dict["final_removal_opacity_threshold"] if iter == densify_dict["stop_after"]
                else densify_dict["removal_opacity_threshold"])
        to_remove = (torch.sigmoid(self.g.params["logit_opacities"].detach()) < rthr).squeeze(-1)
        if iter >= densify_dict["remove_big_after"]:
            to_remove = torch.logical_or(to_remove, big() > 0.1 * scene_radius)
        P = self.remove_points(to_remove)
        self._dens = dict(accum=torch.zeros(P, device=dev), denom=torch.zeros(P, device=dev))
        if iter > 0 and iter % densify_dict["reset_opacities_every"] == 0 and densify_dict["reset_opacities"]:
            self._reset_opacities()
        return P

    def _device_generator(self):
        if self._dev_gen is None:
            self._dev_gen = torch.Generator(device=self.g.flat.device)
            self._dev_gen.manual_seed(12345)
        return self._dev_gen

    def run_state(self):
        """The mapper's part of a checkpoint's run state (slam._run_state), as numpy arrays: `timestep`, the schedule
        generator, the device generator if it has one and the densification statistic if there is one."""
        st = dict(timestep=self.timestep.detach().cpu().numpy(), mapper_gen=self.gen.get_state().numpy())
        if self._dev_gen is not None:
            st["mapper_dev_gen"] = self._dev_gen.get_state().numpy()
        if self._dens is not None:
            st["dens_accum"] = self._dens["accum"].detach().cpu().numpy()
            st["dens_denom"] = self._dens["denom"].detach().cpu().numpy()
        return st

    def load_run_state(self, st):
        """Inverse of run_state on a mapper built from the checkpoint's map; changes nothing if `timestep` does not
        fit the map."""
        import numpy as np
        dev = self.g.flat.device
        P = self.g.shapes["means3D"][0]
        if st["timestep"].shape != (P,):
            raise ValueError("the checkpoint's run state holds %d timesteps for a map of %d Gaussians"
                             % (st["timestep"].shape[0], P))
        self.timestep = torch.from_numpy(np.array(st["timestep"], dtype=np.float32)).to(dev)
        self.gen.set_state(torch.from_numpy(np.array(st["mapper_gen"], dtype=np.uint8)))
        if "mapper_dev_gen" in st:
            self._device_generator().set_state(torch.from_numpy(np.array(st["mapper_dev_gen"], dtype=np.uint8)))
        if "dens_accum" in st:
            self._dens = dict(accum=torch.from_numpy(np.array(st["dens_accum"], dtype=np.float32)).to(dev),
                              denom=torch.from_numpy(np.array(st["dens_denom"], dtype=np.float32)).to(dev))

    def step(self, window):
        """One sharded mapping step over `window` (list of keyframe dicts).  Returns the mean loss."""
        picks = self.schedule(len(window))
        graphed = self._graph is not None
        if graphed:
            self.poll_overflow(window)
            step, frame = self._graph, window[picks[self.rank]]
            step.load(frame)
            if self.refine_poses:
                self._bind_cameras()
                q, tr, col = step.pose_leaves
                with torch.no_grad():
                    q.copy_(self.cam["cam_unnorm_rots"][..., frame["id"]])
                    tr.copy_(self.cam["cam_trans"][..., frame["id"]])
                col.fill_(int(frame["id"]))
            else:
                for static, v in zip(step.frame["pose"], fused_pose_cached(self.params(), frame["id"])):
                    static.copy_(v, non_blocking=True)
            if "exposure" in step.frame:
                step.frame["exposure"].copy_(self.cam["cam_exposure"][0, :, frame["id"]], non_blocking=True)
            step.graph.replay()
        else:
            self.g.zero_grad()
            loss, radius = self.accumulate(window[picks[self.rank]])
            self.g.seen_f.copy_(radius > 0)
            self.g.loss_slot.copy_(loss.reshape(1))
        if self.dist and self.world > 1:
            # ONE collective per step: gradients, seen flags (sum of 0/1 > 0 == OR) and the loss travel together
            self.dist.all_reduce(self.g.bucket, op=self.dist.ReduceOp.SUM, group=self.group)
        if graphed:
            self.opt.step_guarded(self.g.overflow_slot)    # no-op on every rank if any rank's render overflowed
            if self.refine_poses:
                self._cam_step(self.g.overflow_slot)
            host = self._pin[self.step_idx % len(self._pin)]
            host.copy_(self.g.overflow_slot, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self._polls.append((ev, host))
        else:
            self.opt.step()
            if self.refine_poses:
                self._cam_step()
        self.step_idx += 1
        seen = self.g.seen_f > 0
        loss = self.g.loss_slot[0] / self.world
        if graphed:
            return loss.clone(), seen, picks      # device scalar: the graph path never synchronises
        return float(loss), seen, picks
