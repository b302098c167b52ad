"""Per-view training loss of the reference's train.py:151-188 as one fused CUDA pass over the rasterizer's 9-channel
output (csrc/view_loss.cu through the C ABI `gof_view_loss`) -- SURVEY.md section 8(f) rank 1, a CALLER of the rasterizer:

    loss = (1 - lambda_dssim) * L1(rgb, gt) + lambda_dssim * (1 - SSIM(rgb, gt))
           + lambda_depth_normal * mean(1 - n_world . depth_to_normal(depth)) + lambda_distortion * mean(distortion)

    loss, terms = view_loss(rendering, gt_image, viewpoint_cam.world_view_transform, tanfovx, tanfovy,
                            lambda_dssim=0.2, lambda_depth_normal=0.05, lambda_distortion=100.0)
    loss.backward()            # d loss / d rendering comes from the same pass

`terms` = tensor (L1, SSIM, normal-consistency loss, distortion loss, total) for logging.  CUDA tensors only.

With decoupled appearance (train.py:67-88, 157-159) the L1 term is the appearance network's: pass its output for this view
and the fused pass takes mean |mapping * crop(rgb) - crop(gt)| over gof_appearance.crop_window in place of the plain L1
(`gof_view_loss_appearance`); the backward also returns d loss / d mapping, which autograd carries through the network:

    mapping = gof_appearance.appearance_mapping(rendering[:3], network, embedding_row)
    loss, terms = view_loss(rendering, gt_image, ..., appearance=mapping)
"""
import ctypes

import torch

import gof_appearance
from diff_gaussian_rasterization import _C

_lib = _C._lib
_lib.gof_view_loss_scratch_bytes.restype = ctypes.c_size_t
_lib.gof_view_loss_scratch_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
_lib.gof_view_loss.restype = ctypes.c_int
_lib.gof_view_loss.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float,
                               ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                               ctypes.c_void_p, ctypes.c_void_p]
_lib.gof_view_loss_appearance.restype = ctypes.c_int
_lib.gof_view_loss_appearance.argtypes = ([ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_float] * 5 + [ctypes.c_void_p]
                                          + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 5)


def _run(rendering, gt, R9, fx, fy, lam, lam_dn, lam_dist, need_grad, app=None):
    """app = (mapping [3,Hc,Wc] fp32, top, left) for the appearance L1; returns (terms, grad, grad_mapping)."""
    if not (rendering.is_cuda and gt.is_cuda):
        raise RuntimeError("gof_b200 view_loss: CUDA tensors required (no CPU path)")
    if rendering.dim() != 3 or rendering.shape[0] != 9 or gt.shape != (3,) + tuple(rendering.shape[1:]):
        raise RuntimeError("view_loss: rendering must be (9,H,W) and gt (3,H,W)")
    r, g = rendering.detach().contiguous().float(), gt.detach().contiguous().float()
    H, W = int(r.shape[1]), int(r.shape[2])
    dev = r.device
    terms = torch.empty(5, dtype=torch.float32, device=dev)
    grad = torch.empty_like(r) if need_grad else None
    scratch = torch.empty(int(_lib.gof_view_loss_scratch_bytes(W, H)), dtype=torch.uint8, device=dev)
    Rh = (ctypes.c_float * 9)(*[float(x) for x in R9])
    gptr = grad.data_ptr() if need_grad else None
    grad_mapping = None
    with torch.cuda.device(dev):
        if app is None:
            _C._check(_lib.gof_view_loss(W, H, r.data_ptr(), g.data_ptr(), Rh, fx, fy, lam, lam_dn, lam_dist, terms.data_ptr(),
                                         gptr, scratch.data_ptr(), _C._stream()))
        else:
            m, top, left = app
            if not m.is_cuda or m.device != dev:
                raise RuntimeError("view_loss: the appearance mapping must be on the rendering's device")
            m = m.detach().contiguous().float()
            grad_mapping = torch.empty_like(m) if need_grad else None
            _C._check(_lib.gof_view_loss_appearance(
                W, H, r.data_ptr(), g.data_ptr(), Rh, fx, fy, lam, lam_dn, lam_dist, m.data_ptr(), top, left, int(m.shape[1]),
                int(m.shape[2]), terms.data_ptr(), gptr, grad_mapping.data_ptr() if need_grad else None, scratch.data_ptr(),
                _C._stream()))
    return terms, grad, grad_mapping


class _ViewLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rendering, gt, R9, fx, fy, lam, lam_dn, lam_dist):
        terms, grad, _ = _run(rendering, gt, R9, fx, fy, lam, lam_dn, lam_dist, rendering.requires_grad)
        ctx.save_for_backward(grad) if grad is not None else None
        ctx.has_grad = grad is not None
        ctx.mark_non_differentiable(terms)
        return terms[4].clone(), terms

    @staticmethod
    def backward(ctx, g_loss, _g_terms):
        if not ctx.has_grad:
            return (None,) * 8
        (grad,) = ctx.saved_tensors
        return grad * g_loss, None, None, None, None, None, None, None


class _ViewLossAppearance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rendering, mapping, gt, R9, fx, fy, lam, lam_dn, lam_dist, top, left):
        need_grad = rendering.requires_grad or mapping.requires_grad
        m3 = mapping.reshape(mapping.shape[-3:])
        terms, grad, grad_mapping = _run(rendering, gt, R9, fx, fy, lam, lam_dn, lam_dist, need_grad, (m3, top, left))
        ctx.save_for_backward(grad, grad_mapping) if need_grad else None
        ctx.has_grad, ctx.mapping_shape = need_grad, mapping.shape
        ctx.mark_non_differentiable(terms)
        return terms[4].clone(), terms

    @staticmethod
    def backward(ctx, g_loss, _g_terms):
        if not ctx.has_grad:
            return (None,) * 11
        grad, grad_mapping = ctx.saved_tensors
        return (grad * g_loss, (grad_mapping * g_loss).reshape(ctx.mapping_shape)) + (None,) * 9


def camera_rotation(world_view_transform):
    """Row-major camera-to-world rotation as 9 Python floats: ((world_view_transform^T)^-1)[:3,:3] (train.py:178)."""
    c2w = torch.linalg.inv(world_view_transform.detach().double().cpu().t())
    return [float(x) for x in c2w[:3, :3].reshape(-1)]


def view_loss(rendering, gt_image, world_view_transform, tanfovx, tanfovy, lambda_dssim=0.2, lambda_depth_normal=0.05,
              lambda_distortion=100.0, rotation=None, appearance=None):
    """Returns (loss, terms).  `rotation` = camera_rotation(world_view_transform) may be passed to avoid the small
    device->host copy per call (cameras are static during training).  `appearance` = the view's appearance mapping
    ([3,Hc,Wc] or [1,3,Hc,Wc], gof_appearance.appearance_mapping) replaces the L1 term by the decoupled-appearance L1 on
    the crop gof_appearance.crop_window(H, W); terms[0] is then that L1."""
    H, W = int(rendering.shape[1]), int(rendering.shape[2])
    R9 = rotation if rotation is not None else camera_rotation(world_view_transform)
    fx, fy = W / (2.0 * float(tanfovx)), H / (2.0 * float(tanfovy))
    lam = (float(lambda_dssim), float(lambda_depth_normal), float(lambda_distortion))
    if appearance is None:
        return _ViewLoss.apply(rendering, gt_image, R9, fx, fy, *lam)
    top, left, Hc, Wc = gof_appearance.crop_window_checked(H, W)
    if tuple(appearance.shape) not in ((3, Hc, Wc), (1, 3, Hc, Wc)):
        raise ValueError(f"view_loss: the appearance mapping must be [3,{Hc},{Wc}] or [1,3,{Hc},{Wc}] for a {H}x{W} image, "
                         f"not {list(appearance.shape)}")
    return _ViewLossAppearance.apply(rendering, appearance, gt_image, R9, fx, fy, *lam, top, left)
