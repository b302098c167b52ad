"""diff_gaussian_rasterization -- H100-native drop-in for GOF's rasterizer package.

Same import surface as the reference package of the same name
(submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py):

    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

* GaussianRasterizationSettings -- NamedTuple, same fields in the same order (reference :167-181)
* GaussianRasterizer(raster_settings).forward / .integrate / .markVisible (reference :183-305)
* rasterize_gaussians(...) and the autograd Function _RasterizeGaussians (reference :21-165)
* integrate_gaussians(...) (extension): the opacity-field query with alpha_integrated differentiable (_IntegrateGaussians)

so gaussian_renderer/__init__.py:14,99-108,199-209 of the reference runs unmodified on top of it.
The native side is libgof_b200.so (hand-written sm_90a CUDA, C ABI in include/gof_rasterizer.h) reached
through `_C`; there is no CPU or PyTorch fallback.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "integrate_gaussians"]


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float          # or a one-element tensor (extension): one that requires grad receives the focal-length gradient
    tanfovy: float
    kernel_size: float
    subpixel_offset: torch.Tensor
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _to_cpu(args):
    return tuple(a.detach().cpu().clone() if isinstance(a, torch.Tensor) else a for a in args)


def _call_native(fn, args, debug, dump_name, what, **kw):
    """Calls a `_C` entry point; with debug the inputs are snapshotted first and written to
    `dump_name` if the native call raises (reference :89-96, :141-148, :292-301)."""
    if not debug:
        return fn(*args, **kw)
    snapshot = _to_cpu(args)
    try:
        return fn(*args, **kw)
    except Exception:
        torch.save(snapshot, dump_name)
        print(f"\nAn error occured in {what}. Please forward {dump_name} for debugging.")
        raise


def _camera_args(rs):
    return (rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.kernel_size, rs.subpixel_offset)


def _camera_inputs(rs):
    """(viewmatrix, campos) when autograd is to differentiate the render with respect to the camera, otherwise ()."""
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in (rs.viewmatrix, rs.campos)):
        return (rs.viewmatrix, rs.campos)
    return ()


def _intrinsics_inputs(rs):
    """(tanfovx, tanfovy) when autograd is to differentiate the render with respect to the focal length (either is a tensor that
    requires grad), otherwise ()."""
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in (rs.tanfovx, rs.tanfovy)):
        return (rs.tanfovx, rs.tanfovy)
    return ()


def _extra_inputs(rs):
    """The inputs of _RasterizeGaussians after grad_bucket: today's (viewmatrix, campos) or nothing, and, when the focal length
    is to receive gradients, (tanfovx, tanfovy) after them."""
    cam, fov = _camera_inputs(rs), _intrinsics_inputs(rs)
    return (cam or (None, None)) + fov if fov else cam


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                view2gaussian_precomp, raster_settings, grad_bucket=None, viewmatrix=None, campos=None, tanfovx=None,
                tanfovy=None):
        """viewmatrix / campos, tanfovx / tanfovy (extension): raster_settings' own camera tensors, passed as inputs only
        when they are to receive gradients (the render reads them from raster_settings either way)."""
        rs = raster_settings
        ctx.grad_bucket = grad_bucket
        ctx.camera = viewmatrix is not None
        ctx.intrinsics = tanfovx is not None
        # shape, dtype and device of each tan_fov input that is a tensor: its gradient is returned like it
        ctx.fov_like = [(t.shape, t.dtype, t.device) if isinstance(t, torch.Tensor) else None for t in (tanfovx, tanfovy)]
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                view2gaussian_precomp) + _camera_args(rs) + (rs.image_height, rs.image_width, sh, rs.sh_degree,
                                                             rs.campos, rs.prefiltered, rs.debug)
        num_rendered, color, radii, geom, binning, img = _call_native(
            _C.rasterize_gaussians, args, rs.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, view2gaussian_precomp,
                              radii, sh, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii=None):
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, view2gaussian_precomp, radii, sh, geom,
         binning, img) = ctx.saved_tensors
        args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                view2gaussian_precomp) + _camera_args(rs) + (grad_out_color, sh, rs.sh_degree, rs.campos, geom,
                                                             ctx.num_rendered, binning, img, rs.debug)
        bucket = ctx.grad_bucket
        kw = {"_out": bucket.views} if bucket is not None else {}
        if ctx.camera:
            kw["_camera"] = True
        if ctx.intrinsics:
            kw["_intrinsics"] = True
        grads = _call_native(_C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", "backward", **kw)
        (g_means2D, g_colors, g_opacity, g_means3D, g_cov3D, g_sh, g_scales, g_rot, g_v2g) = grads[:9]
        if bucket is not None:
            # extension (view-parallel training, gof_dp.GradBucket): the parameter gradients and this view's densification
            # statistics were written INTO the bucket -- they are read from bucket.views after bucket.all_reduce(), not from
            # .grad (autograd would copy the 256 MB out of the exchange buffer again)
            g_means3D = g_sh = g_opacity = g_scales = g_rot = None
        # one gradient per forward input, in input order (reference :152-163)
        out = (g_means3D, g_means2D, g_sh, g_colors, g_opacity, g_scales, g_rot, g_cov3D, g_v2g, None, None)
        if ctx.camera:
            out += tuple(g if need else None for g, need in zip(grads[9:11], ctx.needs_input_grad[11:13]))
        if ctx.intrinsics:
            if not ctx.camera:
                out += (None, None)
            out += tuple(g.to(dtype=like[1], device=like[2]).reshape(like[0]) if need and like is not None else None
                         for g, like, need in zip(grads[-2:], ctx.fov_like, ctx.needs_input_grad[13:15]))
        return out


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        view2gaussian_precomp, raster_settings):
    """With grad mode on and raster_settings.viewmatrix or .campos requiring grad, the backward also differentiates the
    render with respect to them (DESIGN.md 4.9); projmatrix is treated as a constant.  Likewise for raster_settings.tanfovx /
    .tanfovy given as tensors that require grad (DESIGN.md 4.10): their gradients come back in their shape, dtype and
    device."""
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, view2gaussian_precomp, raster_settings, None,
                                     *_extra_inputs(raster_settings))


def _integrate_args(rs, points3D, means3D, colors_precomp, opacities, scales, rotations, cov3D_precomp, view2gaussian_precomp, shs):
    return (rs.bg, points3D, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3D_precomp,
            view2gaussian_precomp) + _camera_args(rs) + (rs.image_height, rs.image_width, shs, rs.sh_degree, rs.campos,
                                                         rs.prefiltered, rs.debug)


def _integrate_backward_args(rs, points3D, means3D, radii, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp,
                             shs, grad_alpha, num_rendered, geom, binning, img, pts, pbin):
    """The argument tuple of _C.integrate_gaussians_to_points_backward for the state of a query made with _integrate_args."""
    return (rs.bg, points3D, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3D_precomp,
            view2gaussian_precomp) + _camera_args(rs) + (rs.image_height, rs.image_width, shs, rs.sh_degree, rs.campos,
                                                         grad_alpha, num_rendered, geom, binning, img, pts, pbin, rs.debug)


class _IntegrateGaussians(torch.autograd.Function):
    """The opacity-field query with alpha_integrated differentiable with respect to points3D, means3D, opacities, scales,
    rotations and view2gaussian_precomp (DESIGN.md 4.11), and color_integrated with respect to the same Gaussian inputs, shs and
    colors_precomp (DESIGN.md 4.13; the points get nothing from it).  color and radii carry no gradient."""

    @staticmethod
    def forward(ctx, points3D, means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                view2gaussian_precomp, raster_settings):
        rs = raster_settings
        args = _integrate_args(rs, points3D, means3D, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                               view2gaussian_precomp, shs)
        (num_rendered, color, alpha_integrated, color_integrated, radii, geom, binning, img, pts, pbin) = _call_native(
            _C.integrate_gaussians_to_points_state, args, rs.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(points3D, means3D, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp, shs,
                              radii, geom, binning, img, pts, pbin)
        ctx.mark_non_differentiable(color, radii)
        ctx.set_materialize_grads(False)   # a color_integrated without a gradient keeps the alpha-only backward
        return color, alpha_integrated, color_integrated, radii

    @staticmethod
    def backward(ctx, _grad_color, grad_alpha, grad_color_integrated, _grad_radii):
        rs = ctx.raster_settings
        (points3D, means3D, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp, shs, radii, geom, binning, img,
         pts, pbin) = ctx.saved_tensors
        if grad_alpha is None and grad_color_integrated is None:
            grad_alpha = torch.zeros(points3D.size(0), dtype=torch.float32, device=points3D.device)
        args = _integrate_backward_args(rs, points3D, means3D, radii, colors_precomp, scales, rotations, cov3D_precomp,
                                        view2gaussian_precomp, shs, grad_alpha, ctx.num_rendered, geom, binning, img, pts, pbin)
        g_pts, g_opacity, g_means3D, g_scales, g_rot, g_cov3D, g_v2g, g_colors, g_sh = _call_native(
            _C.integrate_gaussians_to_points_backward, args, rs.debug, "snapshot_bw.dump", "backward",
            points_grad=ctx.needs_input_grad[0], dL_dcolor=grad_color_integrated)
        need = ctx.needs_input_grad
        pick = lambda g, i: g if need[i] else None   # noqa: E731
        return (pick(g_pts, 0), pick(g_means3D, 1), None, pick(g_opacity, 3), pick(g_sh, 4), pick(g_colors, 5), pick(g_scales, 6),
                pick(g_rot, 7), pick(g_cov3D, 8), pick(g_v2g, 9), None)


def integrate_gaussians(points3D, means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                        view2gaussian_precomp, raster_settings):
    """GaussianRasterizer.integrate with alpha_integrated (extension, DESIGN.md 4.11) and color_integrated (DESIGN.md 4.13)
    differentiable: returns the same (color[9,H,W], alpha_integrated[PN], color_integrated[PN,3], radii[P]).  Optional inputs
    are None or empty tensors, as for rasterize_gaussians.  With grad mode off, or with no input requiring grad, this is
    GaussianRasterizer.integrate."""
    shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp = _normalise_optionals(
        None if shs is None or shs.numel() == 0 else shs, None if colors_precomp is None or colors_precomp.numel() == 0 else colors_precomp,
        None if scales is None or scales.numel() == 0 else scales, None if rotations is None or rotations.numel() == 0 else rotations,
        None if cov3D_precomp is None or cov3D_precomp.numel() == 0 else cov3D_precomp,
        None if view2gaussian_precomp is None or view2gaussian_precomp.numel() == 0 else view2gaussian_precomp)
    inputs = (points3D, means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp)
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs):
        return _IntegrateGaussians.apply(points3D, means3D, means2D, opacities, shs, colors_precomp, scales, rotations,
                                         cov3D_precomp, view2gaussian_precomp, raster_settings)
    rs = raster_settings
    (_num_rendered, color, alpha_integrated, color_integrated, radii, _g, _b, _i) = _call_native(
        _C.integrate_gaussians_to_points, _integrate_args(rs, points3D, means3D, colors_precomp, opacities, scales, rotations,
                                                          cov3D_precomp, view2gaussian_precomp, shs),
        rs.debug, "snapshot_fw.dump", "forward")
    return color, alpha_integrated, color_integrated, radii


def _absent():
    # the reference encodes "not given" as an empty CPU float tensor (reference :209-224)
    return torch.Tensor([])


def _normalise_optionals(shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp):
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    has_partial_sr = (scales is not None) or (rotations is not None)
    has_full_sr = (scales is not None) and (rotations is not None)
    if (not has_full_sr and cov3D_precomp is None) or (has_partial_sr and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    fill = lambda t: _absent() if t is None else t
    return (fill(shs), fill(colors_precomp), fill(scales), fill(rotations), fill(cov3D_precomp),
            fill(view2gaussian_precomp))


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings, grad_bucket=None):
        """`grad_bucket` (extension, not in the reference): a gof_dp.GradBucket -- the backward then writes the gradients of
        means3D / shs / opacities / scales / rotations and the view's densification statistics into the bucket (the buffer a
        view-parallel step exchanges) instead of returning them to autograd."""
        super().__init__()
        self.raster_settings = raster_settings
        self.grad_bucket = grad_bucket

    def markVisible(self, positions):
        """bool[P]: view-space z > 0.2 (rasterizer_impl.cu:54-66)."""
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, view2gaussian_precomp=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp = _normalise_optionals(
            shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp)
        if self.grad_bucket is not None:
            if _camera_inputs(self.raster_settings):
                raise NotImplementedError("camera gradients (viewmatrix / campos requiring grad) are not available with a grad_bucket")
            if _intrinsics_inputs(self.raster_settings):
                raise NotImplementedError("focal-length gradients (tanfovx / tanfovy requiring grad) are not available with a grad_bucket")
            return _RasterizeGaussians.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                             cov3D_precomp, view2gaussian_precomp, self.raster_settings, self.grad_bucket)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, view2gaussian_precomp, self.raster_settings)

    def integrate(self, points3D, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                  rotations=None, cov3D_precomp=None, view2gaussian_precomp=None):
        """Opacity-field query (no gradients): (color[9,H,W], alpha_integrated[PN], color_integrated[PN,3],
        radii[P])  (reference :239-305)."""
        rs = self.raster_settings
        shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp = _normalise_optionals(
            shs, colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp)
        args = _integrate_args(rs, points3D, means3D, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                               view2gaussian_precomp, shs)
        (_num_rendered, color, alpha_integrated, color_integrated, radii, _g, _b, _i) = _call_native(
            _C.integrate_gaussians_to_points, args, rs.debug, "snapshot_fw.dump", "forward")
        return color, alpha_integrated, color_integrated, radii
