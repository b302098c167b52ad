"""diff_gaussian_rasterization -- H100-native drop-in for GOF's rasterizer package.

Same import surface as the reference package of the same name
(submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py):

    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

* GaussianRasterizationSettings -- NamedTuple, same fields in the same order (reference :167-181)
* GaussianRasterizer(raster_settings).forward / .integrate / .markVisible (reference :183-305)
* rasterize_gaussians(...) and the autograd Function _RasterizeGaussians (reference :21-165)

so gaussian_renderer/__init__.py:14,99-108,199-209 of the reference runs unmodified on top of it.
The native side is libgof_b200.so (hand-written sm_90a CUDA, C ABI in include/gof_rasterizer.h) reached
through `_C`; there is no CPU or PyTorch fallback.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"]


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
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


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                view2gaussian_precomp, raster_settings, grad_bucket=None):
        rs = raster_settings
        ctx.grad_bucket = grad_bucket
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
        (g_means2D, g_colors, g_opacity, g_means3D, g_cov3D, g_sh, g_scales, g_rot, g_v2g) = _call_native(
            _C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", "backward",
            **({"_out": bucket.views} if bucket is not None else {}))
        if bucket is not None:
            # extension (view-parallel training, gof_dp.GradBucket): the parameter gradients and this view's densification
            # statistics were written INTO the bucket -- they are read from bucket.views after bucket.all_reduce(), not from
            # .grad (autograd would copy the 256 MB out of the exchange buffer again)
            g_means3D = g_sh = g_opacity = g_scales = g_rot = None
        # one gradient per forward input, in input order (reference :152-163)
        return (g_means3D, g_means2D, g_sh, g_colors, g_opacity, g_scales, g_rot, g_cov3D, g_v2g, None, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        view2gaussian_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, view2gaussian_precomp, raster_settings, None)


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
        args = (rs.bg, points3D, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                cov3D_precomp, view2gaussian_precomp) + _camera_args(rs) + (rs.image_height, rs.image_width, shs,
                                                                            rs.sh_degree, rs.campos, rs.prefiltered,
                                                                            rs.debug)
        (_num_rendered, color, alpha_integrated, color_integrated, radii, _g, _b, _i) = _call_native(
            _C.integrate_gaussians_to_points, args, rs.debug, "snapshot_fw.dump", "forward")
        return color, alpha_integrated, color_integrated, radii
