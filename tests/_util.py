"""Shared helpers for the parity tests (test infrastructure, not product code)."""
import glob
import importlib.util
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "gaussian-opacity-fields_b200")
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def load_ref():
    """The UNMODIFIED reference extension built by oracle/build_ref.sh (oracle/_ref/gof_ref_C*.so), or None."""
    hits = glob.glob(os.path.join(ROOT, "oracle", "_ref", "gof_ref_C*.so"))
    if not hits:
        return None
    spec = importlib.util.spec_from_file_location("gof_ref_C", hits[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _align(o, a=128):
    return (o + a - 1) // a * a


def carve_ref_geom(buf, P):
    """Fields of the reference's GeometryState (rasterizer_impl.cu:188-204) up to tiles_touched."""
    o = 0
    out = {}

    def take(name, count, dtype, shape):
        nonlocal o
        o = _align(o)
        nbytes = count * torch.empty(0, dtype=dtype).element_size()
        out[name] = buf[o:o + nbytes].view(dtype).view(shape).clone()
        o += nbytes

    take("depths", P, torch.float32, (P,))
    take("clamped", 3 * P, torch.uint8, (P, 3))
    take("internal_radii", P, torch.int32, (P,))
    take("means2D", 2 * P, torch.float32, (P, 2))
    take("cov3D", 6 * P, torch.float32, (P, 6))
    take("view2gaussian", 10 * P, torch.float32, (P, 10))
    take("conic_opacity", 4 * P, torch.float32, (P, 4))
    take("rgb", 3 * P, torch.float32, (P, 3))
    take("tiles_touched", P, torch.int32, (P,))
    return out


def carve_ref_image(buf, W, H):
    """ImageState (rasterizer_impl.cu:218-228)."""
    N = W * H
    o = 0
    out = {}

    def take(name, count, dtype, shape):
        nonlocal o
        o = _align(o)
        nbytes = count * torch.empty(0, dtype=dtype).element_size()
        if shape is not None:
            out[name] = buf[o:o + nbytes].view(dtype).view(shape).clone()
        o += nbytes

    take("accum_alpha", 4 * N, torch.float32, (4, H, W))
    take("center_depth", N, torch.float32, None)
    take("center_alphas", 4 * N, torch.float32, None)
    take("n_contrib", 2 * N, torch.int32, (2, H, W))
    take("ranges", 2 * N, torch.int32, (N, 2))
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    out["ranges"] = out["ranges"][:tiles].clone()
    return out


def carve_ref_binning(buf, R):
    """BinningState::point_list (rasterizer_impl.cu:230-243): first field."""
    return {"point_list": buf[0:4 * R].view(torch.int32).clone()}


def fwd_args(cam, gs, device, kernel_size=0.0, scale_modifier=1.0, bg=(0.0, 0.0, 0.0), sh_degree=None,
             colors_precomp=None, debug=False):
    """Argument tuple of `_C.rasterize_gaussians` (rasterize_points.cu:36-59)."""
    d = device
    empty = torch.Tensor([])
    deg = gs["sh_degree"] if sh_degree is None else sh_degree
    H, W = cam.image_height, cam.image_width
    return (
        torch.tensor(bg, dtype=torch.float32, device=d), gs["means3D"].to(d),
        empty if colors_precomp is None else colors_precomp.to(d), gs["opacities"].to(d), gs["scales"].to(d),
        gs["rotations"].to(d), scale_modifier, empty, empty, cam.world_view_transform.to(d),
        cam.full_proj_transform.to(d), cam.tanfovx, cam.tanfovy, kernel_size,
        torch.zeros((H, W, 2), dtype=torch.float32, device=d), H, W,
        gs["shs"].to(d) if colors_precomp is None else empty, deg, cam.camera_center.to(d), False, debug)


def bwd_args(fa, radii, geom, R, binning, img, grad):
    """Argument tuple of `_C.rasterize_gaussians_backward` (rasterize_points.cu:124-149) from forward args."""
    (bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D, v2g, viewmatrix, projmatrix, tfx, tfy,
     ks, subpix, H, W, sh, deg, campos, prefiltered, debug) = fa
    return (bg, means3D, radii, colors, scales, rotations, scale_modifier, cov3D, v2g, viewmatrix, projmatrix, tfx,
            tfy, ks, subpix, grad, sh, deg, campos, geom, R, binning, img, debug)


def same_up_to_summation_order(a, b):
    """Two backward runs over the same forward state: max|a - b| <= 1e-6 max|b| (test_gpu_repro's criterion).  The blend backward
    sums each Gaussian's partials in double and rounds once, so the order of its atomics moves a gradient only where a double sum
    lies next to a float rounding boundary."""
    a, b = a.double(), b.double()
    scale = float(b.abs().max()) if b.numel() else 0.0
    if scale == 0.0:
        return a.numel() == 0 or float(a.abs().max()) == 0.0
    return float((a - b).abs().max()) <= 1e-6 * scale


def rel_err(a, b):
    """max-abs-diff / max-abs-ref and relative L2 (the parity metric of SURVEY.md section 4.1)."""
    a = a.double().flatten()
    b = b.double().flatten()
    denom = b.abs().max().clamp_min(1e-30)
    l2 = (a - b).norm() / b.norm().clamp_min(1e-30)
    return float((a - b).abs().max() / denom), float(l2)
