"""Parameter prologue / epilogue around the rasterizer (SURVEY.md section 8(f) rank 2; reference:
scene/gaussian_model.py:152-194 and :360) through the C ABI (`gof_activate_params*`, `gof_adam_step`, csrc/param_ops.cu).
The arithmetic is verified on the CPU against goldens generated from the reference's Python (tests/test_param_ops_host.py);
the CUDA kernels against those goldens (tests/test_gpu_param_ops.py) and against fp64 restatements at up to 10^6 Gaussians
(tests/test_gpu_train_step.py).

    scales, rotations, opacities, shs = activate(_scaling, _rotation, _opacity, filter_3D, _features_dc, _features_rest)
        == (pc.get_scaling_with_3D_filter, pc.get_rotation, pc.get_opacity_with_3D_filter, pc.get_features), differentiable
    adam_step(param, exp_avg, exp_avg_sq, grad, lr, step)      # torch.optim.Adam(eps=1e-15) update, in place
"""
import ctypes

import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib
_v = ctypes.c_void_p
_lib.gof_activate_params.restype = ctypes.c_int
_lib.gof_activate_params.argtypes = [ctypes.c_int, ctypes.c_int] + [_v] * 11
_lib.gof_activate_params_backward.restype = ctypes.c_int
_lib.gof_activate_params_backward.argtypes = [ctypes.c_int, ctypes.c_int] + [_v] * 14
_lib.gof_adam_step.restype = ctypes.c_int
_lib.gof_adam_step.argtypes = [ctypes.c_size_t, _v, _v, _v, _v, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                               ctypes.c_int, _v]


def _f32(t):
    if not t.is_cuda or t.dtype != torch.float32:
        raise RuntimeError("gof_b200 params: CUDA float32 tensors required (no CPU path)")
    return _C._c(t)     # the kernels move rotations as float4


class _Activate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scaling, rotation, opacity, filter_3D, f_dc, f_rest):
        s, q, o, f, dc, fr = (_f32(t.detach()) for t in (scaling, rotation, opacity, filter_3D, f_dc, f_rest))
        P, Mr = int(s.shape[0]), int(fr.shape[1])
        scales, rot, op = torch.empty_like(s), torch.empty_like(q), torch.empty_like(o)
        shs = torch.empty((P, Mr + 1, 3), dtype=torch.float32, device=s.device)
        with torch.cuda.device(s.device):
            _C._check(_lib.gof_activate_params(P, Mr, s.data_ptr(), q.data_ptr(), o.data_ptr(), f.data_ptr(), dc.data_ptr(),
                                               fr.data_ptr() if Mr else None, scales.data_ptr(), rot.data_ptr(), op.data_ptr(),
                                               shs.data_ptr(), _C._stream()))
        ctx.save_for_backward(s, q, o, f)
        ctx.Mr = Mr
        return scales, rot, op, shs

    @staticmethod
    def backward(ctx, g_scales, g_rot, g_op, g_shs):
        s, q, o, f = ctx.saved_tensors
        P, Mr = int(s.shape[0]), ctx.Mr
        z = lambda g, like: _f32(g) if g is not None else torch.zeros_like(like)
        gs, gr, go = z(g_scales, s), z(g_rot, q), z(g_op, o)
        gsh = _f32(g_shs) if g_shs is not None else torch.zeros((P, Mr + 1, 3), dtype=torch.float32, device=s.device)
        ds, dq, do = torch.empty_like(s), torch.empty_like(q), torch.empty_like(o)
        ddc = torch.empty((P, 1, 3), dtype=torch.float32, device=s.device)
        dfr = torch.empty((P, Mr, 3), dtype=torch.float32, device=s.device)
        with torch.cuda.device(s.device):
            _C._check(_lib.gof_activate_params_backward(P, Mr, s.data_ptr(), q.data_ptr(), o.data_ptr(), f.data_ptr(), gs.data_ptr(),
                                                        gr.data_ptr(), go.data_ptr(), gsh.data_ptr(), ds.data_ptr(), dq.data_ptr(),
                                                        do.data_ptr(), ddc.data_ptr(), dfr.data_ptr() if Mr else None, _C._stream()))
        return ds, dq, do, None, ddc, dfr


def activate(scaling, rotation, opacity, filter_3D, features_dc, features_rest):
    return _Activate.apply(scaling, rotation, opacity, filter_3D, features_dc, features_rest)


@torch.no_grad()
def adam_step(param, exp_avg, exp_avg_sq, grad, lr, step, beta1=0.9, beta2=0.999, eps=1e-15):
    """In-place torch.optim.Adam update of `param` (and its two moment buffers); `step` counts from 1."""
    for t in (param, exp_avg, exp_avg_sq, grad):
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError("gof_b200 adam_step: contiguous CUDA float32 tensors required")
    with torch.cuda.device(param.device):
        _C._check(_lib.gof_adam_step(param.numel(), param.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(), grad.data_ptr(),
                                     float(lr), float(beta1), float(beta2), float(eps), int(step), _C._stream()))
    return param


_lib.gof_compute_3d_filter.restype = ctypes.c_int
_lib.gof_compute_3d_filter.argtypes = [ctypes.c_int, _v, ctypes.c_int, _v, ctypes.c_float, _v, _v, _v]


def pack_cameras(cameras, device):
    """[n,16] float32 table for compute_3d_filter from objects with the reference Camera's attributes
    (R, T, focal_x, focal_y, image_width, image_height; scene/cameras.py)."""
    rows = []
    for c in cameras:
        rows.append(torch.cat([torch.as_tensor(c.R, dtype=torch.float32).reshape(-1), torch.as_tensor(c.T, dtype=torch.float32).reshape(-1),
                               torch.tensor([c.focal_x, c.focal_y, c.image_width, c.image_height], dtype=torch.float32)]))
    return torch.stack(rows).contiguous().to(device)


@torch.no_grad()
def compute_3d_filter(xyz, cam_table, max_focal):
    """== GaussianModel.compute_3D_filter (scene/gaussian_model.py:262-311): returns filter_3D [P,1]."""
    x = _f32(xyz)
    P = int(x.shape[0])
    out = torch.empty(P, dtype=torch.float32, device=x.device)
    scratch = torch.empty(1, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        _C._check(_lib.gof_compute_3d_filter(P, x.data_ptr(), int(cam_table.shape[0]), _f32(cam_table).data_ptr(), float(max_focal),
                                             out.data_ptr(), scratch.data_ptr(), _C._stream()))
    # the reference raises here too (distance[valid_points].max() of an empty tensor, :301) -- and synchronises, like this read
    if P and int(scratch.item()) == 0:
        raise RuntimeError("compute_3D_filter: no point is seen by any camera")
    return out[:, None]
