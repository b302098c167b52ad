"""GaussianModel.densify_and_prune (scene/gaussian_model.py:683-707 with densify_and_clone / densify_and_split / prune_points /
cat_tensors_to_optimizer / _prune_optimizer, :549-681) through the C ABI (csrc/densify.cu) -- SURVEY.md 8(f) rank 4.

The reference re-allocates every parameter and both Adam moment tensors three times per call through boolean masks and
torch.cat; here the decision of every Gaussian (keep / clone / split / prune) is taken by one kernel, four scans give the output
rows, and every tensor is rebuilt once by a row gather.  Same result: the surviving rows are [kept originals | clones | first
split children | second split children], new rows carry zero Adam moments, all densification statistics restart at zero.

    new = densify_and_prune(params, exp_avg, exp_avg_sq, xyz_gradient_accum, xyz_gradient_accum_abs, denom,
                            max_grad=0.0002, min_opacity=0.05, extent=scene.cameras_extent, max_screen_size=size_threshold)
    new.params["xyz"], new.exp_avg["xyz"], ... ; new.counts = (kept, cloned, split children 1, split children 2)

`params` maps the reference's optimizer group names ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation") to the RAW
parameter tensors.  The new positions are drawn from the library's Philox generator (`seed`), or from `noise` ([3, P, 3] standard
normal samples: clone, first child, second child -- used by the parity test against the reference's own code)."""
import ctypes
from typing import NamedTuple

import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib
_v = ctypes.c_void_p
_lib.gof_densify_scratch_bytes.restype = ctypes.c_size_t
_lib.gof_densify_scratch_bytes.argtypes = [ctypes.c_int]
_lib.gof_densify_plan.restype = ctypes.c_int
_lib.gof_densify_plan.argtypes = [ctypes.c_int] + [_v] * 5 + [ctypes.c_float] * 5 + [_v] * 5
_lib.gof_densify_emit.restype = ctypes.c_int
_lib.gof_densify_emit.argtypes = [ctypes.c_int, _v, _v, _v, _v, _v, _v, _v, ctypes.c_ulonglong, _v, _v, _v, _v, _v]
_lib.gof_gather_rows_f32.restype = ctypes.c_int
_lib.gof_gather_rows_f32.argtypes = [_v, ctypes.c_int, _v, _v, ctypes.c_size_t, ctypes.c_int, _v, _v]

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


class Densified(NamedTuple):
    params: dict
    exp_avg: dict
    exp_avg_sq: dict
    counts: tuple
    src_index: torch.Tensor
    kind: torch.Tensor


def _f32(t):
    if not t.is_cuda or t.dtype != torch.float32:
        raise RuntimeError("gof_b200 densify: CUDA float32 tensors required (no CPU path)")
    return t.detach().contiguous()


@torch.no_grad()
def densify_and_prune(params, exp_avg, exp_avg_sq, xyz_gradient_accum, xyz_gradient_accum_abs, denom, max_grad, min_opacity, extent,
                      max_screen_size, percent_dense=0.01, noise=None, seed=0):
    p = {k: _f32(params[k]) for k in GROUPS}
    P = int(p["xyz"].shape[0])
    dev = p["xyz"].device
    acc, acc_abs, den = _f32(xyz_gradient_accum).reshape(-1), _f32(xyz_gradient_accum_abs).reshape(-1), _f32(denom).reshape(-1)
    # the two scalars of gaussian_model.py:684-690 (a mean and a quantile of P values: plain torch)
    grads = acc / den
    grads[grads.isnan()] = 0.0
    grads_abs = acc_abs / den
    grads_abs[grads_abs.isnan()] = 0.0
    ratio = (grads >= max_grad).float().mean()
    Q = float(torch.quantile(grads_abs, 1 - ratio)) if P else 0.0
    flags = torch.empty(4 * max(P, 1), dtype=torch.int32, device=dev)
    offsets = torch.empty_like(flags)
    totals = torch.zeros(4, dtype=torch.int32, device=dev)
    tmp = torch.empty(max(int(_lib.gof_densify_scratch_bytes(P)), 1), dtype=torch.uint8, device=dev)
    st = _C._stream()
    with torch.cuda.device(dev):
        _C._check(_lib.gof_densify_plan(P, acc.data_ptr(), acc_abs.data_ptr(), den.data_ptr(), p["scaling"].data_ptr(), p["opacity"].data_ptr(),
                                        float(max_grad), Q, float(percent_dense) * float(extent), float(min_opacity),
                                        0.1 * float(extent) if max_screen_size else 0.0, flags.data_ptr(), offsets.data_ptr(),
                                        totals.data_ptr(), tmp.data_ptr(), st))
        counts = tuple(int(x) for x in totals.cpu())            # sizes the outputs (the reference synchronises at every mask)
        N = sum(counts)
        src = torch.empty(max(N, 1), dtype=torch.int32, device=dev)
        kind = torch.empty(max(N, 1), dtype=torch.uint8, device=dev)
        new_xyz = torch.empty((N, 3), dtype=torch.float32, device=dev)
        new_scaling = torch.empty((N, 3), dtype=torch.float32, device=dev)
        tot_host = (ctypes.c_uint32 * 4)(*counts)
        nz = _f32(noise) if noise is not None else None
        if nz is not None and tuple(nz.shape) != (3, P, 3):
            raise RuntimeError("densify: noise must be [3, P, 3]")
        if P and N:
            _C._check(_lib.gof_densify_emit(P, flags.data_ptr(), offsets.data_ptr(), tot_host, p["xyz"].data_ptr(), p["scaling"].data_ptr(),
                                            p["rotation"].data_ptr(), nz.data_ptr() if nz is not None else None, int(seed), src.data_ptr(),
                                            kind.data_ptr(), new_xyz.data_ptr(), new_scaling.data_ptr(), st))

        def gather(t, zero_new):
            t = _f32(t)
            row = int(t[0].numel()) if P else 1
            out = torch.empty((N,) + tuple(t.shape[1:]), dtype=torch.float32, device=dev)
            if N:
                _C._check(_lib.gof_gather_rows_f32(t.data_ptr(), row, src.data_ptr(), kind.data_ptr(), N, 1 if zero_new else 0, out.data_ptr(), st))
            return out

        out_p, out_m, out_v = {}, {}, {}
        for k in GROUPS:
            out_p[k] = new_xyz if k == "xyz" else (new_scaling if k == "scaling" else gather(p[k], False))
            out_m[k] = gather(exp_avg[k], True)
            out_v[k] = gather(exp_avg_sq[k], True)
    return Densified(out_p, out_m, out_v, counts, src[:N], kind[:N])
