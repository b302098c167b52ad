"""simple_knn._C.distCUDA2 on this package's CUDA library (csrc/knn.cu through the C ABI `gof_knn_mean_dist`).

    from simple_knn._C import distCUDA2
    dist2 = distCUDA2(points)        # points: CUDA float32 [P,3] -> float32 [P] on the same device

dist2[i] is the mean squared distance from point i to its three nearest other points, bit-identical to the reference
(spatial.cu:15-25, simple_knn.cu:147-183; the contract is in include/gof_rasterizer.h and DESIGN section 4.5).  Clamping
and the logarithm stay with the caller, as in GaussianModel.create_from_pcd (scene/gaussian_model.py:327).  The call runs
on the current stream of the points' device, takes its scratch from torch's caching allocator and never synchronises
with the host, so it can be captured in a CUDA graph.
"""
import ctypes

import torch

from diff_gaussian_rasterization import _C as _gof

_lib = _gof._lib

_lib.gof_knn_scratch_bytes.restype = ctypes.c_size_t
_lib.gof_knn_scratch_bytes.argtypes = [ctypes.c_int]
_lib.gof_knn_mean_dist.restype = ctypes.c_int
_lib.gof_knn_mean_dist.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                   ctypes.c_void_p]


def distCUDA2(points):
    if not isinstance(points, torch.Tensor):
        raise TypeError(f"distCUDA2: expected a torch.Tensor, got {type(points).__name__}")
    if not points.is_cuda:
        raise RuntimeError("distCUDA2: points must be a CUDA tensor (there is no CPU path)")
    if points.dtype != torch.float32:
        raise RuntimeError(f"distCUDA2: points must be float32, got {points.dtype}")
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError(f"distCUDA2: points must have shape [P, 3], got {list(points.shape)}")
    P = int(points.shape[0])
    if P >= 2 ** 31:
        raise RuntimeError(f"distCUDA2: {P} points; at most 2^31 - 1 are supported (the reference's int P)")
    dev = points.device
    with torch.cuda.device(dev):
        out = torch.empty(P, dtype=torch.float32, device=dev)
        if P == 0:
            return out
        pts = points.detach().contiguous()
        if pts.data_ptr() & 3:
            pts = pts.clone(memory_format=torch.contiguous_format)
        nbytes = int(_lib.gof_knn_scratch_bytes(P))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _gof._check(_lib.gof_knn_mean_dist(P, pts.data_ptr(), out.data_ptr(), scratch.data_ptr(), nbytes, _gof._stream()))
    return out
