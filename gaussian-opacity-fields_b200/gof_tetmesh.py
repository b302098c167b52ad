"""marching_tetrahedra -- drop-in for the reference's utils/tetmesh.py:141-189 on the GPU.

Same call and return structure as the reference (`extract_mesh.py:70`):

    verts_list, scale_list, faces_list, _ = marching_tetrahedra(vertices[None], tets, sdf[None], scales[None])
    end_points, end_sdf = verts_list[0]        # (E,2,3), (E,2,1)
    end_scales = scale_list[0]                 # (E,2,1)
    faces = faces_list[0]                      # (F,3) int64

implemented by libgof_b200.so (csrc/tetmesh.cu: crossing-edge sort + scans instead of torch.unique).  CUDA tensors only.
"""
import ctypes

import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib
_lib.gof_marching_tets_count.restype = ctypes.c_int
_lib.gof_marching_tets_count.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, _C._ALLOC_FN, ctypes.c_void_p,
                                         ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p]
_lib.gof_marching_tets_emit.restype = ctypes.c_int
_lib.gof_marching_tets_emit.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                        ctypes.c_int64, ctypes.c_int64] + [ctypes.c_void_p] * 7 + [ctypes.c_void_p]

CHUNK_TETS = 32 * 1024 * 1024   # utils/tetmesh.py:55


def chunk_rows(num_tets, chunk_tets=CHUNK_TETS):
    """Rows per chunk of the reference's split: torch.chunk(tets, T // chunk_size + 1) when T > chunk_size (utils/tetmesh.py:55-58),
    else one chunk; chunk_tets <= 0 also means one chunk.  The CUDA face order takes these rows (gof_marching_tets_emit)."""
    if chunk_tets <= 0 or num_tets <= chunk_tets:
        return max(int(num_tets), 1)
    n = num_tets // chunk_tets + 1
    return -(-num_tets // n)


def _unbatched_marching_tetrahedra(vertices, tets, sdf, scales, chunk_tets=CHUNK_TETS, rows=None):
    """`rows`: rows per chunk stated directly, in place of chunk_rows(T, chunk_tets) (gof_extract's tet shards cut where the
    unsharded call cuts)."""
    if not (vertices.is_cuda and tets.is_cuda and sdf.is_cuda and scales.is_cuda):
        raise RuntimeError("gof_b200 marching_tetrahedra: CUDA tensors required (no CPU path)")
    dev = vertices.device
    v = vertices.contiguous().float()
    t = tets.contiguous().long()
    s = sdf.contiguous().float().reshape(-1)
    sc = scales.contiguous().float().reshape(-1)
    V, T = int(v.shape[0]), int(t.shape[0])
    rows = int(rows) if rows is not None else chunk_rows(T, chunk_tets)
    scratch = _C._Scratch(dev, "tets")
    nE, nF = ctypes.c_int64(0), ctypes.c_int64(0)
    with torch.cuda.device(dev):
        _C._check(_lib.gof_marching_tets_count(V, s.data_ptr(), T, t.data_ptr() if T else None, scratch.cb, None, ctypes.byref(nE),
                                               ctypes.byref(nF), _C._stream()))
        E, F = nE.value, nF.value
        interp_v = torch.empty((E, 2), dtype=torch.long, device=dev)
        faces = torch.empty((F, 3), dtype=torch.long, device=dev)
        edge_pos = torch.empty((E, 2, 3), dtype=torch.float32, device=dev)
        edge_sdf = torch.empty((E, 2, 1), dtype=torch.float32, device=dev)
        edge_scales = torch.empty((E, 2, 1), dtype=torch.float32, device=dev)
        if T and (E or F):
            _C._check(_lib.gof_marching_tets_emit(V, s.data_ptr(), T, t.data_ptr(), rows, scratch.tensor.data_ptr(), E, F,
                                                  interp_v.data_ptr() if E else None, faces.data_ptr() if F else None, v.data_ptr(),
                                                  sc.data_ptr(), edge_pos.data_ptr() if E else None, edge_sdf.data_ptr() if E else None,
                                                  edge_scales.data_ptr() if E else None, _C._stream()))
    return (edge_pos, edge_sdf), edge_scales, faces, interp_v


def marching_tetrahedra(vertices, tets, sdf, scales):
    outs = [_unbatched_marching_tetrahedra(vertices[b], tets, sdf[b], scales[b]) for b in range(vertices.shape[0])]
    return list(zip(*outs))
