"""Inputs of the TSDF tests: analytic depth maps of a sphere seen by gof_synth.make_surface_views cameras."""
import numpy as np


def view_params(view):
    """(fx, fy, cx, cy, extrinsic [4,4] float32) of a gof_synth.SurfaceView, by the reference's formula."""
    W, H = view.image_width, view.image_height
    P = view.projection_matrix.double().numpy()
    fx, fy = np.float32(np.float32(W / 2) * np.float32(P[0, 0])), np.float32(np.float32(H / 2) * np.float32(P[1, 1]))
    cx, cy = np.float32((W - 1) / 2), np.float32((H - 1) / 2)
    E = view.world_view_transform.t().contiguous().numpy().astype(np.float32)
    return fx, fy, cx, cy, E


def sphere_depth(view, radius=1.0, center=(0.0, 0.0, 0.0)):
    """Depth (camera z) of the first hit of every pixel's ray with the sphere, 0 where the ray misses; float64 ray-sphere
    intersection rounded to float32 once."""
    fx, fy, cx, cy, E = view_params(view)
    H, W = view.image_height, view.image_width
    R, t = E[:3, :3].astype(np.float64), E[:3, 3].astype(np.float64)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    dc = np.stack([(u - float(cx)) / float(fx), (v - float(cy)) / float(fy), np.ones_like(u)], -1)   # z = 1: lambda = depth
    dw = dc @ R                                   # R^T dc, row-vector form
    o = -R.T @ t - np.asarray(center, np.float64)
    a = (dw * dw).sum(-1)
    b = 2.0 * (dw @ o)
    c = o @ o - radius * radius
    disc = b * b - 4 * a * c
    lam = (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a)
    return np.where((disc > 0) & (lam > 0), lam, 0.0).astype(np.float32)


def sphere_color(view, rgb=(0.25, 0.5, 0.75)):
    H, W = view.image_height, view.image_width
    return np.broadcast_to(np.asarray(rgb, np.float32)[:, None, None], (3, H, W)).copy()


def mesh_topology(faces):
    """(closed_and_oriented, euler characteristic) of a triangle mesh given as [F,3] vertex ids."""
    f = np.asarray(faces, np.int64)
    if not f.size:
        return False, 0
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    V = np.unique(f).size
    und = np.sort(directed, 1)
    uniq, cnt = np.unique(und, axis=0, return_counts=True)
    dir_uniq = np.unique(directed, axis=0)
    oriented = bool(np.all(cnt == 2)) and dir_uniq.shape[0] == directed.shape[0]
    return oriented, V - uniq.shape[0] + f.shape[0]


def signed_volume(vertices, faces):
    v = np.asarray(vertices, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)
