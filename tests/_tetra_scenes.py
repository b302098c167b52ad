"""TEST INFRASTRUCTURE for the tetrahedra points (csrc/tetra_points.cu): seeded Gaussians and views, points placed exactly on
the frustum's edges, and the reference's own get_frustum_mask / GaussianModel.get_tetra_points loaded from its staged source."""
import math
import types
import typing

import numpy as np
import torch

import _refpy
import gof_synth
import tetra_points_oracle as tpo


class Cam:
    """The attributes of the reference's scene.cameras.Camera that get_frustum_mask reads."""

    def __init__(self, world_view_transform, focal_x, focal_y, image_width, image_height):
        self.world_view_transform = world_view_transform
        self.focal_x, self.focal_y = focal_x, focal_y
        self.image_width, self.image_height = image_width, image_height


def _cam(c, device):
    return Cam(c.world_view_transform.to(device), c.focal_x, c.image_height / (2.0 * c.tanfovy), c.image_width, c.image_height)


def ring_views(n, width, height, device="cpu", radius=4.0):
    return [_cam(gof_synth.make_camera(width, height, view=i, n_views=n, radius=radius), device) for i in range(n)]


def surface_views(n, width, height, device="cpu"):
    return [_cam(c, device) for c in gof_synth.make_surface_views(width, height, n, radius=3.0)]


def gaussians(P, seed, kind="random"):
    """(xyz, scales, raw rotations) float32 CPU tensors.  The raw quaternions have norms between 0.2 and 3, as unnormalised
    `_rotation` parameters do."""
    if kind == "surface":
        gs = gof_synth.make_surface_gaussians(P, seed)
        gs["scales"] = gs["scales"] * 4.0
    else:
        gs = gof_synth.make_gaussians(P, seed, focal_x=400.0, extent=2.5)
        gs["scales"] = gs["scales"] * 20.0
    g = torch.Generator().manual_seed(seed + 1)
    k = torch.exp(torch.rand(P, 1, generator=g, dtype=torch.float64) * math.log(15.0) + math.log(0.2))
    rot = (gs["rotations"].to(torch.float64) * k).to(torch.float32).contiguous()
    return gs["means3D"].contiguous(), gs["scales"].to(torch.float32).contiguous(), rot


def edge_scene(near=0.02, far=1e6, device="cpu"):
    """One camera at the origin looking down +z (identity world_view_transform), W = 64, H = 48, fx = fy = 32, and points whose
    float32 u, v or depth land exactly on each bound of the frustum, and one float32 step beyond it, in every evaluation order
    (every product and sum is exact).  Returns (view, points float32 [n,3], expected mask)."""
    W, H, f = 64, 48, 32.0
    view = Cam(torch.eye(4, dtype=torch.float32, device=device), f, f, W, H)
    f32 = np.float32
    near32, far32 = f32(near), f32(far)

    def edge(bound, half, direction):
        # at depth 1: u = f x + W/2.  The coordinate on the bound, and the first float32 coordinate beyond it whose u is a
        # float32 number (so that no evaluation order rounds it back onto the bound)
        c0 = (bound - half) / f
        assert float(f32(c0)) == c0
        c = f32(c0)
        while True:
            c = np.nextafter(c, f32(direction * np.inf), dtype=np.float32)
            q = f * float(c) + half
            if float(f32(q)) == q and (q - bound) * direction > 0:
                return c0, float(c)

    pts, exp = [], []
    for bound, direction in ((0.0, -1), (W - 1.0, 1)):
        on, out = edge(bound, W / 2, direction)
        pts += [[on, 0.0, 1.0], [out, 0.0, 1.0]]
        exp += [True, False]
    for bound, direction in ((0.0, -1), (H - 1.0, 1)):
        on, out = edge(bound, H / 2, direction)
        pts += [[0.0, on, 1.0], [0.0, out, 1.0]]
        exp += [True, False]
    up = lambda a, d: np.nextafter(f32(a), f32(d), dtype=np.float32)   # noqa: E731
    for z, ok in ((near32, True), (up(near32, 0), False), (far32, True), (up(far32, np.inf), False)):
        pts.append([0.0, 0.0, float(z)]), exp.append(ok)        # u = W/2, v = H/2 exactly at any depth
    for p in ([0.0, 0.0, -1.0], [0.0, 0.0, -near], [np.inf, 0.0, 1.0], [0.0, -np.inf, 1.0], [0.0, 0.0, np.inf], [np.nan, 0.0, 1.0],
              [0.0, np.nan, 1.0]):
        pts.append(p), exp.append(False)                        # behind the camera, non-finite
    return view, np.array(pts, np.float32), np.array(exp)


def ref_frustum_mask():
    """The reference's get_frustum_mask, compiled from its unmodified source (None when the source is not staged)."""
    import einops
    glb = {"torch": torch, "einsum": einops.einsum, "List": typing.List, "Camera": Cam}
    return _refpy.ref_function("gaussian_model.py", "get_frustum_mask", glb) if _refpy.staged("text", "gaussian_model.py") else None


def ref_tetra_points(xyz, scales, rotation, views, near=0.02, far=1e6):
    """GaussianModel.get_tetra_points run from the reference's source text on a stub model, with its build_rotation and a
    trimesh.creation.box stub built from the box table.  Returns (points, scales) as the reference does, plus the unmasked
    vertices and mask it handed to get_frustum_mask.  None when the source is not staged."""
    gmask = ref_frustum_mask()
    gu = _refpy.ref_utils("general_utils")
    if gmask is None or gu is None:
        return None
    seen = {}

    def spy(vertices, views_, near_, far_):
        m = gmask(vertices, views_, near_, far_)
        seen["vertices"], seen["mask"] = vertices, m
        return m

    box = types.SimpleNamespace(vertices=tpo.BOX_SIGNS.astype(np.float64) / 2)   # trimesh's unit cube, before `*= 2`
    trimesh = types.SimpleNamespace(creation=types.SimpleNamespace(box=lambda: types.SimpleNamespace(vertices=box.vertices.copy())))
    glb = {"torch": torch, "trimesh": trimesh, "build_rotation": gu.build_rotation, "get_frustum_mask": spy, "List": typing.List,
           "Camera": Cam}
    ns = {}
    exec(_refpy.ref_method_source("gaussian_model.py", "GaussianModel", "get_tetra_points"), glb, ns)
    model = types.SimpleNamespace(_rotation=rotation, get_xyz=xyz, get_scaling_with_3D_filter=scales)
    with torch.no_grad():
        pts, sc = ns["get_tetra_points"](model, views, near, far)
    return pts, sc, seen["vertices"], seen["mask"]
