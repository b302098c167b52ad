"""Seeded synthetic workloads (SURVEY.md section 8(d)): pinhole cameras on a ring and random Gaussians.

Camera matrices are built the way the reference builds them (scene/cameras.py:56-59 with
utils/graphics_utils.py:38-71): row-vector convention, i.e. the tensors handed to the rasterizer are the
transposes of the usual column-vector matrices, which the CUDA side reads as column-major.
Everything is generated on the CPU with an explicit torch.Generator so fixtures are reproducible on any box.
"""
import math
from typing import NamedTuple

import torch


class SynthCamera(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    world_view_transform: torch.Tensor   # (4,4) = W2V^T
    full_proj_transform: torch.Tensor    # (4,4)
    camera_center: torch.Tensor          # (3,)
    focal_x: float


def _projection(znear, zfar, tan_half_x, tan_half_y):
    # utils/graphics_utils.py:51-71
    top, right = tan_half_y * znear, tan_half_x * znear
    P = torch.zeros(4, 4, dtype=torch.float32)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def make_camera(width, height, view=0, n_views=64, radius=4.0, fovx_deg=60.0, elevation=0.35,
                znear=0.01, zfar=100.0):
    """Camera `view` of a ring of `n_views` cameras of radius `radius` looking at the origin."""
    th = 2.0 * math.pi * (view % n_views) / n_views
    C = torch.tensor([radius * math.cos(th) * math.cos(elevation), -radius * math.sin(elevation),
                      radius * math.sin(th) * math.cos(elevation)], dtype=torch.float64)
    z = -C / C.norm()
    up = torch.tensor([0.0, -1.0, 0.0], dtype=torch.float64)
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    R = torch.stack([x, y, z], dim=1)          # camera-to-world rotation (columns = camera axes)
    T = -(R.t() @ C)
    Rt = torch.eye(4, dtype=torch.float64)     # getWorld2View2: [R^T | T]
    Rt[:3, :3] = R.t()
    Rt[:3, 3] = T
    w2v = Rt.to(torch.float32)
    tan_x = math.tan(math.radians(fovx_deg) / 2.0)
    tan_y = tan_x * height / width
    world_view = w2v.t().contiguous()
    proj = _projection(znear, zfar, tan_x, tan_y).t().contiguous()
    full = (world_view.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = torch.linalg.inv(world_view)[3, :3].contiguous()
    return SynthCamera(height, width, tan_x, tan_y, world_view, full, center, width / (2.0 * tan_x))


def make_gaussians(P, seed, focal_x, sh_degree=3, sigma_px=2.0, sigma_spread=0.7, extent=1.5, radius=4.0):
    """P random Gaussians: dict of CPU float32 tensors shaped like GaussianModel's activated properties.

    Everything is drawn and transformed in float64 and rounded to float32 ONCE at the end.  Round 1 generated in float32, and
    torch's vectorised CPU exp / sigmoid / normal sampling differ by an ulp between hosts (AVX2 vs AVX-512 code paths of
    SLEEF): one Gaussian's footprint then touched one tile more or less and `num_rendered` of the same workload differed by one
    between the bench box and the scaling box.  A float64 ulp survives the final rounding only when the value sits within
    2^-29 of a float32 rounding boundary, so the float32 scene is the same on every host."""
    g = torch.Generator().manual_seed(int(seed))
    f64 = torch.float64
    means3D = (torch.rand(P, 3, generator=g, dtype=f64) * 2.0 - 1.0) * extent
    sig = torch.exp(math.log(sigma_px) + sigma_spread * torch.randn(P, 1, generator=g, dtype=f64))
    aniso = torch.exp(torch.rand(P, 3, generator=g, dtype=f64) * math.log(1.0 / 0.3) + math.log(0.3))
    scales = (sig * radius / focal_x) * aniso
    rot = torch.randn(P, 4, generator=g, dtype=f64)
    rotations = rot / rot.norm(dim=1, keepdim=True)
    opacities = torch.sigmoid(1.5 * torch.randn(P, 1, generator=g, dtype=f64))
    M = 16
    shs = torch.zeros(P, M, 3, dtype=f64)
    shs[:, 0, :] = (torch.rand(P, 3, generator=g, dtype=f64) * 2.0 - 1.0) * 1.77
    shs[:, 1:, :] = 0.1 * torch.randn(P, M - 1, 3, generator=g, dtype=f64)
    f32 = lambda t: t.to(torch.float32).contiguous()   # noqa: E731
    return {"means3D": f32(means3D), "scales": f32(scales), "rotations": f32(rotations), "opacities": f32(opacities), "shs": f32(shs),
            "sh_degree": sh_degree}


# the configurations of BASELINE.json / BASELINE.md section 2.2
CONFIGS = {
    "C1": dict(P=10_000, width=256, height=256, seed=0),
    "C2": dict(P=200_000, width=800, height=800, seed=1),
    "C3": dict(P=1_000_000, width=1920, height=1080, seed=2),
    "C4": dict(P=2_500_000, width=1920, height=1080, seed=3, appearance=True),
    # mesh extraction: 3 M Gaussians, 27 M tetrahedra vertices (9 per Gaussian, as get_tetra_points), 64 views, ~6.5 tets
    # per point -- sized so that the whole extraction (64 cached views, ~176 M tets and the marching-tetrahedra scratch of
    # ~150 B/tet) fits one 80 GB GPU
    "C5": dict(P=3_000_000, width=1920, height=1080, seed=4, points=27_000_000, tets_per_point=6.5, n_views=64),
}


def make_tetra_points(gs, n_points, seed, device):
    """Query points of the extraction workload, generated ON `device`: like GaussianModel.get_tetra_points
    (scene/gaussian_model.py:433-463) the 8 corners of every Gaussian's 3-sigma box plus its centre (9 P points), topped up
    to `n_points` with points drawn uniformly inside the 3-sigma boxes.  Points of one Gaussian are contiguous, so nearby
    indices are nearby in space.  Returns (points [n,3], scale [n,1])."""
    g = torch.Generator(device=device).manual_seed(int(seed))
    xyz, scales, q = gs["means3D"].to(device), gs["scales"].to(device), gs["rotations"].to(device)
    P = xyz.shape[0]
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(P, 3, 3)
    corners = torch.tensor([[sx, sy, sz] for sx in (-1.0, 1.0) for sy in (-1.0, 1.0) for sz in (-1.0, 1.0)], device=device)   # [8,3]
    per = max(int(n_points) // P, 1)
    n_rand = max(per - 9, 0)
    parts = []
    if per >= 9:
        local = torch.cat([corners[None].expand(P, 8, 3), torch.zeros(P, 1, 3, device=device)], dim=1)
        if n_rand:
            local = torch.cat([local, torch.rand(P, n_rand, 3, generator=g, device=device) * 2 - 1], dim=1)
    else:
        local = torch.rand(P, per, 3, generator=g, device=device) * 2 - 1
    k = local.shape[1]
    pts = torch.einsum("pij,pkj->pki", R, local * (3.0 * scales)[:, None, :]) + xyz[:, None, :]
    parts.append(pts.reshape(-1, 3))
    sc = (3.0 * scales).amax(dim=1, keepdim=True)[:, None, :].expand(P, k, 1).reshape(-1, 1)
    points = parts[0]
    if points.shape[0] < n_points:          # remainder: extra samples around the first Gaussians
        m = int(n_points) - points.shape[0]
        idx = torch.arange(m, device=device) % P
        extra = torch.einsum("pij,pj->pi", R[idx], (torch.rand(m, 3, generator=g, device=device) * 2 - 1) * 3.0 * scales[idx]) + xyz[idx]
        points = torch.cat([points, extra])
        sc = torch.cat([sc, (3.0 * scales[idx]).amax(dim=1, keepdim=True)])
    return points[:n_points].contiguous(), sc[:n_points].contiguous()


def make_local_tets(n_points, n_tets, seed, device):
    """Synthetic tetrahedralisation of the query points for the marching-tetrahedra workload (CGAL's Delaunay, the
    reference's tet source, is a single-threaded CPU library that is not part of this image): every tet joins a vertex with
    three others at most 17 indices away -- the point cluster of the same Gaussian (make_tetra_points keeps it contiguous) or
    of its index neighbour -- so that tets are small and the gather locality resembles a Delaunay mesh of the same size.
    int64 [n_tets, 4], generated on `device`."""
    g = torch.Generator(device=device).manual_seed(int(seed))
    a = torch.randint(0, int(n_points), (int(n_tets),), generator=g, device=device)
    o1 = torch.randint(1, 4, (int(n_tets),), generator=g, device=device)
    o2 = torch.randint(4, 10, (int(n_tets),), generator=g, device=device)
    o3 = torch.randint(10, 18, (int(n_tets),), generator=g, device=device)
    return torch.stack([a, (a + o1) % n_points, (a + o2) % n_points, (a + o3) % n_points], dim=1).contiguous()


def make_scene(name_or_cfg, view=0, device="cpu", **overrides):
    cfg = dict(CONFIGS[name_or_cfg]) if isinstance(name_or_cfg, str) else dict(name_or_cfg)
    cfg.update(overrides)
    cam = make_camera(cfg["width"], cfg["height"], view=view)
    gs = make_gaussians(cfg["P"], cfg["seed"], cam.focal_x, sh_degree=cfg.get("sh_degree", 3),
                        sigma_px=cfg.get("sigma_px", 2.0))
    if device != "cpu":
        gs = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    return cam, gs


def raster_settings(cam, sh_degree, device, kernel_size=0.0, scale_modifier=1.0, bg=(0.0, 0.0, 0.0), debug=False,
                    settings_cls=None):
    """GaussianRasterizationSettings exactly as gaussian_renderer/__init__.py:39-54 fills it."""
    if settings_cls is None:
        from diff_gaussian_rasterization import GaussianRasterizationSettings as settings_cls
    return settings_cls(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx,
        tanfovy=cam.tanfovy, kernel_size=kernel_size,
        subpixel_offset=torch.zeros((cam.image_height, cam.image_width, 2), dtype=torch.float32, device=device),
        bg=torch.tensor(bg, dtype=torch.float32, device=device), scale_modifier=scale_modifier,
        viewmatrix=cam.world_view_transform.to(device), projmatrix=cam.full_proj_transform.to(device),
        sh_degree=sh_degree, campos=cam.camera_center.to(device), prefiltered=False, debug=debug)
