"""GPU: the callers of the opacity-field query (SURVEY 8(a) rows a24-a26, 8(f) rank 3) at extract_mesh.py's structure.

* CachedIntegrator (Gaussian side prepared once per view) is bit-identical to GaussianRasterizer.integrate;
* gof_extract.evaluate_alpha equals the reference's OWN `evaluage_alpha` (extract_mesh.py:17-34) driving the reference's
  gaussian_renderer.integrate on the reference's compiled rasterizer, and the 8-step bisection (extract_mesh.py:88-102) on
  top of either gives the same mesh vertices -- the reference's side stored in tests/golden/extract_ref.npz
  (tests/golden/make_golden_ref_python.py);
* tet-sharded marching tetrahedra (shards run one after the other on this GPU, merged as the ranks would) equals the unsharded call;
* extract_level_set end to end on an analytic blob."""
import math
import types

import numpy as np
import pytest
import torch

import _liveref
import gof_extract
import gof_synth

pytestmark = pytest.mark.gpu


def _scene(P=40_000, W=480, H=320, seed=61, n_views=6):
    dev = torch.device("cuda")
    cams = [gof_synth.make_scene(dict(P=P, width=W, height=H, seed=seed), view=v * 9)[0] for v in range(n_views)]
    gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=seed), view=0)[1]
    g = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    return dev, cams, gs, g


def _settings_for(dev):
    def f(cam):
        return gof_synth.raster_settings(cam, 3, dev)
    return f


def _points(gs, n, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, gs["means3D"].shape[0], (n,), generator=gen)
    return (gs["means3D"][idx] + gs["scales"][idx] * 3.0 * (torch.rand(n, 3, generator=gen) * 2 - 1)).contiguous().to(dev)


def test_cached_integrator_is_bit_identical_to_integrate():
    from diff_gaussian_rasterization import GaussianRasterizer
    dev, cams, gs, g = _scene()
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3, _settings_for(dev))
    for seed in (1, 2):                       # second point set: the cache is reused
        pts = _points(gs, 150_000 + seed, seed, dev)
        for cam in cams[:3]:
            a, c = ci(pts, cam)
            rs = gof_synth.raster_settings(cam, 3, dev)
            _img, a0, c0, _r = GaussianRasterizer(rs).integrate(points3D=pts, means3D=g["means3D"], means2D=torch.zeros_like(g["means3D"]),
                                                                opacities=g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
            assert torch.equal(a, a0) and torch.equal(c, c0)
    assert len(ci._cache) == 3 and ci.cached_bytes > 0


class _Stub:
    def __init__(self, g):
        self.max_sh_degree = self.active_sh_degree = 3
        self.g = g
    get_xyz = property(lambda s: s.g["means3D"])
    get_opacity_with_3D_filter = property(lambda s: s.g["opacities"])
    get_scaling_with_3D_filter = property(lambda s: s.g["scales"])
    get_rotation = property(lambda s: s.g["rotations"])
    get_features = property(lambda s: s.g["shs"])


def _ref_views(cams, dev):
    return [types.SimpleNamespace(FoVx=2.0 * math.atan(c.tanfovx), FoVy=2.0 * math.atan(c.tanfovy), image_height=c.image_height,
                                  image_width=c.image_width, world_view_transform=c.world_view_transform.to(dev),
                                  full_proj_transform=c.full_proj_transform.to(dev), camera_center=c.camera_center.to(dev)) for c in cams]


def extract_case():
    """Scene, query points and this package's alpha / colour of the evaluate_alpha comparison, and the bisection edges built
    from them (pairs of points inside / outside the 0.5 level set)."""
    dev, cams, gs, g = _scene()
    pts = _points(gs, 200_000, 5, dev)
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3, _settings_for(dev))
    alpha, color = gof_extract.evaluate_alpha(pts, cams, ci, return_color=True)
    inside, outside = torch.nonzero(alpha > 0.6).flatten()[:20_000], torch.nonzero(alpha < 0.4).flatten()[:20_000]
    n = min(inside.numel(), outside.numel())
    end_points = torch.stack([pts[inside[:n]], pts[outside[:n]]], dim=1)
    end_sdf = torch.stack([alpha[inside[:n]], alpha[outside[:n]]], dim=1)[..., None] - 0.5
    return dict(dev=dev, cams=cams, g=g, pts=pts, ci=ci, alpha=alpha, color=color, end_points=end_points, end_sdf=end_sdf)


def sample(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, min(n, k), replace=False))


def record(ref_eval):
    """The reference's side of test_evaluate_alpha_and_bisection_equal_the_reference_loop: `ref_eval` is its evaluage_alpha
    bound to its own gaussian_renderer.integrate on its compiled rasterizer."""
    c = extract_case()
    dev, g, end_points, end_sdf = c["dev"], c["g"], c["end_points"], c["end_sdf"]
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, compute_view2gaussian_python=False, convert_SHs_python=False)
    bg = torch.zeros(3, device=dev)
    rv = _ref_views(c["cams"], dev)
    ralpha, rcolor = ref_eval(c["pts"], rv, _Stub(g), pipe, bg, 0.0, return_color=True)
    # extract_mesh.py:73-102 with the reference's evaluage_alpha
    lp, rp = end_points[:, 0, :].clone(), end_points[:, 1, :].clone()
    ls, rs_ = end_sdf[:, 0, :].clone(), end_sdf[:, 1, :].clone()
    for _step in range(8):
        mid = (lp + rp) / 2
        msdf = (ref_eval(mid, rv, _Stub(g), pipe, bg, 0.0) - 0.5).squeeze().unsqueeze(-1)
        low = ((msdf < 0) & (ls < 0)) | ((msdf > 0) & (ls > 0))
        ls[low] = msdf[low]; rs_[~low] = msdf[~low]
        lp[low.flatten()] = mid[low.flatten()]; rp[~low.flatten()] = mid[~low.flatten()]
    want = (lp + rp) / 2
    ip = sample(ralpha.shape[0], 4096, 3)
    tp = torch.from_numpy(ip).to(dev)
    return {"end_points": _liveref.digest(end_points), "pt_rows": ip.astype(np.int32), "alpha": ralpha[tp].cpu().numpy(),
            "color": rcolor[tp].cpu().numpy(), "color_absmax": float(rcolor.abs().max()), "want": want.cpu().numpy()}


def test_evaluate_alpha_and_bisection_equal_the_reference_loop():
    """Against the stored reference results: alpha and colour on a seeded sample of the points, the bisection's end points on
    every edge.  As in test_integrate.py's 1080p comparison, the reference's sm_90a build rounds a few ray depths differently
    from the sm_100a build this implementation restates, so alpha is compared as the share of points that agree to 5e-6, with
    every sampled point within 0.02."""
    z = _liveref.load_npz("extract_ref.npz")
    c = extract_case()
    dev, cams, ci, alpha, color, end_points, end_sdf = c["dev"], c["cams"], c["ci"], c["alpha"], c["color"], c["end_points"], c["end_sdf"]
    assert _liveref.digest(end_points) == str(z["end_points"]) and end_points.shape[0] > 1000
    ip = torch.from_numpy(z["pt_rows"]).to(dev)
    a, ra = alpha[ip].cpu().double().numpy(), z["alpha"].astype(np.float64)
    assert np.mean(np.abs(a - ra) < 5e-6) > 0.995 and np.abs(a - ra).max() <= 0.02
    same = np.abs(a - ra) < 1e-7          # colour = the arg-min view's pixel colour: compare where the minima agree to the bit-ish
    assert same.mean() > 0.99
    got = color[ip].cpu().double().numpy()[same]
    assert np.abs(got - z["color"][same]).max() / max(float(z["color_absmax"]), 1e-30) < 1e-5
    assert torch.equal(gof_extract.evaluate_alpha(c["pts"], cams, ci), alpha)

    ours = gof_extract.binary_search(end_points, end_sdf, lambda p: gof_extract.evaluate_alpha(p, cams, ci))
    # a mid-point whose alpha sits within 5e-6 of 0.5 may take the other branch: such an edge ends at most one interval off
    d = (ours - torch.from_numpy(z["want"]).to(dev)).norm(dim=1)
    edge = (end_points[:, 0] - end_points[:, 1]).norm(dim=1)
    assert float((d <= 1e-6 * edge.clamp_min(1e-3)).float().mean()) > 0.999
    assert bool((d <= edge / 2 + 1e-6).all())


def test_tet_sharded_marching_tetrahedra_equals_unsharded():
    import gof_tetmesh
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(3)
    V, T, chunk = 60_000, 400_003, 50_000
    v = (torch.rand(V, 3, generator=gen) * 2 - 1)
    a = torch.randint(0, V, (T,), generator=gen)
    tets = torch.stack([a, (a + torch.randint(1, 50, (T,), generator=gen)) % V, (a + torch.randint(50, 400, (T,), generator=gen)) % V,
                        (a + torch.randint(400, 3000, (T,), generator=gen)) % V], dim=1)
    sdf = 0.8 - v.norm(dim=1) + 0.05 * torch.randn(V, generator=gen)
    sc = torch.rand(V, 1, generator=gen) * 0.1
    v, tets, sdf, sc = v.to(dev), tets.to(dev), sdf.to(dev), sc.to(dev)
    (pos0, sdf0), sc0, f0, iv0 = gof_tetmesh._unbatched_marching_tetrahedra(v, tets, sdf, sc, chunk_tets=chunk)
    rows = gof_tetmesh.chunk_rows(T, chunk)
    for world in (2, 3, 8):
        keys, faces = [], []
        for r in range(world):
            b, e = gof_extract.shard_tet_range(T, rows, r, world)
            if e > b:
                (_p, _s), _c, f, iv = gof_tetmesh._unbatched_marching_tetrahedra(v, tets[b:e], sdf, sc, rows=rows)
            else:
                f, iv = torch.zeros((0, 3), dtype=torch.long, device=dev), torch.zeros((0, 2), dtype=torch.long, device=dev)
            keys.append(gof_extract._edge_keys(iv)); faces.append(f)
        (pos, esdf), esc, f, iv = gof_extract.merge_tet_shards(v, sdf, sc, keys, faces)
        assert torch.equal(iv, iv0) and torch.equal(f, f0), world
        assert torch.equal(pos, pos0) and torch.equal(esdf, sdf0) and torch.equal(esc, sc0)


def test_extract_level_set_end_to_end():
    """A dense blob of Gaussians: the extracted vertices lie on the alpha = 0.5 surface of the min-over-views opacity field."""
    dev, cams, gs, g = _scene(P=30_000, W=320, H=240, seed=71, n_views=8)
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3, _settings_for(dev))
    gen = torch.Generator().manual_seed(9)
    pts = ((torch.rand(40_000, 3, generator=gen) * 2 - 1) * 1.8)
    V = pts.shape[0]
    a = torch.randint(0, V, (250_000,), generator=gen)
    tets = torch.stack([a, (a + 1) % V, (a + 7) % V, (a + 31) % V], dim=1).to(dev)
    pts = pts.to(dev)
    tm = {}
    out = gof_extract.extract_level_set(pts, torch.full((V, 1), 0.05, device=dev), tets, cams, ci, n_binary_steps=8, return_color=True,
                                        chunk_tets=100_000, timings=tm)
    assert out["faces"].numel() > 0 and out["vertices"].shape[0] == int(out["faces"].max()) + 1
    alpha = gof_extract.evaluate_alpha(out["vertices"], cams, ci)
    # after 8 halvings of edges that straddle the level set the opacity is close to 0.5 wherever the field is continuous along the edge
    assert float(((alpha - 0.5).abs() < 0.2).float().mean()) > 0.5
    assert out["colors"].shape == (out["vertices"].shape[0], 3) and out["mask"].dtype == torch.bool
    assert set(tm) >= {"evaluate_alpha_vertices_s", "marching_tetrahedra_s", "binary_search_s"}
