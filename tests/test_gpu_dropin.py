"""GPU: the drop-in proof.  The reference's UNMODIFIED `gaussian_renderer.render()` / `.integrate()`
(gaussian_renderer/__init__.py:18-115, 118-218; staged by baseline/stage_ref.sh, loaded by tests/_refpy.py) is executed
twice on the same model and camera: once importing THIS repo's `diff_gaussian_rasterization`, once importing the reference's
own package on top of its compiled extension (oracle/_ref).  Images, radii, visibility and every parameter gradient that
render() exposes must agree.  Skipped when the staged reference files are absent."""
import math
import types

import pytest
import torch

import _refpy
import _util
import gof_synth

pytestmark = pytest.mark.gpu


class StubGaussianModel:
    """Minimal stand-in for scene/gaussian_model.py::GaussianModel: exactly the attributes render()/integrate() read.
    `get_view2gaussian` is the reference's own method text (scene/gaussian_model.py:202-260), bound below."""

    def __init__(self, gs, dev):
        self.max_sh_degree = 3
        self.active_sh_degree = int(gs["sh_degree"])
        self._xyz = gs["means3D"].to(dev).requires_grad_(True)
        self._scales = gs["scales"].to(dev).requires_grad_(True)
        self._rotation = gs["rotations"].to(dev).requires_grad_(True)
        self._opacity = gs["opacities"].to(dev).requires_grad_(True)
        self._features = gs["shs"].to(dev).requires_grad_(True)

    get_xyz = property(lambda s: s._xyz)
    get_opacity_with_3D_filter = property(lambda s: s._opacity)
    get_scaling_with_3D_filter = property(lambda s: s._scales)
    get_rotation = property(lambda s: s._rotation)
    get_features = property(lambda s: s._features)

    def params(self):
        return {"xyz": self._xyz, "scales": self._scales, "rotation": self._rotation, "opacity": self._opacity, "features": self._features}


def _camera(cam, dev):
    return types.SimpleNamespace(FoVx=2.0 * math.atan(cam.tanfovx), FoVy=2.0 * math.atan(cam.tanfovy), image_height=cam.image_height,
                                 image_width=cam.image_width, world_view_transform=cam.world_view_transform.to(dev),
                                 full_proj_transform=cam.full_proj_transform.to(dev), camera_center=cam.camera_center.to(dev))


@pytest.fixture(scope="module")
def renderers():
    import diff_gaussian_rasterization as ours
    refpkg = _refpy.ref_rasterizer_package()
    if refpkg is None:
        pytest.skip("the original project's Python (baseline/stage_ref.sh) or its extension (oracle/_ref) is not staged")
    a, b = _refpy.ref_gaussian_renderer(ours, "gof_gr_on_ours"), _refpy.ref_gaussian_renderer(refpkg, "gof_gr_on_ref")
    assert a.GaussianRasterizer is ours.GaussianRasterizer and b.GaussianRasterizer is refpkg.GaussianRasterizer
    src = _refpy.ref_method_source("gaussian_model.py", "GaussianModel", "get_view2gaussian")
    glb = {"torch": torch}
    exec(src, glb)
    StubGaussianModel.get_view2gaussian = glb["get_view2gaussian"]
    return a, b


PIPES = {
    "default": dict(debug=False, compute_cov3D_python=False, compute_view2gaussian_python=False, convert_SHs_python=False),
    "sh_python": dict(debug=False, compute_cov3D_python=False, compute_view2gaussian_python=False, convert_SHs_python=True),
    "v2g_python": dict(debug=False, compute_cov3D_python=False, compute_view2gaussian_python=True, convert_SHs_python=False),
    "debug": dict(debug=True, compute_cov3D_python=False, compute_view2gaussian_python=False, convert_SHs_python=False),
}


@pytest.mark.parametrize("pipe_name", list(PIPES))
def test_reference_render_runs_on_this_package(renderers, pipe_name):
    on_ours, on_ref = renderers
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=60_000, width=640, height=416, seed=51), view=13)
    pipe = types.SimpleNamespace(**PIPES[pipe_name])
    vc = _camera(cam, dev)
    bg = torch.tensor([0.1, 0.3, 0.2], device=dev)
    grad = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(5)).to(dev)
    res = []
    for gr in (on_ours, on_ref, on_ref):       # the second reference run measures its own atomic-order noise
        pc = StubGaussianModel(gs, dev)
        pkg = gr.render(vc, pc, pipe, bg, kernel_size=0.1)
        (pkg["render"] * grad).sum().backward()
        torch.cuda.synchronize()
        res.append((pkg, {k: v.grad.clone() for k, v in pc.params().items()}, pkg["viewspace_points"].grad.clone()))
    (po, go, vo), (pr, gr1, vr1), (_p2, gr2, vr2) = res
    assert torch.equal(po["radii"], pr["radii"]) and torch.equal(po["visibility_filter"], pr["visibility_filter"])
    for ch in range(9):
        tol = 2e-5 if ch == 8 else 2e-6
        if pipe_name == "v2g_python":
            tol = 1e-4 if ch != 8 else 1e-3     # torch's own float matmuls feed both arms identically; rounding noise is larger
        assert _util.rel_err(po["render"][ch], pr["render"][ch])[0] < tol, f"channel {ch}"
    assert _util.rel_err(vo, vr1)[0] <= max(1e-4, 6 * _util.rel_err(vr2, vr1)[0])
    for k in go:
        j = 1 if k in ("xyz", "scales", "rotation") else 0      # noise-amplified gradients: relative L2 (see test_gpu_live_ref._grad_close)
        noise = _util.rel_err(gr2[k], gr1[k])[j]
        err = _util.rel_err(go[k], gr1[k])[j]
        assert err <= max(1e-4, (3.0 if j else 6.0) * noise), f"{pipe_name}/{k}: ours-vs-ref {err}, ref-vs-ref {noise}"


def test_reference_integrate_runs_on_this_package(renderers):
    on_ours, on_ref = renderers
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=60_000, width=640, height=416, seed=52), view=30)
    pipe = types.SimpleNamespace(**PIPES["default"])
    vc = _camera(cam, dev)
    bg = torch.zeros(3, device=dev)
    g = torch.Generator().manual_seed(7)
    pts = torch.cat([gs["means3D"][:30_000] + 0.01 * torch.randn(30_000, 3, generator=g), (torch.rand(30_000, 3, generator=g) * 2 - 1) * 1.7]).to(dev)
    outs = []
    with torch.no_grad():
        for gr in (on_ours, on_ref):
            outs.append(gr.integrate(pts, vc, StubGaussianModel(gs, dev), pipe, bg, kernel_size=0.0))
    o, r = outs
    assert torch.equal(o["radii"], r["radii"])
    assert float((o["alpha_integrated"] - r["alpha_integrated"]).abs().max()) < 5e-6
    assert _util.rel_err(o["color_integrated"], r["color_integrated"])[0] < 1e-5
    for ch in (0, 1, 2, 6, 7):
        assert _util.rel_err(o["render"][ch], r["render"][ch])[0] < 1e-5, f"channel {ch}"
    assert torch.equal(o["render"][8], r["render"][8])       # projected points per pixel
