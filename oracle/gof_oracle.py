"""ctypes binding of the CPU oracle (oracle/gof_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
All arrays are numpy, C-contiguous; layouts are the reference's (GeometryState etc.).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libgof_oracle.so")


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE, "libgof_oracle.so"])
    return _LIB


def _load():
    if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(os.path.join(_HERE, "gof_oracle.c")):
        build()
    return ctypes.CDLL(_LIB)


_lib = _load()
_f = ctypes.POINTER(ctypes.c_float)


class _Scene(ctypes.Structure):
    _fields_ = [("P", ctypes.c_int), ("D", ctypes.c_int), ("M", ctypes.c_int), ("W", ctypes.c_int), ("H", ctypes.c_int),
                ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float), ("kernel_size", ctypes.c_float),
                ("scale_modifier", ctypes.c_float)] + [(n, ctypes.c_void_p) for n in (
                    "background", "means3D", "shs", "colors_precomp", "opacities", "scales", "rotations",
                    "cov3D_precomp", "v2g_precomp", "viewmatrix", "projmatrix", "cam_pos")]


class _Geom(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("radii", "means2D", "depths", "cov3D", "view2gaussian", "rgb",
                                                 "conic_opacity", "tiles_touched", "clamped")]


_lib.oracle_bin.restype = ctypes.c_longlong
_lib.oracle_num_threads.restype = ctypes.c_int


def num_threads():
    return int(_lib.oracle_num_threads())


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _np(t, dtype=np.float32):
    if t is None:
        return None
    if hasattr(t, "detach"):
        if t.numel() == 0:
            return None
        t = t.detach().cpu().numpy()
    return np.ascontiguousarray(t, dtype=dtype)


class Scene:
    """Numpy-side view of one (camera, Gaussians) pair; mirrors gof_scene_t."""

    def __init__(self, W, H, tan_fovx, tan_fovy, viewmatrix, projmatrix, cam_pos, means3D, opacities, scales=None,
                 rotations=None, shs=None, colors_precomp=None, sh_degree=3, kernel_size=0.0, scale_modifier=1.0,
                 bg=(0.0, 0.0, 0.0), cov3D_precomp=None, v2g_precomp=None):
        self.W, self.H = int(W), int(H)
        self.tan_fovx, self.tan_fovy = float(tan_fovx), float(tan_fovy)
        self.kernel_size, self.scale_modifier = float(kernel_size), float(scale_modifier)
        self.D = int(sh_degree)
        self.arr = dict(background=_np(np.asarray(bg, dtype=np.float32) if not hasattr(bg, "detach") else bg),
                        means3D=_np(means3D), shs=_np(shs), colors_precomp=_np(colors_precomp),
                        opacities=_np(opacities), scales=_np(scales), rotations=_np(rotations),
                        cov3D_precomp=_np(cov3D_precomp), v2g_precomp=_np(v2g_precomp), viewmatrix=_np(viewmatrix),
                        projmatrix=_np(projmatrix), cam_pos=_np(cam_pos))
        self.P = int(self.arr["means3D"].shape[0])
        self.M = int(self.arr["shs"].shape[1]) if self.arr["shs"] is not None else 0

    def c(self):
        s = _Scene()
        s.P, s.D, s.M, s.W, s.H = self.P, self.D, self.M, self.W, self.H
        s.tan_fovx, s.tan_fovy, s.kernel_size, s.scale_modifier = self.tan_fovx, self.tan_fovy, self.kernel_size, self.scale_modifier
        for k, v in self.arr.items():
            setattr(s, k, _p(v))
        return s


def scene_from_synth(cam, gs, **kw):
    return Scene(cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, cam.world_view_transform,
                 cam.full_proj_transform, cam.camera_center, gs["means3D"], gs["opacities"], scales=gs["scales"],
                 rotations=gs["rotations"], shs=gs.get("shs"), sh_degree=gs.get("sh_degree", 3), **kw)


def preprocess(scene):
    P = scene.P
    g = dict(radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
             cov3D=np.zeros((P, 6), np.float32), view2gaussian=np.zeros((P, 10), np.float32),
             rgb=np.zeros((P, 3), np.float32), conic_opacity=np.zeros((P, 4), np.float32),
             tiles_touched=np.zeros(P, np.uint32), clamped=np.zeros((P, 3), np.uint8))
    if scene.arr["colors_precomp"] is not None:
        g["rgb"][:] = scene.arr["colors_precomp"]
    if scene.arr["v2g_precomp"] is not None:
        g["view2gaussian"][:] = scene.arr["v2g_precomp"]
    cg = _Geom()
    for k, v in g.items():
        setattr(cg, k, _p(v))
    cs = scene.c()
    _lib.oracle_preprocess(ctypes.byref(cs), ctypes.byref(cg))
    return g


def bin_tiles(W, H, radii, means2D, depths, tiles_touched):
    P = int(radii.shape[0])
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    R = int(np.asarray(tiles_touched, dtype=np.uint64).sum())
    point_list = np.zeros(max(R, 1), np.uint32)
    ranges = np.zeros((tiles, 2), np.uint32)
    r = _lib.oracle_bin(P, W, H, _p(np.ascontiguousarray(radii, np.int32)), _p(np.ascontiguousarray(means2D, np.float32)),
                        _p(np.ascontiguousarray(depths, np.float32)), _p(np.ascontiguousarray(tiles_touched, np.uint32)),
                        _p(point_list), _p(ranges), None)
    assert r == R
    return R, point_list[:R], ranges


def render_forward(scene, g, point_list, ranges, checked=False):
    """Blend forward: (out_color [9,H,W], final_T [4,H,W], n_contrib [2,H,W]).  checked=True appends a dict of the optional
    outputs of oracle_render_forward_checked: marginal_pix [H,W] bool, n_blended [H,W], blended [H,W,nwords] u32 (bit p:
    entry p of the pixel's tile list was blended) and accum_err [4,H,W] float64; the three arrays above are the same."""
    W, H = scene.W, scene.H
    out = np.zeros((9, H, W), np.float32)
    final_T = np.zeros((4, H, W), np.float32)
    n_contrib = np.zeros((2, H, W), np.uint32)
    args = (W, H, ctypes.c_float(scene.tan_fovx), ctypes.c_float(scene.tan_fovy),
            _p(np.ascontiguousarray(ranges, np.uint32)), _p(np.ascontiguousarray(point_list, np.uint32)),
            _p(np.ascontiguousarray(g["rgb"], np.float32)), _p(np.ascontiguousarray(g["view2gaussian"], np.float32)),
            _p(np.ascontiguousarray(g["conic_opacity"], np.float32)), _p(scene.arr["background"]), _p(out), _p(final_T), _p(n_contrib))
    if not checked:
        _lib.oracle_render_forward(*args)
        return out, final_T, n_contrib
    r = np.asarray(ranges, np.int64).reshape(-1, 2)
    nwords = max(1, int(((r[:, 1] - r[:, 0]).max(initial=0) + 31) // 32))
    ex = dict(marginal_pix=np.zeros((H, W), np.uint8), n_blended=np.zeros((H, W), np.uint32),
              blended=np.zeros((H, W, nwords), np.uint32), accum_err=np.zeros((4, H, W), np.float64))
    _lib.oracle_render_forward_checked(*args, _p(ex["marginal_pix"]), _p(ex["n_blended"]), _p(ex["blended"]), nwords, _p(ex["accum_err"]))
    ex["marginal_pix"] = ex["marginal_pix"].astype(bool)
    return out, final_T, n_contrib, ex


BOUND_COMPONENTS = 17   # columns of `mag` / `marginal`: dL_dcolors 0-2 | dL_dmean2D 3-5 | dL_dopacity 6 | dL_dv2g 7-16


def render_backward(scene, g, point_list, ranges, final_T, n_contrib, dL_dpix, bounds=False):
    """Blend backward from a given forward state.  bounds=True adds the error scales "mag" and "marginal", [P,17] float64
    each (see oracle_render_backward); the gradients are the same either way."""
    P, W, H = scene.P, scene.W, scene.H
    d = dict(dL_dmean2D=np.zeros((P, 3), np.float32), dL_dopacity=np.zeros((P, 1), np.float32),
             dL_dcolors=np.zeros((P, 3), np.float32), dL_dv2g=np.zeros((P, 10), np.float32))
    if bounds:
        d.update(mag=np.zeros((P, BOUND_COMPONENTS), np.float64), marginal=np.zeros((P, BOUND_COMPONENTS), np.float64))
    _lib.oracle_render_backward(P, W, H, ctypes.c_float(scene.tan_fovx), ctypes.c_float(scene.tan_fovy),
                                _p(np.ascontiguousarray(ranges, np.uint32)), _p(np.ascontiguousarray(point_list, np.uint32)),
                                _p(scene.arr["background"]), _p(np.ascontiguousarray(g["means2D"], np.float32)),
                                _p(np.ascontiguousarray(g["conic_opacity"], np.float32)), _p(np.ascontiguousarray(g["rgb"], np.float32)),
                                _p(np.ascontiguousarray(g["view2gaussian"], np.float32)), _p(np.ascontiguousarray(final_T, np.float32)),
                                _p(np.ascontiguousarray(n_contrib, np.uint32)), _p(np.ascontiguousarray(dL_dpix, np.float32)),
                                _p(d["dL_dmean2D"]), _p(d["dL_dopacity"]), _p(d["dL_dcolors"]), _p(d["dL_dv2g"]),
                                _p(d.get("mag")), _p(d.get("marginal")))
    return d


def preprocess_backward(scene, radii, clamped, dL_dcolor, dL_dv2g):
    P, M = scene.P, scene.M
    d = dict(dL_dmean3D=np.zeros((P, 3), np.float32), dL_dsh=np.zeros((P, M, 3), np.float32),
             dL_dscale=np.zeros((P, 3), np.float32), dL_drot=np.zeros((P, 4), np.float32))
    cs = scene.c()
    _lib.oracle_preprocess_backward(ctypes.byref(cs), _p(np.ascontiguousarray(radii, np.int32)),
                                    _p(np.ascontiguousarray(clamped, np.uint8)), _p(np.ascontiguousarray(dL_dcolor, np.float32)),
                                    _p(np.ascontiguousarray(dL_dv2g, np.float32)), _p(d["dL_dmean3D"]), _p(d["dL_dsh"]),
                                    _p(d["dL_dscale"]), _p(d["dL_drot"]))
    return d


def forward(scene, checked=False):
    """Full forward: (out_color, radii, state dict with every intermediate).  checked=True adds the optional outputs of
    render_forward(checked=True) to the state."""
    g = preprocess(scene)
    R, point_list, ranges = bin_tiles(scene.W, scene.H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    res = render_forward(scene, g, point_list, ranges, checked=checked)
    out, final_T, n_contrib = res[:3]
    st = dict(g)
    st.update(num_rendered=R, point_list=point_list, ranges=ranges, accum_alpha=final_T, n_contrib=n_contrib)
    if checked:
        st.update(res[3])
    return out, g["radii"], st


def backward(scene, st, dL_dpix):
    g = {k: st[k] for k in ("radii", "means2D", "depths", "cov3D", "view2gaussian", "rgb", "conic_opacity", "tiles_touched", "clamped")}
    d = render_backward(scene, g, st["point_list"], st["ranges"], st["accum_alpha"], st["n_contrib"], dL_dpix)
    d2 = preprocess_backward(scene, st["radii"], st["clamped"], d["dL_dcolors"], d["dL_dv2g"])
    d.update(d2)
    return d


def mark_visible(means3D, viewmatrix):
    m = _np(means3D)
    out = np.zeros(m.shape[0], np.uint8)
    _lib.oracle_mark_visible(int(m.shape[0]), _p(m), _p(_np(viewmatrix)), _p(out))
    return out.astype(bool)


def alpha_map(W, H, tan_fovx, tan_fovy, v2g, opacity):
    out = np.zeros((H, W), np.float32)
    v = np.ascontiguousarray(v2g, np.float32)
    _lib.oracle_alpha_map(int(W), int(H), ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), _p(v), ctypes.c_float(float(opacity)), _p(out))
    return out


def ray_mask_map(W, H, tan_fovx, tan_fovy, v2g, opacity):
    """[H,W] uint8: bit k set where ray k of the opacity-field query (0 centre, 1-4 corners) accepts the Gaussian."""
    out = np.zeros((H, W), np.uint8)
    v = np.ascontiguousarray(v2g, np.float32)
    _lib.oracle_ray_mask_map(int(W), int(H), ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), _p(v), ctypes.c_float(float(opacity)), _p(out))
    return out


def project_points(scene, points3D):
    """The query's projection of points3D [PN,3]: (xy [PN,2], depth [PN], ok [PN] bool); xy / depth are NaN where the point
    does not project into the image."""
    pts = _np(points3D)
    PN = int(pts.shape[0])
    xy, depth, ok = np.full((PN, 2), np.nan, np.float32), np.full(PN, np.nan, np.float32), np.zeros(PN, np.uint8)
    _lib.oracle_project_points(scene.W, scene.H, ctypes.c_float(scene.tan_fovx), ctypes.c_float(scene.tan_fovy),
                               _p(scene.arr["viewmatrix"]), PN, _p(pts), _p(xy), _p(depth), _p(ok))
    return xy, depth, ok.astype(bool)


def integrate(scene, points3D):
    """Opacity-field query of `points3D` [PN,3] for one view: (out_color[9,H,W], alpha_integrated[PN],
    color_integrated[PN,3], radii[P], state) -- the 4 tensors GaussianRasterizer.integrate returns, plus state.  The state
    also holds n_recorded [H,W], marginal_pix [H,W], marginal_pt [PN] and pt_clamp [PN,2] (see oracle_integrate)."""
    g = preprocess(scene)
    R, point_list, ranges = bin_tiles(scene.W, scene.H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    pts = _np(points3D)
    PN = int(pts.shape[0])
    W, H = scene.W, scene.H
    out = np.zeros((9, H, W), np.float32)
    final_T = np.zeros((H, W), np.float32)
    n_contrib = np.zeros((H, W), np.uint32)
    alpha_int = np.ones(PN, np.float32)
    color_int = np.zeros((PN, 3), np.float32)
    n_recorded = np.zeros((H, W), np.uint32)
    marginal_pix, marginal_pt = np.zeros((H, W), np.uint8), np.zeros(PN, np.uint8)
    pt_clamp = np.zeros((PN, 2), np.uint32)
    if scene.P and PN:
        _lib.oracle_integrate_checked(W, H, ctypes.c_float(scene.tan_fovx), ctypes.c_float(scene.tan_fovy), _p(scene.arr["viewmatrix"]),
                                      PN, _p(pts), _p(np.ascontiguousarray(ranges, np.uint32)), _p(np.ascontiguousarray(point_list, np.uint32)),
                                      _p(np.ascontiguousarray(g["rgb"], np.float32)), _p(np.ascontiguousarray(g["view2gaussian"], np.float32)),
                                      _p(np.ascontiguousarray(g["conic_opacity"], np.float32)), _p(scene.arr["background"]), _p(out),
                                      _p(final_T), _p(n_contrib), _p(alpha_int), _p(color_int), _p(n_recorded), _p(marginal_pix),
                                      _p(marginal_pt), _p(pt_clamp))
    st = dict(g)
    st.update(num_rendered=R, point_list=point_list, ranges=ranges, final_T=final_T, n_contrib=n_contrib,
              n_recorded=n_recorded, marginal_pix=marginal_pix.astype(bool), marginal_pt=marginal_pt.astype(bool),
              pt_clamp=pt_clamp)
    return out, alpha_int, color_int, g["radii"], st
