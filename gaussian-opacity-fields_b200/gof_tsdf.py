"""TSDF mesh extraction on the GPU -- the path of the reference's extract_mesh_tsdf.py:16-83 without Open3D.

    vol = TSDFVolume(voxel_size=0.002)                  # VoxelBlockGrid(('tsdf','weight','color'), block_resolution=16, ...)
    vol.integrate(depth, rgb, fx, fy, cx, cy, extrinsic, depth_max=6.0)   # compute_unique_block_coordinates + integrate
    mesh = vol.extract_triangle_mesh(weight_threshold=3.0)                # {'vertices', 'faces', 'colors'}
    write_ply(path, mesh)

or the whole loop at once: `write_ply(path, tsdf_fusion(views, make_render_fn(...)))`.  The arithmetic, the block layout
and the canonical output order are specified in DESIGN section 4.4; csrc/tsdf.cu implements it through libgof_b200.so.
CUDA tensors only.
"""
import ctypes

import numpy as np
import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib
_fp = ctypes.c_void_p
_i64p = ctypes.POINTER(ctypes.c_int64)


class _Params(ctypes.Structure):
    _fields_ = [("voxel_size", ctypes.c_float), ("block_resolution", ctypes.c_int), ("trunc", ctypes.c_float),
                ("depth_max", ctypes.c_float)]


class _Camera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("extrinsic", ctypes.c_float * 12)]


_P, _Cm = ctypes.POINTER(_Params), ctypes.POINTER(_Camera)
for _name, _args in (
        ("gof_tsdf_touch_count", [_P, _Cm, _fp, _C._ALLOC_FN, _fp, _i64p, _fp]),
        ("gof_tsdf_touch_emit", [_P, _Cm, _fp, ctypes.c_int64, _fp, _fp]),
        ("gof_tsdf_activate_count", [ctypes.c_int64, _fp, ctypes.c_int64, _fp, _C._ALLOC_FN, _fp, _i64p, _fp]),
        ("gof_tsdf_activate_emit", [ctypes.c_int64, _fp, _fp, ctypes.c_int64, _fp, _fp, ctypes.c_int64, _fp, _fp, _fp, _fp]),
        ("gof_tsdf_integrate", [_P, _Cm, _fp, _fp, ctypes.c_int64, _fp, _fp, _fp, _fp, _fp]),
        ("gof_tsdf_extract_count", [_P, ctypes.c_int64, _fp, _fp, _fp, ctypes.c_float, _C._ALLOC_FN, _fp, _i64p, _i64p, _fp]),
        ("gof_tsdf_extract_emit", [_P, ctypes.c_int64, _fp, _fp, _fp, ctypes.c_float, _fp, ctypes.c_int64, ctypes.c_int64,
                                   _fp, _fp, _fp, _fp])):
    getattr(_lib, _name).restype = ctypes.c_int
    getattr(_lib, _name).argtypes = _args

PLANES = 5   # tsdf, weight, r, g, b per block


def _f32(x):
    return float(np.float32(x))


def _ptr(t):
    return t.data_ptr() if t.numel() else None


def intrinsics_from_view(view):
    """(fx, fy, cx, cy) as the reference computes them (extract_mesh_tsdf.py:50-55):
    intrins = (view.projection_matrix @ ndc2pix)[:3,:3].T, i.e. fx = W/2 * P00, cx = (W-1)/2 and likewise for y.  Every other
    term of the product is a product with zero, so the result is exact on any matmul path."""
    W, H = int(view.image_width), int(view.image_height)
    P = view.projection_matrix.detach().to("cpu", torch.float32)
    fx = np.float32(np.float32(W / 2) * np.float32(P[0, 0].item()))
    fy = np.float32(np.float32(H / 2) * np.float32(P[1, 1].item()))
    return float(fx), float(fy), float(np.float32((W - 1) / 2)), float(np.float32((H - 1) / 2))


def extrinsic_from_view(view):
    """world -> camera [R|t] (4x4 float32, CPU): the reference's world_view_transform.T."""
    return view.world_view_transform.detach().to("cpu", torch.float32).t().contiguous()


class TSDFVolume:
    """Sparse TSDF volume of voxel blocks (Open3D's VoxelBlockGrid with attributes tsdf, weight, color, as the reference
    configures it).  `block_count` is the initial capacity of the voxel pool, which grows as blocks are added."""

    def __init__(self, voxel_size=0.002, block_resolution=16, trunc_voxel_multiplier=8.0, block_count=50000, device=None):
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != "cuda":
            raise RuntimeError("gof_b200 TSDFVolume: a CUDA device is required (no CPU path)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        B = int(block_resolution)
        if not (1 <= B <= 64) or not voxel_size > 0 or not trunc_voxel_multiplier > 0:
            raise ValueError("TSDFVolume: voxel_size > 0, trunc_voxel_multiplier > 0 and block_resolution in 1..64 required")
        self.device = dev
        self.voxel_size = _f32(voxel_size)
        self.block_resolution = B
        self.trunc = _f32(np.float32(trunc_voxel_multiplier) * np.float32(voxel_size))
        self.keys = torch.zeros(0, dtype=torch.int64, device=dev)       # sorted block keys
        self.slots = torch.zeros(0, dtype=torch.int32, device=dev)      # pool slot of each key
        self.pool = torch.zeros((max(int(block_count), 1), PLANES, B ** 3), dtype=torch.float32, device=dev)
        self.num_updates = torch.zeros(1, dtype=torch.int64, device=dev)   # voxel updates so far

    @property
    def num_blocks(self):
        return int(self.keys.numel())

    def _params(self, depth_max=6.0):
        return _Params(self.voxel_size, self.block_resolution, self.trunc, _f32(depth_max))

    def _check_image(self, t, shape, name):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f"gof_b200 TSDFVolume: {name} must be a CUDA tensor (no CPU path)")
        if t.device != self.device:
            raise RuntimeError(f"gof_b200 TSDFVolume: {name} on {t.device}, volume on {self.device}")
        if t.dtype != torch.float32 or tuple(t.shape) != shape:
            raise ValueError(f"TSDFVolume: {name} must be float32 {shape}, got {t.dtype} {tuple(t.shape)}")
        return t.contiguous()

    def _grow(self, needed):
        cap = self.pool.shape[0]
        if needed <= cap:
            return
        new = torch.zeros((max(needed, 2 * cap),) + tuple(self.pool.shape[1:]), dtype=torch.float32, device=self.device)
        new[:self.num_blocks] = self.pool[:self.num_blocks]      # slots 0..n-1 are in use; the rest stay zero
        self.pool = new

    def _camera(self, H, W, fx, fy, cx, cy, extrinsic):
        E = torch.as_tensor(np.asarray(extrinsic.detach().cpu() if isinstance(extrinsic, torch.Tensor) else extrinsic, np.float32))
        if tuple(E.shape) not in ((3, 4), (4, 4)):
            raise ValueError("TSDFVolume: extrinsic must be a [4,4] or [3,4] world->camera transform")
        cam = _Camera(int(W), int(H), _f32(fx), _f32(fy), _f32(cx), _f32(cy))
        for i, x in enumerate(E[:3, :4].reshape(-1).tolist()):
            cam.extrinsic[i] = x
        return cam

    def _touch(self, depth, cam, par):
        scratch = _C._Scratch(self.device, "tsdf_touch")
        n = ctypes.c_int64(0)
        with torch.cuda.device(self.device):
            _C._check(_lib.gof_tsdf_touch_count(ctypes.byref(par), ctypes.byref(cam), depth.data_ptr(), scratch.cb, None,
                                                ctypes.byref(n), _C._stream()))
            keys = torch.empty(n.value, dtype=torch.int64, device=self.device)
            if n.value:
                _C._check(_lib.gof_tsdf_touch_emit(ctypes.byref(par), ctypes.byref(cam), scratch.tensor.data_ptr(), n.value,
                                                   keys.data_ptr(), _C._stream()))
        return keys

    def _activate(self, view_keys):
        nt, nv = self.num_blocks, int(view_keys.numel())
        scratch = _C._Scratch(self.device, "tsdf_activate")
        n_new = ctypes.c_int64(0)
        with torch.cuda.device(self.device):
            _C._check(_lib.gof_tsdf_activate_count(nt, _ptr(self.keys), nv, view_keys.data_ptr(), scratch.cb, None,
                                                   ctypes.byref(n_new), _C._stream()))
            self._grow(nt + n_new.value)
            keys = torch.empty(nt + n_new.value, dtype=torch.int64, device=self.device)
            slots = torch.empty(nt + n_new.value, dtype=torch.int32, device=self.device)
            view_slots = torch.empty(nv, dtype=torch.int32, device=self.device)
            _C._check(_lib.gof_tsdf_activate_emit(nt, _ptr(self.keys), _ptr(self.slots), nv, view_keys.data_ptr(),
                                                  scratch.tensor.data_ptr(), n_new.value, keys.data_ptr(), slots.data_ptr(),
                                                  view_slots.data_ptr(), _C._stream()))
        self.keys, self.slots = keys, slots
        return view_slots

    def integrate(self, depth, color, fx, fy, cx, cy, extrinsic, depth_max=6.0):
        """Fuses one view: depth [H,W] (or [1,H,W]) float32, 0 = no depth; color [3,H,W] float32; pinhole intrinsics;
        extrinsic = world->camera [R|t] (the reference's world_view_transform.T).  Returns the view's block keys."""
        if isinstance(depth, torch.Tensor) and depth.dim() == 3 and depth.shape[0] == 1:
            depth = depth[0]
        if not isinstance(depth, torch.Tensor) or depth.dim() != 2:
            raise ValueError("TSDFVolume: depth must be a [H,W] (or [1,H,W]) tensor")
        H, W = depth.shape
        depth = self._check_image(depth, (H, W), "depth")
        color = self._check_image(color, (3, H, W), "color")
        cam = self._camera(H, W, fx, fy, cx, cy, extrinsic)
        par = self._params(depth_max)
        view_keys = self._touch(depth, cam, par)
        if view_keys.numel() == 0:
            return view_keys
        view_slots = self._activate(view_keys)
        with torch.cuda.device(self.device):
            _C._check(_lib.gof_tsdf_integrate(ctypes.byref(par), ctypes.byref(cam), depth.data_ptr(), color.data_ptr(),
                                              int(view_keys.numel()), view_keys.data_ptr(), view_slots.data_ptr(),
                                              self.pool.data_ptr(), self.num_updates.data_ptr(), _C._stream()))
        return view_keys

    def extract_triangle_mesh(self, weight_threshold=3.0):
        """Marching cubes: dict(vertices [V,3] float32, faces [F,3] int64, colors [V,3] float32) in canonical order."""
        par = self._params()
        n = self.num_blocks
        scratch = _C._Scratch(self.device)
        nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
        th = _f32(weight_threshold)
        with torch.cuda.device(self.device):
            _C._check(_lib.gof_tsdf_extract_count(ctypes.byref(par), n, _ptr(self.keys), _ptr(self.slots), self.pool.data_ptr(), th,
                                                  scratch.cb, None, ctypes.byref(nv), ctypes.byref(nf), _C._stream()))
            V, F = nv.value, nf.value
            out = {"vertices": torch.empty((V, 3), dtype=torch.float32, device=self.device),
                   "faces": torch.empty((F, 3), dtype=torch.int64, device=self.device),
                   "colors": torch.empty((V, 3), dtype=torch.float32, device=self.device)}
            if V or F:
                _C._check(_lib.gof_tsdf_extract_emit(ctypes.byref(par), n, _ptr(self.keys), _ptr(self.slots), self.pool.data_ptr(),
                                                     th, scratch.tensor.data_ptr(), V, F, _ptr(out["vertices"]),
                                                     _ptr(out["colors"]), _ptr(out["faces"]), _C._stream()))
        return out

    def state(self):
        """Sorted block keys [n] and, per block in that order, tsdf [n,B^3], weight [n,B^3], color [n,3,B^3] (voxel i + B j + B^2 k)."""
        s = self.slots.long()
        blk = self.pool[s]
        return {"keys": self.keys.clone(), "tsdf": blk[:, 0].clone(), "weight": blk[:, 1].clone(), "color": blk[:, 2:5].clone()}


def make_render_fn(means3D, opacities, scales, rotations, shs, sh_degree, settings_for_view):
    """settings_for_view(view) -> GaussianRasterizationSettings (which carries sh_degree, as in gof_extract.make_integrate_fn).
    Returns render_fn(view) -> the rasterizer's 9-channel image, for tsdf_fusion."""
    from diff_gaussian_rasterization import GaussianRasterizer

    def fn(view):
        rs = settings_for_view(view)
        color, _ = GaussianRasterizer(rs)(means3D=means3D, means2D=torch.zeros_like(means3D), opacities=opacities, shs=shs,
                                          scales=scales, rotations=rotations)
        return color
    return fn


def tsdf_fusion(views, render_fn, alpha_thres=0.5, voxel_size=0.002, depth_max=6.0, weight_threshold=3.0, block_resolution=16,
                trunc_voxel_multiplier=8.0, block_count=50000, device=None):
    """extract_mesh_tsdf.py:35-80: render every view, zero the median depth (channel 6) where the view's gt_alpha_mask is
    below 0.5 and where alpha (channel 7) is below alpha_thres, fuse depth and colour (channels 0-2), extract the mesh."""
    vol = None
    with torch.no_grad():
        for view in views:
            rendering = render_fn(view)
            if vol is None:
                vol = TSDFVolume(voxel_size, block_resolution, trunc_voxel_multiplier, block_count,
                                 device=device if device is not None else rendering.device)
            depth = rendering[6].clone()
            alpha = rendering[7]
            mask = getattr(view, "gt_alpha_mask", None)
            if mask is not None:
                depth[mask.to(depth.device).reshape(depth.shape) < 0.5] = 0
            depth[alpha < alpha_thres] = 0
            fx, fy, cx, cy = intrinsics_from_view(view)
            vol.integrate(depth, rendering[:3].contiguous(), fx, fy, cx, cy, extrinsic_from_view(view), depth_max=depth_max)
    if vol is None:
        raise ValueError("tsdf_fusion: no views")
    return vol.extract_triangle_mesh(weight_threshold)


def write_ply(path, mesh):
    """Binary little-endian PLY: float x y z, then float nx ny nz when the mesh has "normals" (not None), uchar red green blue
    (colour * 255 clipped to [0, 255] and truncated), int32 vertex_indices lists -- what evaluate_dtu_mesh.py loads."""
    v = np.ascontiguousarray(torch.as_tensor(mesh["vertices"]).detach().cpu().numpy(), np.float32)
    f = np.ascontiguousarray(torch.as_tensor(mesh["faces"]).detach().cpu().numpy()).astype(np.int32)
    c = torch.as_tensor(mesh["colors"]).detach().cpu().numpy().astype(np.float32)
    rgb = np.clip(c * np.float32(255.0), 0, 255).astype(np.uint8)
    normals = mesh.get("normals")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if normals is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    vert = np.empty(v.shape[0], dtype=fields + [("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    if normals is not None:
        n = torch.as_tensor(normals).detach().cpu().numpy().astype(np.float32)
        vert["nx"], vert["ny"], vert["nz"] = n[:, 0], n[:, 1], n[:, 2]
    vert["red"], vert["green"], vert["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    face = np.empty(f.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    face["n"] = 3
    face["i"] = f
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
              + ("property float nx\nproperty float ny\nproperty float nz\n" if normals is not None else "")
              + "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())


def read_ply(path):
    """Reads back what write_ply writes: dict(vertices [V,3] float32, colors_u8 [V,3] uint8, faces [F,3] int64), and
    normals [V,3] float32 when the header declares nx ny nz."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    nv = int(next(ln for ln in lines if ln.startswith("element vertex")).split()[-1])
    nf = int(next(ln for ln in lines if ln.startswith("element face")).split()[-1])
    has_normals = "property float nx" in lines
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if has_normals:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    vdt = np.dtype(fields + [("red", "u1"), ("green", "u1"), ("blue", "u1")])
    fdt = np.dtype([("n", "u1"), ("i", "<i4", (3,))])
    vert = np.frombuffer(data, vdt, nv, end)
    face = np.frombuffer(data, fdt, nf, end + nv * vdt.itemsize)
    if nf and not np.all(face["n"] == 3):
        raise ValueError("read_ply: only triangles are supported")
    out = {"vertices": np.stack([vert["x"], vert["y"], vert["z"]], 1),
           "colors_u8": np.stack([vert["red"], vert["green"], vert["blue"]], 1),
           "faces": face["i"].astype(np.int64).reshape(-1, 3)}
    if has_normals:
        out["normals"] = np.stack([vert["nx"], vert["ny"], vert["nz"]], 1)
    return out
