"""CPU: the argument checks and scratch query of gof_rasterize_backward_ex (the backward with its outputs in gof_backward_out_t:
the gradients, the densification statistics, the factored SH gradient, and the camera (DESIGN.md 4.9) and focal-length (DESIGN.md
4.10) gradients), through the built library.  Every case is decided before any device work, so no GPU is needed: the device
pointers are never dereferenced."""
import ctypes

import pytest

from diff_gaussian_rasterization import _C

FAKE = 256
W, H = 64, 48


def _fake_scene(P):
    """A scene whose pointers pass validation; the calls below fail before any of them is dereferenced."""
    s = _C._Scene()
    s.P, s.D, s.M, s.width, s.height = P, 3, 16, W, H
    s.tan_fovx = s.tan_fovy = 0.5
    s.scale_modifier = 1.0
    for n in ("background", "means3D", "shs", "opacities", "scales", "rotations", "viewmatrix", "projmatrix", "cam_pos"):
        setattr(s, n, FAKE)
    return s


def _scratch_bytes(P, width, height, camera, intrinsics):
    return int(_C._lib.gof_rasterize_backward_scratch_bytes(P, width, height, camera, intrinsics))


def _out(**kw):
    """The gradients every call needs, plus `kw` (field name -> pointer or None)."""
    o = dict(dL_dmean2D=FAKE, dL_dopacity=FAKE, dL_dcolor=FAKE, dL_dmean3D=FAKE, dL_dsh=FAKE, dL_dscale=FAKE, dL_drot=FAKE,
             dL_dview2gaussian=FAKE)
    o.update(kw)
    return _C._BackwardOut(**o)


def _camera(P=300, **kw):
    return _out(dL_dviewmatrix=FAKE, dL_dcampos=2 * FAKE, scratch=3 * FAKE, scratch_bytes=_scratch_bytes(P, W, H, 1, 0), **kw)


def _intrinsics(P=300, **kw):
    return _out(dL_dtan_fov=4 * FAKE, scratch=3 * FAKE, scratch_bytes=_scratch_bytes(P, W, H, 0, 1), **kw)


def _call(s, out, radii=FAKE):
    """gof_rasterize_backward_ex with num_rendered = 0 (so no binning buffer) and the forward state at FAKE."""
    rc = _C._lib.gof_rasterize_backward_ex(ctypes.byref(s), 0, radii, FAKE, None, FAKE, FAKE,
                                           None if out is None else ctypes.byref(out), None)
    return rc, _C._lib.gof_last_error()


def _positional(s, radii=FAKE, **kw):
    """The positional gof_rasterize_backward with the arguments of _call and _out's gradients, updated by `kw`."""
    lib = _C._lib
    lib.gof_rasterize_backward.restype = ctypes.c_int
    lib.gof_rasterize_backward.argtypes = [ctypes.POINTER(_C._Scene), ctypes.c_int] + [ctypes.c_void_p] * 16
    g = {n: getattr(_out(**kw), n) for n in ("dL_dmean2D", "dL_dopacity", "dL_dcolor", "dL_dmean3D", "dL_dsh", "dL_dscale", "dL_drot",
                                             "dL_dview2gaussian")}
    rc = lib.gof_rasterize_backward(ctypes.byref(s), 0, radii, FAKE, None, FAKE, FAKE, g["dL_dmean2D"], None, g["dL_dopacity"],
                                    g["dL_dcolor"], g["dL_dmean3D"], None, g["dL_dsh"], g["dL_dscale"], g["dL_drot"],
                                    g["dL_dview2gaussian"], None)
    return rc, lib.gof_last_error()


def test_backward_entry_points_are_exported():
    for name in ("gof_rasterize_backward", "gof_rasterize_backward_ex", "gof_rasterize_backward_scratch_bytes"):
        assert hasattr(_C._lib, name), name


@pytest.mark.parametrize("P,rows", [(-1, 0), (0, 0), (1, 1), (127, 1), (128, 1), (129, 2), (1_000_000, 7813)])
def test_camera_scratch_is_one_row_of_16_doubles_per_128_gaussians(P, rows):
    """The camera-only size does not depend on the image size; without a camera or focal-length gradient nothing is needed."""
    assert _scratch_bytes(P, W, H, 1, 0) == _scratch_bytes(P, 0, 0, 1, 0) == rows * 16 * 8
    assert _scratch_bytes(P, W, H, 0, 0) == 0


@pytest.mark.parametrize("P,W,H", [(-1, 64, 48), (0, 64, 48), (5, 0, 48), (5, 64, -1), (1, 16, 16), (129, 203, 117),
                                   (1_000_000, 1920, 1080)])
def test_intrinsics_scratch_is_16_bytes_per_pixel_plus_the_camera_rows(P, W, H):
    """The camera pass's rows (one row of 16 doubles per 128 Gaussians, padded to 256 bytes), then [2][H][W] doubles of dL/dr
    and [tiles][2] doubles of tile sums, with or without the camera gradient; zero when there is nothing to render."""
    got = _scratch_bytes(P, W, H, 0, 1)
    assert _scratch_bytes(P, W, H, 1, 1) == got
    if P <= 0 or W <= 0 or H <= 0:
        assert got == 0
        return
    cam = -(-((P + 127) // 128 * 128) // 256) * 256
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    assert got == cam + 16 * W * H + 16 * tiles


def test_null_out_is_refused():
    rc, _ = _call(_fake_scene(300), None)
    assert rc == -1


def test_missing_gradients_are_refused_with_or_without_camera_and_focal_length():
    """radii, dL_dmean2D or dL_dcolor missing: the plain call, the camera request, the focal-length request and the positional
    gof_rasterize_backward all fail with the same error."""
    s = _fake_scene(300)
    for missing in ("radii", "dL_dmean2D", "dL_dcolor"):
        field = {} if missing == "radii" else {missing: None}
        radii = None if missing == "radii" else FAKE
        for out in (_out(**field), _camera(**field), _intrinsics(**field)):
            assert _call(s, out, radii=radii) == (-1, b"backward: NULL argument"), missing
        assert _positional(s, radii=radii, **field) == (-1, b"backward: NULL argument"), missing


def test_misaligned_rotation_and_sh_gradients_are_refused():
    """dL_drot, and dL_dsh with M = 16 and degree 3, are written with 16-byte stores: a pointer that is not 16-byte aligned fails
    with GOF_E_INVALID before any work, through gof_rasterize_backward_ex and the positional gof_rasterize_backward."""
    s = _fake_scene(300)
    assert (s.M, s.D) == (16, 3)
    for field in ("dL_drot", "dL_dsh"):
        for rc, err in (_call(s, _out(**{field: 0x1004})), _positional(s, **{field: 0x1004})):
            assert rc == -1 and f"{field} must be 16-byte aligned".encode() in err, field


def _check_request(request_):
    """The checks every camera or focal-length request gets: dL_dviewmatrix and dL_dcampos come together (both orders), a
    scratch one byte short or NULL is refused, and the factored SH gradient does not combine with it."""
    s = _fake_scene(300)
    for half in (dict(dL_dcampos=None), dict(dL_dviewmatrix=None)):
        o = request_(dL_dviewmatrix=FAKE, dL_dcampos=2 * FAKE) if request_ is _intrinsics else request_()
        for k, v in half.items():
            setattr(o, k, v)
        rc, err = _call(s, o)
        assert rc == -1 and b"come together" in err, half
    o = request_()
    assert o.scratch_bytes > 0
    o.scratch_bytes -= 1
    rc, err = _call(s, o)
    assert rc == -1 and b"scratch" in err
    o = request_()
    o.scratch = None
    rc, err = _call(s, o)
    assert rc == -1 and b"scratch" in err
    rc, err = _call(s, request_(sh_rgb=5 * FAKE, sh_hdr=6 * FAKE))
    assert rc == -1 and b"sh_rgb" in err


def test_camera_arguments_are_checked():
    _check_request(_camera)


def test_intrinsics_arguments_are_checked():
    _check_request(_intrinsics)
