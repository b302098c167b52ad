"""CPU: the argument checks of gof_integrate_min (the per-view running minimum of the multi-view opacity field, DESIGN.md 4.12),
through the built library.  Every case is decided before any device work, so no GPU is needed: the device pointers are never
dereferenced."""
import ctypes

import pytest

GOF_OK, GOF_E_INVALID, GOF_E_ALLOC = 0, -1, -3
FAKE = 0x1000


def _abi():
    try:
        from diff_gaussian_rasterization import _C
    except ImportError as e:   # the library is built by __graft_entry__.build()
        pytest.skip(str(e))
    return _C


def _scene(_C, P=10):
    s = _C._Scene()
    s.P, s.width, s.height, s.tan_fovx, s.tan_fovy = P, 32, 32, 0.5, 0.5
    for name in ("means3D", "opacities", "viewmatrix", "projmatrix", "background", "colors_precomp", "scales", "rotations"):
        setattr(s, name, FAKE)
    return s


class _Allocs:
    """The five allocator callbacks; `fail` lists the ones that return NULL (a buffer the caller could not provide)."""

    def __init__(self, _C, fail=()):
        self.calls = []

        def make(i):
            def f(_user, nbytes):
                self.calls.append((i, nbytes))
                return 0 if i in fail else FAKE
            return _C._ALLOC_FN(f)
        self.cbs = [make(i) for i in range(5)]

    def args(self):
        out = []
        for cb in self.cbs:
            out += [cb, None]
        return out


def _call(_C, s, PN=4, points=FAKE, view=0, allocs=None, radii=FAKE, alpha_min=FAKE, argmin=FAKE, color_min=None):
    allocs = allocs if allocs is not None else _Allocs(_C)
    return _C._lib.gof_integrate_min(ctypes.byref(s), PN, points, view, *allocs.args(), radii, alpha_min, argmin, color_min, None)


def test_null_buffers_are_refused():
    _C = _abi()
    s = _scene(_C)
    for kw in (dict(points=None), dict(radii=None), dict(alpha_min=None), dict(argmin=None)):
        assert _call(_C, s, **kw) == GOF_E_INVALID, kw
        assert b"NULL" in _C._lib.gof_last_error()


def test_null_allocator_is_refused():
    _C = _abi()
    s = _scene(_C)
    a = _Allocs(_C)
    a.cbs[3] = _C._ALLOC_FN()   # a NULL function pointer
    assert _call(_C, s, allocs=a) == GOF_E_INVALID
    assert b"allocators" in _C._lib.gof_last_error()


def test_allocator_returning_null_fails_before_any_work():
    """A scratch buffer the caller cannot provide (the geometry or the image buffer) is GOF_E_ALLOC, before any launch."""
    _C = _abi()
    s = _scene(_C)
    for fail in (0, 2):
        a = _Allocs(_C, fail=(fail,))
        assert _call(_C, s, allocs=a) == GOF_E_ALLOC, fail
        assert b"NULL" in _C._lib.gof_last_error()


def test_view_outside_range_is_refused():
    _C = _abi()
    s = _scene(_C)
    for view in (-1, 2 ** 30):
        assert _call(_C, s, view=view) == GOF_E_INVALID, view
        assert b"view" in _C._lib.gof_last_error()


def test_nothing_to_do_writes_nothing():
    """PN == 0 (or negative, as gof_integrate) and P == 0 return GOF_OK without allocating or touching a buffer, even NULL ones."""
    _C = _abi()
    for P, PN in ((10, 0), (10, -3), (0, 4)):
        s = _scene(_C, P=P)
        a = _Allocs(_C)
        assert _call(_C, s, PN=PN, allocs=a, points=None, radii=None, alpha_min=None, argmin=None) == GOF_OK, (P, PN)
        assert a.calls == []


def test_bad_scene_is_refused():
    _C = _abi()
    s = _scene(_C)
    s.P = -1
    assert _call(_C, s) == GOF_E_INVALID
    s = _scene(_C)
    s.colors_precomp = None   # neither SHs nor colours
    assert _call(_C, s) == GOF_E_INVALID
    assert _C._lib.gof_integrate_min(None, 4, FAKE, 0, *_Allocs(_C).args(), FAKE, FAKE, FAKE, None, None) == GOF_E_INVALID


def test_binding_checks_the_running_minimum_tensors():
    """_C.integrate_gaussians_to_points_min refuses alpha_min / argmin of the wrong dtype or length before calling the library."""
    import torch
    _C = _abi()
    pts = torch.zeros(5, 3)
    for am, ai in ((torch.ones(5, dtype=torch.float64), torch.zeros(5, dtype=torch.int32)),
                   (torch.ones(5), torch.zeros(5, dtype=torch.int64)),
                   (torch.ones(4), torch.zeros(5, dtype=torch.int32))):
        with pytest.raises(RuntimeError, match="alpha_min|argmin"):
            _C.integrate_gaussians_to_points_min(None, pts, None, None, None, None, None, 1.0, None, None, None, None, 0.5, 0.5, 0.0,
                                                 None, 8, 8, None, 0, None, False, False, 0, am, ai)
