"""CPU: the argument checks of gof_integrate_cached_min (the multi-view opacity field's running minimum against a cached Gaussian
side, with the winning view's point gradient, DESIGN.md 4.14), through the built library.  Every case is decided before any
device work, so no GPU is needed: the device pointers are never dereferenced."""
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
    """The scene fields gof_integrate_cached reads: P, width, height, tan_fov, viewmatrix and background."""
    s = _C._Scene()
    s.P, s.width, s.height, s.tan_fovx, s.tan_fovy = P, 32, 32, 0.5, 0.5
    s.viewmatrix, s.background = FAKE, FAKE
    return s


class _Allocs:
    """The three allocator callbacks (image, point, point binning); `fail` lists the ones that return NULL."""

    def __init__(self, _C, fail=()):
        self.calls = []

        def make(i):
            def f(_user, nbytes):
                self.calls.append((i, nbytes))
                return 0 if i in fail else FAKE
            return _C._ALLOC_FN(f)
        self.cbs = [make(i) for i in range(3)]

    def args(self):
        out = []
        for cb in self.cbs:
            out += [cb, None]
        return out


def _call(_C, s, PN=4, points=FAKE, view=0, cache=FAKE, num_rendered=7, allocs=None, alpha_min=FAKE, argmin=FAKE, color_min=None,
          grad_min=FAKE):
    allocs = allocs if allocs is not None else _Allocs(_C)
    return _C._lib.gof_integrate_cached_min(ctypes.byref(s) if s is not None else None, PN, points, view, cache, num_rendered,
                                            *allocs.args(), alpha_min, argmin, color_min, grad_min, None)


def test_null_buffers_are_refused():
    _C = _abi()
    s = _scene(_C)
    for kw in (dict(points=None), dict(cache=None), dict(alpha_min=None), dict(argmin=None), dict(num_rendered=-1)):
        assert _call(_C, s, **kw) == GOF_E_INVALID, kw
        assert b"NULL" in _C._lib.gof_last_error()


def test_null_allocator_is_refused():
    _C = _abi()
    s = _scene(_C)
    for i in range(3):
        a = _Allocs(_C)
        a.cbs[i] = _C._ALLOC_FN()   # a NULL function pointer
        assert _call(_C, s, allocs=a) == GOF_E_INVALID, i
        assert b"allocators" in _C._lib.gof_last_error()


def test_allocator_returning_null_fails_before_any_work():
    """A scratch buffer the caller cannot provide is GOF_E_ALLOC, before any launch."""
    _C = _abi()
    s = _scene(_C)
    for fail in range(3):
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
    """PN <= 0 and P == 0 return GOF_OK without allocating or touching a buffer, even NULL ones (colour and gradient included)."""
    _C = _abi()
    for P, PN in ((10, 0), (10, -3), (0, 4)):
        s = _scene(_C, P=P)
        a = _Allocs(_C)
        assert _call(_C, s, PN=PN, allocs=a, points=None, cache=None, alpha_min=None, argmin=None, grad_min=None) == GOF_OK, (P, PN)
        assert a.calls == []


def test_bad_scene_is_refused():
    _C = _abi()
    assert _call(_C, None) == GOF_E_INVALID
    for field, value in (("P", -1), ("width", 0), ("height", -2), ("viewmatrix", None), ("background", None)):
        s = _scene(_C)
        setattr(s, field, value)
        assert _call(_C, s) == GOF_E_INVALID, field
        assert b"scene" in _C._lib.gof_last_error()


def test_binding_checks_the_running_minimum_tensors():
    """_C.integrate_points_cached_min refuses alpha_min / argmin / color_min / grad_min of the wrong dtype, shape or layout
    before calling the library."""
    import torch
    _C = _abi()
    pts = torch.zeros(5, 3)
    cache = _C.IntegrateCache(torch.zeros(1, dtype=torch.uint8), 0, None, 10, 8, 8)
    am, ai, c3 = torch.ones(5), torch.zeros(5, dtype=torch.int32), torch.zeros(5, 3)
    bad = (dict(alpha_min=torch.ones(5, dtype=torch.float64)), dict(argmin=torch.zeros(5, dtype=torch.int64)),
           dict(alpha_min=torch.ones(4)), dict(color_min=torch.zeros(5, 4)), dict(grad_min=torch.zeros(5, 3, dtype=torch.float64)),
           dict(grad_min=torch.zeros(3, 5).t()))
    for kw in bad:
        args = dict(alpha_min=am, argmin=ai, color_min=c3, grad_min=c3)
        args.update(kw)
        with pytest.raises(RuntimeError, match=next(iter(kw))):
            _C.integrate_points_cached_min(cache, None, pts, None, 0.5, 0.5, 0, **args)


def test_field_gradient_needs_a_cached_integrator():
    import torch
    import gof_extract
    with pytest.raises(TypeError, match="CachedIntegrator"):
        gof_extract.field_gradient(torch.zeros(3, 3), [], lambda p, v: None)
