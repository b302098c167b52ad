"""CPU: the argument checks of the opacity-field query, gof_integrate and gof_integrate_cached, in both modes of their outputs
(gof_integrate_out_t): the query's own outputs and the running minimum over views of the multi-view opacity field (DESIGN.md
4.12-4.14), through the built library.  Every case is decided before any device work, so no GPU is needed: the device pointers
are never dereferenced."""
import ctypes

import pytest

GOF_OK, GOF_E_INVALID, GOF_E_ALLOC = 0, -1, -3
FAKE = 0x1000
QUERY = dict(out_color=FAKE, out_alpha_integrated=FAKE, out_color_integrated=FAKE)
ENTRIES = ("integrate", "integrate_cached")
CASES = [(entry, mode) for entry in ENTRIES for mode in ("query", "min")]
N_ALLOCS = {"integrate": 5, "integrate_cached": 3}


def _abi():
    try:
        from diff_gaussian_rasterization import _C
    except ImportError as e:   # the library is built by __graft_entry__.build()
        pytest.skip(str(e))
    return _C


def _scene(_C, entry, P=10):
    """A valid scene: gof_integrate's, or only the fields gof_integrate_cached reads (P, width, height, tan_fov, viewmatrix and
    background)."""
    s = _C._Scene()
    s.P, s.width, s.height, s.tan_fovx, s.tan_fovy = P, 32, 32, 0.5, 0.5
    s.viewmatrix, s.background = FAKE, FAKE
    if entry == "integrate":
        for name in ("means3D", "opacities", "projmatrix", "colors_precomp", "scales", "rotations"):
            setattr(s, name, FAKE)
    return s


def _fields(entry, mode):
    """The outputs of `mode`; the cached running minimum also forms grad_min."""
    if mode == "query":
        return dict(QUERY)
    return dict(alpha_min=FAKE, argmin=FAKE, **(dict(grad_min=FAKE) if entry == "integrate_cached" else {}))


class _Allocs:
    """The entry point's allocator callbacks (gof_integrate: geometry, binning, image, point, point binning; gof_integrate_cached:
    image, point, point binning); `fail` lists the ones that return NULL (a buffer the caller could not provide)."""

    def __init__(self, _C, entry, fail=()):
        self.calls = []

        def make(i):
            def f(_user, nbytes):
                self.calls.append((i, nbytes))
                return 0 if i in fail else FAKE
            return _C._ALLOC_FN(f)
        self.cbs = [make(i) for i in range(N_ALLOCS[entry])]

    def args(self):
        out = []
        for cb in self.cbs:
            out += [cb, None]
        return out


def _call(_C, entry, s, PN=4, points=FAKE, allocs=None, radii=FAKE, cache=FAKE, num_rendered=7, out=True, **fields):
    """gof_<entry> with fake buffers and a gof_integrate_out_t of `fields` (out=None: a NULL out).  gof_integrate takes radii and
    a host num_rendered (None: NULL), gof_integrate_cached a cache and its num_rendered."""
    allocs = allocs if allocs is not None else _Allocs(_C, entry)
    o = ctypes.byref(_C._IntegrateOut(**fields)) if out else None
    sp = ctypes.byref(s) if s is not None else None
    if entry == "integrate":
        rendered = ctypes.byref(ctypes.c_int(-1)) if num_rendered is not None else None
        return _C._lib.gof_integrate(sp, PN, points, *allocs.args(), radii, rendered, o, None)
    return _C._lib.gof_integrate_cached(sp, PN, points, cache, num_rendered, *allocs.args(), o, None)


@pytest.mark.parametrize("entry,mode", CASES)
def test_null_buffers_are_refused(entry, mode):
    _C = _abi()
    s = _scene(_C, entry)
    buffers = [dict(points=None)] + ([dict(radii=None)] if entry == "integrate" else [dict(cache=None), dict(num_rendered=-1)])
    for kw in buffers + [{name: None} for name in ("alpha_min", "argmin") if mode == "min"]:
        assert _call(_C, entry, s, **{**_fields(entry, mode), **kw}) == GOF_E_INVALID, kw
        assert b"NULL" in _C._lib.gof_last_error()
    if mode == "query":   # each of the query's outputs is required
        for name in QUERY:
            assert _call(_C, entry, s, **{**QUERY, name: None}) == GOF_E_INVALID, name
            assert b"NULL" in _C._lib.gof_last_error()


@pytest.mark.parametrize("entry,mode", CASES)
def test_null_allocator_is_refused(entry, mode):
    """Before the nothing-to-do return too (PN == 0)."""
    _C = _abi()
    s = _scene(_C, entry)
    for PN in (4, 0):
        for i in range(N_ALLOCS[entry]):
            a = _Allocs(_C, entry)
            a.cbs[i] = _C._ALLOC_FN()   # a NULL function pointer
            assert _call(_C, entry, s, PN=PN, allocs=a, **_fields(entry, mode)) == GOF_E_INVALID, (PN, i)
            assert b"allocators" in _C._lib.gof_last_error()
    if entry == "integrate":   # gof_integrate writes num_rendered in both modes
        assert _call(_C, entry, s, num_rendered=None, **_fields(entry, mode)) == GOF_E_INVALID
        assert b"num_rendered" in _C._lib.gof_last_error()


@pytest.mark.parametrize("entry,mode", CASES)
def test_allocator_returning_null_fails_before_any_work(entry, mode):
    """A scratch buffer the caller cannot provide is GOF_E_ALLOC, before any launch: of gof_integrate's, the geometry and the
    image buffer (the others are taken after the Gaussian side has been launched), and each of gof_integrate_cached's."""
    _C = _abi()
    s = _scene(_C, entry)
    for fail in ((0, 2) if entry == "integrate" else (0, 1, 2)):
        a = _Allocs(_C, entry, fail=(fail,))
        assert _call(_C, entry, s, allocs=a, **_fields(entry, mode)) == GOF_E_ALLOC, fail
        assert b"NULL" in _C._lib.gof_last_error()


@pytest.mark.parametrize("entry", ENTRIES)
def test_view_outside_range_is_refused(entry):
    _C = _abi()
    s = _scene(_C, entry)
    for view in (-1, 2 ** 30):
        assert _call(_C, entry, s, view=view, **_fields(entry, "min")) == GOF_E_INVALID, view
        assert b"view" in _C._lib.gof_last_error()


@pytest.mark.parametrize("entry,mode", CASES)
def test_nothing_to_do_writes_nothing(entry, mode):
    """PN <= 0 and P == 0 return GOF_OK without allocating or touching a buffer, even NULL ones (outputs included)."""
    _C = _abi()
    for P, PN in ((10, 0), (10, -3), (0, 4)):
        s = _scene(_C, entry, P=P)
        for fields in (_fields(entry, mode), {}):
            a = _Allocs(_C, entry)
            assert _call(_C, entry, s, PN=PN, allocs=a, points=None, radii=None, cache=None, **fields) == GOF_OK, (P, PN, fields)
            assert a.calls == []


@pytest.mark.parametrize("entry", ENTRIES)
def test_null_out_is_refused(entry):
    _C = _abi()
    for PN in (4, 0):
        assert _call(_C, entry, _scene(_C, entry), PN=PN, out=None) == GOF_E_INVALID
        assert b"out is NULL" in _C._lib.gof_last_error()


@pytest.mark.parametrize("entry", ENTRIES)
def test_fields_of_both_modes_are_refused(entry):
    """The query's outputs with alpha_min / argmin, and color_min / grad_min without them, even with nothing to do."""
    _C = _abi()
    s = _scene(_C, entry)
    for PN in (4, 0):
        for name in QUERY:
            for minimum in (dict(alpha_min=FAKE, argmin=FAKE), dict(alpha_min=FAKE), dict(argmin=FAKE)):
                assert _call(_C, entry, s, PN=PN, **{name: FAKE}, **minimum) == GOF_E_INVALID, (PN, name, minimum)
                assert b"must be NULL with alpha_min / argmin" in _C._lib.gof_last_error()
        for name in ("color_min", "grad_min"):
            for query in (QUERY, {}):
                assert _call(_C, entry, s, PN=PN, **{name: FAKE}, **query) == GOF_E_INVALID, (PN, name, query)
                assert b"need alpha_min and argmin" in _C._lib.gof_last_error()


def test_gof_integrate_refuses_grad_min():
    _C = _abi()
    s = _scene(_C, "integrate")
    for PN in (4, 0):
        assert _call(_C, "integrate", s, PN=PN, grad_min=FAKE, **_fields("integrate", "min")) == GOF_E_INVALID
        assert b"grad_min" in _C._lib.gof_last_error()


def test_min_color_refusals():
    """gof_integrate's running minimum with color_min."""
    _C = _abi()
    err = _C._lib.gof_last_error
    s = _scene(_C, "integrate")

    def call(**kw):
        return _call(_C, "integrate", s, **{"alpha_min": FAKE, "argmin": FAKE, "color_min": FAKE, **kw})
    for kw in (dict(points=None), dict(radii=None), dict(alpha_min=None), dict(argmin=None)):
        assert call(**kw) == GOF_E_INVALID and b"NULL" in err(), kw
    for view in (-1, 2 ** 30):
        assert call(view=view) == GOF_E_INVALID and b"view" in err()
    a = _Allocs(_C, "integrate")
    a.cbs[1] = _C._ALLOC_FN()
    assert call(allocs=a) == GOF_E_INVALID and b"allocators" in err()
    assert call(allocs=_Allocs(_C, "integrate", fail=(0,))) == GOF_E_ALLOC
    a = _Allocs(_C, "integrate")
    assert call(PN=0, allocs=a, points=None, radii=None, alpha_min=None, argmin=None, color_min=None) == GOF_OK and a.calls == []


def test_bad_scene_is_refused():
    """gof_integrate validates the whole scene."""
    _C = _abi()
    for entry_fields in (_fields("integrate", "query"), _fields("integrate", "min")):
        s = _scene(_C, "integrate")
        s.P = -1
        assert _call(_C, "integrate", s, **entry_fields) == GOF_E_INVALID
        s = _scene(_C, "integrate")
        s.colors_precomp = None   # neither SHs nor colours
        assert _call(_C, "integrate", s, **entry_fields) == GOF_E_INVALID
        assert _call(_C, "integrate", None, **entry_fields) == GOF_E_INVALID


def test_bad_cached_scene_is_refused():
    """gof_integrate_cached checks the fields it reads."""
    _C = _abi()
    for entry_fields in (_fields("integrate_cached", "query"), _fields("integrate_cached", "min")):
        assert _call(_C, "integrate_cached", None, **entry_fields) == GOF_E_INVALID
        for field, value in (("P", -1), ("width", 0), ("height", -2), ("viewmatrix", None), ("background", None)):
            s = _scene(_C, "integrate_cached")
            setattr(s, field, value)
            assert _call(_C, "integrate_cached", s, **entry_fields) == GOF_E_INVALID, field
            assert b"scene" in _C._lib.gof_last_error()


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


def test_binding_checks_the_cached_running_minimum_tensors():
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
