"""CPU: the per-view loss with the decoupled-appearance L1 (train.py:67-88, 157-159 of the reference).

- the fp64 oracle (tests/_loss_app_oracle.py) against the goldens the reference's own Python produced
  (tests/golden/make_golden_loss_appearance.py);
- the kernel source (csrc/view_loss.cuh in appearance mode), compiled for the host and run phase by phase
  (tests/hostmath/view_loss_app_host.cpp), against those goldens and against the oracle on ragged shapes;
- the argument checks of gof_view_loss_appearance, which all come before any device work, so no GPU is needed."""
import ctypes
import glob
import math
import os
import subprocess

import numpy as np
import pytest

import _loss_app_oracle
import loss_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = sorted(glob.glob(os.path.join(HERE, "golden", "loss_app_*.npz")))
TERMS = ("Ll1", "ssim", "depth_normal_loss", "distortion_loss", "loss")


@pytest.fixture(scope="module")
def hm():
    d = os.path.join(HERE, "hostmath")
    lib, src = os.path.join(d, "libviewloss_app_host.so"), os.path.join(d, "view_loss_app_host.cpp")
    hdr = os.path.join(HERE, "..", "gaussian-opacity-fields_b200", "csrc", "view_loss.cuh")
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-x", "c++", src, "-o", lib])
    return ctypes.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def run_host(hm, render, gt, wvt, tanfovx, tanfovy, lambdas, mapping, top, left, need_grad=True):
    _, H, W = render.shape
    c2w = np.linalg.inv(np.asarray(wvt, np.float64).T)
    R9 = np.ascontiguousarray(c2w[:3, :3], np.float32).reshape(9)
    g = np.array([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)], np.float32)
    g = (g / g.sum()).astype(np.float32)
    render, gt = np.ascontiguousarray(render, np.float32), np.ascontiguousarray(gt, np.float32)
    mapping = np.ascontiguousarray(mapping, np.float32)
    Hc, Wc = mapping.shape[1:]
    terms = np.zeros(5, np.float32)
    grad = np.zeros_like(render) if need_grad else None
    grad_m = np.zeros_like(mapping) if need_grad else None
    hm.hm_view_loss_app(W, H, _p(render), _p(gt), _p(R9), ctypes.c_float(W / (2 * tanfovx)), ctypes.c_float(H / (2 * tanfovy)),
                        _p(g), ctypes.c_float(lambdas[0]), ctypes.c_float(lambdas[1]), ctypes.c_float(lambdas[2]), _p(mapping),
                        top, left, Hc, Wc, _p(terms), _p(grad) if need_grad else None, _p(grad_m) if need_grad else None)
    return terms, grad, grad_m


def golden(path):
    """(inputs, expected): the appearance loss of a golden file in the oracle's keys."""
    fx = np.load(path)
    inp = dict(render=fx["render"], gt=fx["gt"], wvt=fx["world_view_transform"], tanfovx=float(fx["tanfovx"]),
               tanfovy=float(fx["tanfovy"]), lambdas=[float(x) for x in fx["lambdas"]], mapping=fx["mapping"],
               top=int(fx["top"]), left=int(fx["left"]))
    grad = fx["grad"].astype(np.float64).copy()
    grad[:3] = fx["app_grad_rgb"]
    exp = dict(Ll1=float(fx["app_Ll1"]), ssim=float(fx["ssim"]), depth_normal_loss=float(fx["depth_normal_loss"]),
               distortion_loss=float(fx["distortion_loss"]), loss=float(fx["app_loss"]), grad=grad,
               grad_mapping=fx["grad_mapping"].astype(np.float64))
    return inp, exp


def oracle(inp, need_grad=True):
    return _loss_app_oracle.view_loss(inp["render"], inp["gt"], inp["wvt"], inp["tanfovx"], inp["tanfovy"], inp["lambdas"],
                                      inp["mapping"], inp["top"], inp["left"], need_grad)


def check(terms, grad, grad_m, exp, keep=None, rtol=1e-5, gtol=None):
    """terms within rtol relative; each gradient channel and the mapping gradient within 1e-4 (gtol per channel) of its
    largest magnitude, over the crop pixels `keep` [3,Hc,Wc] (None: all) for the L1-bearing values."""
    for i, k in enumerate(TERMS):
        assert abs(float(terms[i]) - exp[k]) <= rtol * max(1.0, abs(exp[k])), (k, float(terms[i]), exp[k])
    top, left = exp["top"], exp["left"]
    Hc, Wc = exp["grad_mapping"].shape[1:]
    mask = np.ones(grad.shape, bool)
    if keep is not None:
        mask[:3, top:top + Hc, left:left + Wc] = keep
    for ch in range(9):
        den = max(np.abs(exp["grad"][ch]).max(), 1e-12)
        err = np.abs(grad[ch] - exp["grad"][ch])[mask[ch]].max() / den
        assert err < (gtol or {}).get(ch, 1e-4), (ch, err)
    mk = np.ones(grad_m.shape, bool) if keep is None else keep
    den = max(np.abs(exp["grad_mapping"]).max(), 1e-12)
    assert np.abs(grad_m - exp["grad_mapping"])[mk].max() / den < 1e-4


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-4] for p in FIX])
def test_oracle_matches_reference_goldens(path):
    inp, exp = golden(path)
    exp.update(top=inp["top"], left=inp["left"])
    out = oracle(inp)
    marginal = out["marginal"]
    assert marginal.mean() < 1e-3
    check([out[k] for k in TERMS], out["grad"], out["grad_mapping"], exp, keep=~marginal, rtol=2e-6)
    # the terms and gradient channels the appearance L1 does not touch are the plain oracle's
    plain = loss_oracle.view_loss(inp["render"], inp["gt"], inp["wvt"], inp["tanfovx"], inp["tanfovy"], inp["lambdas"])
    assert np.array_equal(plain["grad"][3:], out["grad"][3:]) and plain["ssim"] == out["ssim"]


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-4] for p in FIX])
def test_kernel_source_matches_goldens_and_oracle(hm, path):
    inp, exp = golden(path)
    exp.update(top=inp["top"], left=inp["left"])
    terms, grad, grad_m = run_host(hm, inp["render"], inp["gt"], inp["wvt"], inp["tanfovx"], inp["tanfovy"], inp["lambdas"],
                                   inp["mapping"], inp["top"], inp["left"])
    check(terms, grad, grad_m, exp)                       # the goldens' float32 products decide the same signs
    out = oracle(inp)
    out.update(top=inp["top"], left=inp["left"])
    check(terms, grad, grad_m, out, keep=~out["marginal"])


@pytest.mark.parametrize("H,W,top,left,Hc,Wc", [(33, 40, 0, 4, 32, 32), (37, 50, 2, 9, 32, 32), (70, 101, 3, 2, 64, 96),
                                                (45, 64, 6, 0, 32, 64), (35, 17, 1, 3, 9, 5)])
def test_kernel_source_vs_oracle_on_ragged_crops(hm, H, W, top, left, Hc, Wc):
    """Image and crop edges off the 16-pixel tile grid, a crop of full width, and a crop that is not a multiple of 32 (the
    kernels take any crop inside the image); values-only terms bit-equal to the gradient run."""
    import gof_synth
    rng = np.random.default_rng(H * 1000 + W)
    cam = gof_synth.make_camera(W, H, view=12)
    render = rng.uniform(0, 1, size=(9, H, W)).astype(np.float32)
    render[3:6] -= 0.5
    render[6] = 2.0 + render[6]
    gt = rng.uniform(0, 1, size=(3, H, W)).astype(np.float32)
    mapping = rng.uniform(0, 1.5, size=(3, Hc, Wc)).astype(np.float32)
    inp = dict(render=render, gt=gt, wvt=cam.world_view_transform.numpy(), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
               lambdas=(0.2, 0.05, 100.0), mapping=mapping, top=top, left=left)
    terms, grad, grad_m = run_host(hm, render, gt, inp["wvt"], cam.tanfovx, cam.tanfovy, inp["lambdas"], mapping, top, left)
    out = oracle(inp)
    out.update(top=top, left=left)
    check(terms, grad, grad_m, out, keep=~out["marginal"], gtol={6: 2e-3})
    t2, _, _ = run_host(hm, render, gt, inp["wvt"], cam.tanfovx, cam.tanfovy, inp["lambdas"], mapping, top, left, need_grad=False)
    assert np.array_equal(t2, terms)
    outside = np.ones((H, W), bool)
    outside[top:top + Hc, left:left + Wc] = False
    # outside the crop only the SSIM term: with lambda_dssim = 0 the rgb gradient there is exactly 0
    _, g0, _ = run_host(hm, render, gt, inp["wvt"], cam.tanfovx, cam.tanfovy, (0.0, 0.05, 100.0), mapping, top, left)
    assert (g0[:3][:, outside] == 0).all()


# ---------------------------------------------------------------------------------------------------- C ABI refusals
GOF_OK, GOF_E_INVALID = 0, -1
FAKE = 0x1000


def _abi():
    try:
        import gof_loss
    except ImportError as e:   # the library is built by __graft_entry__.build()
        pytest.skip(str(e))
    return gof_loss._lib


def _call(lib, W=64, H=48, render=FAKE, gt=FAKE, fx=50.0, fy=50.0, mapping=FAKE, top=8, left=0, Hc=32, Wc=64, terms=FAKE,
          grad=FAKE, grad_mapping=FAKE, scratch=FAKE):
    R9 = (ctypes.c_float * 9)(*np.eye(3).reshape(-1))
    return lib.gof_view_loss_appearance(W, H, render, gt, R9, fx, fy, 0.2, 0.05, 100.0, mapping, top, left, Hc, Wc, terms, grad,
                                        grad_mapping, scratch, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(mapping=None), b"mapping is NULL"),
    (dict(Hc=0), b"crop"), (dict(Wc=0), b"crop"), (dict(Hc=-32), b"crop"),
    (dict(top=-1), b"crop"), (dict(left=-1), b"crop"), (dict(top=17), b"crop"), (dict(left=1), b"crop"),
    (dict(Hc=49, top=0), b"crop"), (dict(Wc=65), b"crop"), (dict(top=2 ** 31 - 1), b"crop"),
    (dict(grad=None), b"grad_mapping"), (dict(grad_mapping=None), b"grad_mapping"),
    (dict(render=None), b"bad arguments"), (dict(scratch=None), b"bad arguments"), (dict(terms=None), b"bad arguments"),
    (dict(W=0), b"bad arguments"), (dict(fx=0.0), b"bad arguments"),
])
def test_bad_arguments_are_refused(kw, msg):
    lib = _abi()
    assert _call(lib, **kw) == GOF_E_INVALID, kw
    assert msg in lib.gof_last_error(), lib.gof_last_error()


def test_binding_refuses_small_images_and_mismatched_mappings():
    """view_loss(appearance=...) checks the image size and the mapping's shape before touching a device."""
    import torch
    import gof_loss
    wvt = torch.eye(4)
    for (H, W) in ((31, 64), (64, 31)):
        with pytest.raises(ValueError, match="32 x 32"):
            gof_loss.view_loss(torch.zeros(9, H, W), torch.zeros(3, H, W), wvt, 0.5, 0.5, appearance=torch.zeros(3, 0, 0))
    for shape in ((3, 32, 32), (1, 3, 32, 64, 1), (2, 3, 32, 64), (3, 64, 32), (1, 32, 64)):
        with pytest.raises(ValueError, match="appearance mapping"):
            gof_loss.view_loss(torch.zeros(9, 48, 72), torch.zeros(3, 48, 72), wvt, 0.5, 0.5, appearance=torch.zeros(shape))
