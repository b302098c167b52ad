"""The view-parallel exchange's own kernels at every world size, on one device.

  gof_p2p_allreduce_f32   (csrc/exchange.cu)  N distinct allocations on one device stand for the N ranks' buckets: calling the
                          entry point once per rank leaves what N processes would, since the ranks' slices are disjoint.  Every
                          add is one fp32 rounding in rank order 0..N-1 and the MAX tail is fmaxf, so torch's `s += b_r` chain
                          (one IEEE round-to-nearest per elementwise add) and torch.maximum restate it exactly: every buffer
                          must carry the reference's bits, whatever order the ranks are called in, and the guard floats
                          around each slice must keep their NaN pattern.  N = 2..8 covers k_p2p_allreduce<2>, <4>, <8> and
                          k_p2p_allreduce_any (3, 5, 6, 7).
  gof_sh_grad_from_views  (csrc/sh_views.cu)  against tests/_sh_views_oracle.py, a numpy float32 restatement of the same
                          explicitly rounded operations: bit for bit, at every NV instantiation and both sides of its bounds,
                          M in {1, 4, 9, 16} (the scalar M < 16 store path and the float4 one) and P at partial warps and CTAs,
                          with each view's record in its own allocation and NaN past P.

Tests without the gpu mark pin the oracle on the CPU and check the host-side refusals of the three entry points in a process
that sees no device."""
import ctypes
import json
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import _sh_views_oracle as shv

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(ROOT, "gaussian-opacity-fields_b200", "diff_gaussian_rasterization", "libgof_b200.so")
GOF_OK, GOF_E_INVALID = 0, -1
GUARD = 64                          # guard floats after each buffer
NAN_BITS = 0x7FC0DEAD               # a quiet NaN with a payload no arithmetic produces
gpu = pytest.mark.gpu


def _nan_fill(n, dev):
    return torch.full((n,), NAN_BITS, dtype=torch.int32, device=dev).view(torch.float32)


# ========================================================================================================================
# 1. gof_p2p_allreduce_f32
# ========================================================================================================================

def _p2p():
    from diff_gaussian_rasterization import _C
    f = _C._lib.gof_p2p_allreduce_f32
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p]
    return f


def _reduce(peers, n_sum, n, order):
    """Runs every rank's call of gof_p2p_allreduce_f32 over the buffers `peers`, in `order`."""
    from diff_gaussian_rasterization import _C
    f, N = _p2p(), len(peers)
    arr = (ctypes.c_void_p * N)(*[p.data_ptr() for p in peers])
    for r in order:
        _C._check(f(arr, N, int(r), n_sum, n, _C._stream()))
    torch.cuda.synchronize()


class _Peers:
    """N buffers of n floats with at least GUARD NaN-pattern floats after each: N allocations, or (shared=True) N views at
    16-byte aligned offsets that are not multiples of 256 bytes into one allocation."""

    def __init__(self, N, n, dev, shared=False):
        if shared:
            stride = (n + GUARD + 63) // 64 * 64 + 4
            offs = [4 + r * stride for r in range(N)]
            assert all(o % 4 == 0 and o % 64 != 0 for o in offs)
            self.backing = [_nan_fill(4 + N * stride + GUARD, dev)]
            self.peers = [self.backing[0][o:o + n] for o in offs]
            self.spans = [(0, o) for o in offs]
        else:
            self.backing = [_nan_fill(n + GUARD, dev) for _ in range(N)]
            self.peers = [b[:n] for b in self.backing]
            self.spans = [(r, 0) for r in range(N)]
        self.n = n

    def load(self, vals):
        for p, v in zip(self.peers, vals):
            p.copy_(v)

    def guards_intact(self):
        for i, b in enumerate(self.backing):
            keep = torch.ones(b.numel(), dtype=torch.bool, device=b.device)
            for j, o in self.spans:
                if j == i:
                    keep[o:o + self.n] = False
            if not bool((b.view(torch.int32)[keep] == NAN_BITS).all()):
                return False
        return True


def _inputs(N, n, n_sum, seed, dev):
    """Rank r's bucket: SUM part of normal floats of mixed sign and exponent, with exact cancellations, +-0 and subnormals; MAX
    tail non-negative (as the statistics are), with ties and zeros."""
    g = torch.Generator(device=dev).manual_seed(seed)
    i = torch.arange(n, device=dev)
    vals = []
    for r in range(N):
        v = torch.randn(n, generator=g, device=dev) * torch.exp2(torch.randint(-20, 21, (n,), generator=g, device=dev).float())
        sub = torch.randint(-(1 << 22), 1 << 22, (n,), generator=g, device=dev).float() * 2.0 ** -149     # subnormals (and 0)
        v = torch.where(i % 13 == 4, sub, v)                       # all ranks subnormal: every partial sum is exact
        v = torch.where((i % 13 == 8) & (r % 2 == 1), sub, v)      # subnormals added to normals
        v = torch.where(i % 11 == 5, torch.full_like(v, 0.0 if r % 2 == 0 else -0.0), v)    # +0 + -0 + ...
        v = torch.where(i % 11 == 6, torch.full_like(v, -0.0), v)                           # -0 + -0 + ... = -0
        vals.append(v)
    if N >= 2:
        vals[1] = torch.where(i % 7 == 0, -vals[0], vals[1])       # the partial sum of ranks 0, 1 cancels exactly
    if N >= 3:                                                     # the last rank cancels the whole partial sum: +0
        part = vals[0].clone()
        for v in vals[1:-1]:
            part += v
        vals[-1] = torch.where(i % 7 == 3, -part, vals[-1])
    for r, v in enumerate(vals):
        tail = v[n_sum:].abs()
        tail = torch.where(i[n_sum:] % 5 == 0, torch.zeros_like(tail), tail)
        tail = torch.where(i[n_sum:] % 5 == 1, torch.full_like(tail, 0.75), tail)           # ties between ranks
        v[n_sum:] = tail
    return vals


def _reference(vals, n_sum):
    """The kernel restated: rank-order fp32 sum over [0, n_sum), rank-order fmax over [n_sum, n)."""
    s = vals[0][:n_sum].clone()
    for v in vals[1:]:
        s += v[:n_sum]
    m = vals[0][n_sum:].clone()
    for v in vals[1:]:
        m = torch.maximum(m, v[n_sum:])
    return torch.cat([s, m])


def _check_reduction(N, n, n_sum, dev, seed, shared=False):
    what = f"N={N} n={n} n_sum={n_sum} shared={shared}"
    vals = _inputs(N, n, n_sum, seed, dev)
    ref = _reference(vals, n_sum)
    # the reference is what "exact" means here: the rank-order fp32 sum, within (N-1) 2^-24 sum_r |b_r| of the fp64 sum
    if n_sum:
        exact = torch.zeros(n_sum, dtype=torch.float64, device=dev)
        mag = torch.zeros(n_sum, dtype=torch.float64, device=dev)
        for v in vals:
            exact += v[:n_sum].double()
            mag += v[:n_sum].double().abs()
        assert bool(((ref[:n_sum].double() - exact).abs() <= (N - 1) * 2.0 ** -24 * mag).all()), what
        del exact, mag
    ref_bits = ref.view(torch.int32)
    buf = _Peers(N, n, dev, shared)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(seed)).tolist()
    for order in (list(range(N)), list(range(N - 1, -1, -1)), perm):
        buf.load(vals)
        _reduce(buf.peers, n_sum, n, order)
        for r, p in enumerate(buf.peers):
            assert torch.equal(p.view(torch.int32), ref_bits), (what, order, r)
        assert buf.guards_intact(), (what, order)


def _factored_layout(P):
    """(n_sum, n_reduce) of GradBucket(P, M, dev, factor_sh=True): its reduced part is the bucket's fields without dsh (11
    gradient + 5 statistics floats per Gaussian); the constructor itself needs a process group."""
    import gof_dp
    from diff_gaussian_rasterization import _C
    shapes = {name: (P,) + tail for name, tail in gof_dp._FIELDS + gof_dp._STAT_FIELDS if name != "dsh"}
    offsets, n_reduce = _C._layout(shapes)
    return offsets["dens_max"][0], n_reduce


def _sizes(N):
    """(n, n_sum) for world N: n/4 < N (empty slices), slice counts around multiples of N, n_sum on and inside slice
    boundaries, and the real bucket layouts."""
    import gof_dp
    out = [(4, 0), (4, 4), (8, 0), (8, 4), (8, 8)]
    k = 37
    for n4 in (N * k - 1, N * k, N * k + 1):
        bound = [n4 * r // N for r in range(N + 1)]          # float4 index of each rank's slice start
        inside = bound[N - 1] + (bound[N] - bound[N - 1]) // 2     # strictly inside the last rank's slice
        assert bound[N - 1] < inside < bound[N]
        out += [(4 * n4, 0), (4 * n4, 4 * n4), (4 * n4, 4 * bound[N // 2]), (4 * n4, 4 * inside)]
    for P in (1, 257, 100_003):
        b = gof_dp.GradBucket(P, 16, "meta")
        out.append((b.n_reduce, b.n_sum))
        n_sum, n_reduce = _factored_layout(P)
        out.append((n_reduce, n_sum))
    return out


@gpu
@pytest.mark.parametrize("N", range(2, 9))
def test_p2p_allreduce_every_world(N):
    """Every (n, n_sum) of _sizes at world N, in separate allocations and as views into one allocation."""
    dev = torch.device("cuda")
    for i, (n, n_sum) in enumerate(_sizes(N)):
        _check_reduction(N, n, n_sum, dev, seed=100 * N + i)
        _check_reduction(N, n, n_sum, dev, seed=1000 * N + i, shared=True)


@gpu
@pytest.mark.parametrize("N", [3, 8])
def test_p2p_allreduce_production_bucket(N):
    """The bucket of 2.5 M Gaussians (BASELINE C4): 160 M floats, so the grid-stride loop makes many passes over each slice."""
    import gof_dp
    b = gof_dp.GradBucket(2_500_000, 16, "meta")
    _check_reduction(N, b.n_reduce, b.n_sum, torch.device("cuda"), seed=7 + N)
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("N", range(2, 9))
def test_p2p_allreduce_grad_bucket_round_trip(N):
    """N GradBuckets of 100_003 Gaussians filled field by field: after the exchange every bucket's dens_max is the elementwise
    max and every other field the rank-order sum, bit for bit."""
    import gof_dp
    dev = torch.device("cuda")
    P = 100_003
    buckets = [gof_dp.GradBucket(P, 16, dev) for _ in range(N)]
    g = torch.Generator(device=dev).manual_seed(N)
    for b in buckets:
        for name, v in b.views.items():
            x = torch.randn(v.shape, generator=g, device=dev) * torch.exp2(torch.randint(-20, 21, v.shape, generator=g, device=dev).float())
            v.copy_(x.abs() if name == "dens_max" else x)
    want = {}
    for name in buckets[0].views:
        w = buckets[0].views[name].clone()
        for b in buckets[1:]:
            w = torch.maximum(w, b.views[name]) if name == "dens_max" else w.add_(b.views[name])
        want[name] = w
    _reduce([b.flat for b in buckets], buckets[0].n_sum, buckets[0].n_reduce, range(N))
    for r, b in enumerate(buckets):
        for name, w in want.items():
            assert torch.equal(b.views[name].view(torch.int32), w.view(torch.int32)), (r, name)


# ========================================================================================================================
# 2. gof_sh_grad_from_views
# ========================================================================================================================

def test_sh_oracle_against_fp64():
    """The oracle's direction and weights against fp64 (gof_dp.sh_grad_weights_torch at the oracle's own fp32 direction), each
    weight within 8 fp32 roundings of the magnitude of its terms (the degree-3 weights take up to six roundings, the
    constant's own included)."""
    import gof_dp
    rng = np.random.default_rng(3)
    means = rng.uniform(-3, 3, (20_000, 3)).astype(np.float32)
    means[:2000] *= np.float32(1e-4)                                 # near the camera centre below
    cam = np.array([1e-5, -2e-5, 3e-5], np.float32)
    d = shv.view_dir(means, cam)
    d64 = means.astype(np.float64) - cam.astype(np.float64)
    d64 /= np.linalg.norm(d64, axis=1, keepdims=True)
    assert np.abs(d - d64).max() <= 4 * 2.0 ** -24
    x, y, z = (d[:, i].astype(np.float64) for i in range(3))
    ax, ay, az = np.abs(x), np.abs(y), np.abs(z)
    xx, yy, zz = x * x, y * y, z * z
    c2, c3 = [abs(c) for c in gof_dp._SH_C2], [abs(c) for c in gof_dp._SH_C3]
    scale = np.stack([np.full_like(x, 0.28209479177387814), gof_dp._SH_C1 * ay, gof_dp._SH_C1 * az, gof_dp._SH_C1 * ax,
                      c2[0] * ax * ay, c2[1] * ay * az, c2[2] * (2 * zz + xx + yy), c2[3] * ax * az, c2[4] * (xx + yy),
                      c3[0] * ay * (3 * xx + yy), c3[1] * ax * ay * az, c3[2] * ay * (4 * zz + xx + yy), c3[3] * az * (2 * zz + 3 * xx + 3 * yy),
                      c3[4] * ax * (4 * zz + xx + yy), c3[5] * az * (xx + yy), c3[6] * ax * (xx + 3 * yy)], axis=1)
    for D in range(4):
        w = shv.grad_weights(D, d)
        w64 = gof_dp.sh_grad_weights_torch(torch.from_numpy(d.astype(np.float64)), D).numpy()
        nk = (D + 1) ** 2
        assert w.dtype == np.float32 and w.shape == (len(d), nk)
        assert (np.abs(w - w64) <= 8 * 2.0 ** -24 * scale[:, :nk]).all(), D


def test_sh_oracle_exact_at_hand_picked_directions():
    """Bit for bit at directions whose weights are known exactly: axis-aligned ones (every weight is an fp32 constant times a
    small integer) and ones where the bands' differences cancel to exactly zero -- (1,1,1): x = y = z, so 2zz - xx - yy and
    xx - yy vanish; (2,0,1): x = 2z exactly, so 4zz - xx - yy vanishes."""
    C0, C1, C2, C3 = shv.C0, shv.C1, shv.C2, shv.C3
    f = np.float32
    cam = np.array([0.5, -1.0, 2.0], np.float32)
    for off, want_nonzero in (
            ((3.0, 0.0, 0.0), {0: C0, 3: -C1, 6: -C2[2], 8: C2[4], 13: -C3[4], 15: C3[6]}),      # +x
            ((0.0, -3.0, 0.0), {0: C0, 1: C1, 6: -C2[2], 8: -C2[4], 9: C3[0], 11: C3[2]}),       # -y
            ((0.0, 0.0, 4.0), {0: C0, 2: C1, 6: f(2) * C2[2], 12: f(2) * C3[3]}),                # +z
            ((0.0, 0.0, -0.5), {0: C0, 2: -C1, 6: f(2) * C2[2], 12: f(-2) * C3[3]})):            # -z
        m = (cam + np.array(off, np.float32))[None, :]
        d = shv.view_dir(m, cam)
        w = shv.grad_weights(3, d)[0]
        want = np.zeros(16, np.float32)
        for k, v in want_nonzero.items():
            want[k] = v
        assert np.array_equal(w, want), (off, w, want)         # (+0 and -0 compare equal: the signs of zero weights vary)
    # x = y = z: the degree-2 and degree-3 weights that are differences of squares are exactly zero
    m = (cam + np.array([1.0, 1.0, 1.0], np.float32))[None, :]
    d = shv.view_dir(m, cam)
    assert d[0, 0] == d[0, 1] == d[0, 2]
    w = shv.grad_weights(3, d)[0]
    assert w[6] == 0 and w[8] == 0 and w[14] == 0
    assert all(w[k] != 0 for k in (0, 1, 2, 3, 4, 5, 7, 9, 10, 11, 12, 13, 15))
    # x = 2z, y = 0: 4zz - xx - yy is exactly zero, so w13 = 0
    m = (cam + np.array([2.0, 0.0, 1.0], np.float32))[None, :]
    d = shv.view_dir(m, cam)
    assert d[0, 0] == 2 * d[0, 2] and d[0, 1] == 0
    w = shv.grad_weights(3, d)[0]
    assert w[13] == 0 and w[12] != 0 and w[15] != 0


def _sh_case(P, M, nv, seed):
    """Means, per-view (camera centre, degree, rgb [3,P]) with unseen rows, one-channel rows, means near a camera centre (seen)
    and means exactly at one (unseen by that view: its direction would be 0/0).  View 0 sees Gaussian 0, so no case is all
    zeros."""
    rng = np.random.default_rng(seed)
    dmax = math.isqrt(M) - 1
    means = rng.uniform(-2, 2, (P, 3)).astype(np.float32)
    cams = rng.uniform(-4, 4, (nv, 3)).astype(np.float32)
    degrees = rng.integers(0, dmax + 1, nv)
    degrees[rng.integers(0, nv)] = dmax
    rgb = rng.standard_normal((nv, 3, P)).astype(np.float32)
    for v in range(nv):
        zero = rng.random(P) < 0.2
        zero[0] &= v > 0
        rgb[v][:, zero] = np.where(rng.random((3, int(zero.sum()))) < 0.5, np.float32(0.0), np.float32(-0.0))
        one = rng.random(P) < 0.1
        keep = rng.integers(0, 3, P)
        for c in range(3):
            rgb[v][c, one & (keep != c)] = 0.0
    special = rng.permutation(P)[:max(1, P // 50)]
    for j, g in enumerate(special):
        if nv > 1 and (j + seed) % 2 == 0:                        # exactly at view v's centre, which therefore does not see it
            v = int(rng.integers(1, nv))
            means[g] = cams[v]
            rgb[v][:, g] = 0.0
        else:                                                     # close to it, seen: a tiny difference, direction still exact
            v = int(rng.integers(0, nv))
            step = rng.choice([1e-3, 1e-5, 0.0], 3).astype(np.float32) * rng.choice([-1, 1], 3).astype(np.float32)
            step[int(rng.integers(0, 3))] = 0.0
            means[g] = cams[v] + step
            if (means[g] == cams[v]).all():
                means[g][0] = np.nextafter(cams[v][0], np.float32(np.inf))
            rgb[v][:, g] = rng.standard_normal(3).astype(np.float32)
    return means, cams, degrees, rgb


def _sh_records(cams, degrees, rgb, dev):
    """One allocation per view: 64-float header (camera centre, degree; the rest NaN) and three NaN-padded colour planes."""
    nv, _, P = rgb.shape
    plane = shv.sh_plane(P)
    recs = []
    for v in range(nv):
        rec = np.full(shv.SLOT_HEADER + 3 * plane, np.nan, np.float32)
        rec[:3], rec[3] = cams[v], degrees[v]
        rec[shv.SLOT_HEADER:].reshape(3, plane)[:, :P] = rgb[v]
        recs.append(rec)
    return recs, [torch.from_numpy(r).to(dev) for r in recs]


def _sh_kernel(means_t, recs_t, P, M):
    """gof_sh_grad_from_views into a NaN-filled output followed by GUARD NaN-pattern floats: (dL_dsh [P,M,3], guard intact)."""
    from diff_gaussian_rasterization import _C
    out = _nan_fill(P * M * 3 + GUARD, means_t.device)
    ptrs = (ctypes.c_void_p * len(recs_t))(*[r.data_ptr() for r in recs_t])
    _C._check(_C._lib.gof_sh_grad_from_views(P, M, len(recs_t), means_t.data_ptr(), ptrs, out.data_ptr(), _C._stream()))
    torch.cuda.synchronize()
    return out[:P * M * 3].view(P, M, 3), bool((out[P * M * 3:].view(torch.int32) == NAN_BITS).all())


_SH_NV = (1, 2, 3, 4, 5, 8, 9, 15, 16)        # every NV instantiation (2, 4, 8, 16) and both sides of each bound
_SH_M = (1, 4, 9, 16)
_SH_P = (1, 31, 32, 33, 127, 128, 129, 4097)
_SH_CASES = [(P, M, _SH_NV[(4 * i + j) % len(_SH_NV)]) for i, P in enumerate(_SH_P) for j, M in enumerate(_SH_M)] + \
    [(1_000_003, 16, 16), (1_000_003, 9, 5)]


@gpu
@pytest.mark.parametrize("P,M,nv", _SH_CASES)
def test_sh_grad_from_views_matches_oracle(P, M, nv):
    dev = torch.device("cuda")
    means, cams, degrees, rgb = _sh_case(P, M, nv, seed=P * 131 + M * 17 + nv)
    recs, recs_t = _sh_records(cams, degrees, rgb, dev)
    got, guard_ok = _sh_kernel(torch.from_numpy(means).to(dev), recs_t, P, M)
    want = shv.sh_grad_from_views(means, recs, P, M)
    assert np.isfinite(want).all() and np.abs(want).max() > 0
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
    assert guard_ok


@gpu
@pytest.mark.parametrize("M,P,degrees", [(1, 4_097, (0, 0, 0)), (4, 2_051, (1, 0, 1, 1, 1)), (9, 1_027, (2, 1, 2, 0, 2, 2, 1, 2, 2)),
                                         (9, 30_011, (2, 2))])
def test_factored_sh_gradient_is_the_sum_of_the_views_below_degree3(M, P, degrees):
    """test_gpu_bucket's real-backward identity at M < 16 (the kernel's scalar store path): a rasterizer backward per view at
    sh_degree <= sqrt(M) - 1 leaves its record and its own dL_dsh (P,M,3); the kernel's sum over the records (each in its own
    allocation) equals the views' dL_dsh added in view order (bit for bit up to the sign of a zero sum) and the oracle (bit for
    bit)."""
    import _util
    import gof_dp
    import gof_synth
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    H, W = 208, 320
    plane = shv.sh_plane(P)
    grad = torch.randn(9, H, W, generator=torch.Generator().manual_seed(2)).to(dev)
    want, means, recs_t = None, None, []
    for i, deg in enumerate(degrees):
        cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=17), view=(4 + 7 * i) % 64)
        gs = dict(gs, shs=gs["shs"][:, :M, :].contiguous())
        fa = _util.fwd_args(cam, gs, dev, sh_degree=deg)
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
        rec = torch.full((gof_dp.SH_SLOT_HEADER + 3 * plane,), float("nan"), device=dev)
        full = torch.full((P, M, 3), float("nan"), device=dev)
        out = {"sh_hdr": rec[:gof_dp.SH_SLOT_HEADER], "dsh_rgb": rec[gof_dp.SH_SLOT_HEADER:].view(3, plane), "_dsh_full": full}
        _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad), _out=out)
        torch.cuda.synchronize()
        assert float(rec[3]) == deg and not torch.isnan(full).any()
        rec[gof_dp.SH_SLOT_HEADER:].view(3, plane)[:, P:] = float("nan")     # a read past P shows up
        want = full.clone() if want is None else want + full
        means = fa[1]
        recs_t.append(rec)
    got, guard_ok = _sh_kernel(means, recs_t, P, M)
    assert float(want.abs().max()) > 0 and guard_ok
    # Bit for bit wherever the views' sum is non-zero.  A coefficient that every view left at zero comes out +0 (the kernel's
    # accumulator starts at +0, and it skips rows whose dL_dRGB is all zero), while the views' sum is -0 where every view wrote
    # -0 (w_k < 0 times a +0 dL_dRGB, or a clamped channel's -0).  The record cannot carry that sign: an unseen Gaussian's row
    # is written +0, a seen one's all-zero dL_dRGB gives fl(w_k * 0) of either sign.
    nz = want != 0
    assert torch.equal(got, want)
    assert torch.equal(got.view(torch.int32)[nz], want.view(torch.int32)[nz])
    assert bool((got.view(torch.int32)[~nz] == 0).all())
    oracle = shv.sh_grad_from_views(means.cpu().numpy(), [r.cpu().numpy() for r in recs_t], P, M)
    assert np.array_equal(got.cpu().numpy().view(np.int32), oracle.view(np.int32))


# ========================================================================================================================
# 3. Host-side refusals, without a device
# ========================================================================================================================

_REFUSAL_SCRIPT = textwrap.dedent("""
    import ctypes, json, sys
    lib = ctypes.CDLL(sys.argv[1])
    lib.gof_last_error.restype = ctypes.c_char_p
    v, i, z = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    for f in (lib.gof_p2p_allreduce_f32, lib.gof_nvls_allreduce_f32):
        f.restype = i
        f.argtypes = [v, i, i, z, z, v]
    lib.gof_sh_grad_from_views.restype = i
    lib.gof_sh_grad_from_views.argtypes = [i, i, i, v, v, v, v]
    A = 1 << 20                                  # stand-in device addresses: every case must return before any CUDA call
    def peers(bad=None, shift=0):
        p = [A + 4096 * k for k in range(9)]
        if bad is not None:
            p[bad] = None if shift is None else p[bad] + shift
        return (v * 9)(*p)
    out = {}
    def call(name, f, *args):
        out[name] = [f(*args), lib.gof_last_error().decode()]
    p2p, nvls, shv = lib.gof_p2p_allreduce_f32, lib.gof_nvls_allreduce_f32, lib.gof_sh_grad_from_views
    call("p2p_world0", p2p, peers(), 0, 0, 0, 16, None)
    call("p2p_rank_eq_world", p2p, peers(), 2, 2, 0, 16, None)
    call("p2p_rank_negative", p2p, peers(), 2, -1, 0, 16, None)
    call("p2p_n_not_x4", p2p, peers(), 2, 0, 0, 18, None)
    call("p2p_n_sum_not_x4", p2p, peers(), 2, 0, 2, 16, None)
    call("p2p_n_sum_gt_n", p2p, peers(), 2, 0, 20, 16, None)
    call("p2p_world9", p2p, peers(), 9, 0, 0, 16, None)
    call("p2p_peers_null", p2p, None, 2, 0, 0, 16, None)
    call("p2p_peer_null", p2p, peers(3, None), 4, 0, 0, 16, None)
    call("p2p_peer_unaligned", p2p, peers(5, 8), 8, 0, 0, 16, None)
    call("p2p_world1", p2p, peers(), 1, 0, 8, 16, None)
    call("p2p_n0", p2p, peers(), 4, 3, 0, 0, None)
    call("nvls_world0", nvls, A, 0, 0, 0, 16, None)
    call("nvls_rank_eq_world", nvls, A, 2, 2, 0, 16, None)
    call("nvls_rank_negative", nvls, A, 2, -1, 0, 16, None)
    call("nvls_n_not_x4", nvls, A, 2, 0, 0, 18, None)
    call("nvls_n_sum_not_x4", nvls, A, 2, 0, 2, 16, None)
    call("nvls_n_sum_gt_n", nvls, A, 2, 0, 20, 16, None)
    call("nvls_mc_null", nvls, None, 2, 0, 0, 16, None)
    call("nvls_mc_unaligned", nvls, A + 4, 2, 0, 0, 16, None)
    call("nvls_world1", nvls, A, 1, 0, 8, 16, None)
    call("nvls_n0", nvls, A, 4, 3, 0, 0, None)
    call("nvls_world1000_n0", nvls, A, 1000, 999, 0, 0, None)   # no upper bound on the world size
    slots = (v * 17)(*[A + 65536 * k for k in range(17)])
    call("shv_M0", shv, 100, 0, 2, A, slots, A, None)
    call("shv_M17", shv, 100, 17, 2, A, slots, A, None)
    call("shv_views0", shv, 100, 16, 0, A, slots, A, None)
    call("shv_views17", shv, 100, 16, 17, A, slots, A, None)
    call("shv_P_negative", shv, -1, 16, 2, A, slots, A, None)
    call("shv_slots_null", shv, 100, 16, 2, A, None, A, None)
    call("shv_slot_null", shv, 100, 16, 3, A, (v * 3)(A, None, A), A, None)
    call("shv_out_unaligned", shv, 100, 9, 2, A, slots, A + 4, None)
    call("shv_means_null", shv, 100, 9, 2, None, slots, A, None)
    call("shv_P0", shv, 0, 16, 2, A, slots, A, None)
    print(json.dumps(out))
""")


def test_exchange_entry_points_refuse_bad_arguments_without_a_device():
    """CPU: gof_p2p_allreduce_f32, gof_nvls_allreduce_f32 and gof_sh_grad_from_views refuse every malformed argument with
    GOF_E_INVALID on the host, and return GOF_OK for the calls that have nothing to do (world 1, n == 0, P == 0) -- all in a
    process that sees no device, so none of these reaches a CUDA call.  gof_nvls_allreduce_f32 has no upper bound on the world
    size (the multicast object bounds it); gof_p2p_allreduce_f32 takes at most 8 peers."""
    assert os.path.exists(LIB_PATH), "build the library first: python gaussian-opacity-fields_b200/build.py"
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _REFUSAL_SCRIPT, LIB_PATH], env=env, capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    out = json.loads(res.stdout.strip().splitlines()[-1])
    ok = {"p2p_world1", "p2p_n0", "nvls_world1", "nvls_n0", "nvls_world1000_n0", "shv_P0"}
    prefix = {"p2p": "p2p_allreduce", "nvls": "nvls_allreduce", "shv": "sh_grad_from_views"}
    for name, (rc, msg) in out.items():
        if name in ok:
            assert rc == GOF_OK, (name, rc, msg)
        else:
            assert rc == GOF_E_INVALID and msg.startswith(prefix[name.split("_")[0]]), (name, rc, msg)
    for name in ("p2p_peer_null", "p2p_peer_unaligned"):
        assert "peer pointer" in out[name][1], out[name]
    for name in ("shv_slot_null",):
        assert "view record" in out[name][1], out[name]
    for name in ("shv_out_unaligned", "shv_means_null"):
        assert "unaligned" in out[name][1], out[name]
