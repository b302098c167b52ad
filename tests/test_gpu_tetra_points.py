"""GPU: gof_extract.get_tetra_points / get_frustum_mask (csrc/tetra_points.cu) against the reference's own
GaussianModel.get_tetra_points and get_frustum_mask (scene/gaussian_model.py:31-72, 433-463; run from the staged source on the
GPU) and against the numpy oracle (oracle/tetra_points_oracle.py).

Parity rule (DESIGN §4.8): the point scales and the centres are bit-identical; a corner is within the rounding bound of the
3-term product of both evaluations (2 x the oracle's one-evaluation bound); the mask equals the reference's at every point the
float64 decision settles beyond the rounding bound of the float32 evaluation, widened by how far the reference's corner may
lie from ours.  Undecided and disagreeing counts are printed."""
import numpy as np
import pytest
import torch

import _tetra_scenes as ts
import tetra_points_oracle as tpo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# growth of torch.cuda.max_memory_allocated during one get_tetra_points call: the unmasked points, scales and mask (153 B), the
# int64 indices of the boolean selection (72 B) and the selected points and scales (up to 144 B), per Gaussian
BYTES_PER_GAUSSIAN = 400


def _lib():
    import gof_extract
    return gof_extract._tetra_lib()[1]


def _raw(xyz, s, r, table, near=0.02, far=1e6, pad=0):
    """The unmasked outputs of gof_tetra_points, with `pad` guard elements after each output."""
    P = xyz.shape[0]
    pts = torch.full((9 * P * 3 + pad,), 12345.0, device=DEV)
    sc = torch.full((9 * P + pad,), 12345.0, device=DEV)
    m = torch.full((9 * P + pad,), 7, dtype=torch.uint8, device=DEV)
    rc = _lib().gof_tetra_points(P, xyz.data_ptr(), s.data_ptr(), r.data_ptr(), table.shape[0], table.data_ptr(), near, far,
                                 pts.data_ptr(), sc.data_ptr(), m.data_ptr(), None)
    assert rc == 0
    torch.cuda.synchronize()
    return pts, sc, m


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _check_against_oracle(tag, xyz, s, r, views, pts, sc, m, idx=None):
    """ours (unmasked, on the host) against the oracle at Gaussians `idx` (all by default)."""
    P = xyz.shape[0]
    idx = np.arange(P) if idx is None else idx
    rows = np.concatenate([(8 * idx[:, None] + np.arange(8)[None, :]).reshape(-1), 8 * P + idx])
    opts, obnd, osc = tpo.tetra_points(xyz[idx], s[idx], r[idx])
    o_rows = np.concatenate([np.arange(8 * len(idx)), 8 * len(idx) + np.arange(len(idx))])
    got, gsc, gm = pts.reshape(-1, 3)[rows], sc[rows], m[rows].astype(bool)
    assert _same_bits(gsc, osc[o_rows]) and _same_bits(got[8 * len(idx):], xyz[idx])
    fin = np.isfinite(opts).all(1)
    assert (np.abs(got[fin] - opts[fin]) <= obnd[fin]).all(), tag
    mask64, decided = tpo.frustum_decision(got, tpo.pack_views(views))
    bad = decided & (gm != mask64)
    print(f"[tetra gpu/oracle {tag}] points {gm.size}  in {int(gm.sum())}  undecided {int((~decided).sum())}  disagreeing {int(bad.sum())}")
    assert not bad.any()
    return gm


@pytest.mark.parametrize("kind,P,n_views,W,H", [("random", 200_000, 64, 1920, 1080), ("surface", 200_000, 64, 1600, 1200),
                                                ("surface", 50_000, 6, 800, 600)])
def test_against_reference_source(kind, P, n_views, W, H):
    import gof_extract
    xyz, s, r = ts.gaussians(P, 100 + n_views, kind)
    views = (ts.surface_views if kind == "surface" else ts.ring_views)(n_views, W, H, device=DEV)
    if n_views > 2:   # the quirk: a view whose size differs from views[0]'s, which the reference uses for every view
        views[2].image_width, views[2].image_height = W // 2, H // 2
    x, sg, rg = xyz.to(DEV), s.to(DEV), r.to(DEV)
    pts, sc = gof_extract.get_tetra_points(x, sg, rg, views)
    table = gof_extract.pack_views(views, DEV)
    rp, rs, rm = _raw(x, sg, rg, table)
    keep = rm.bool()
    assert torch.equal(pts, rp.reshape(-1, 3)[keep]) and torch.equal(sc, rs.reshape(-1, 1)[keep])
    ours_m = _check_against_oracle(kind, xyz.numpy(), s.numpy(), r.numpy(), views, rp.cpu().numpy(), rs.cpu().numpy(), rm.cpu().numpy())
    assert torch.equal(gof_extract.get_frustum_mask(rp.reshape(-1, 3), views), keep)

    ref = ts.ref_tetra_points(x, sg, rg, views)
    if ref is None:
        pytest.skip("the reference's scene/gaussian_model.py is not staged (baseline/stage_ref.sh)")
    ref_pts, ref_sc, ref_verts, ref_mask = ref
    torch.cuda.synchronize()
    ours = rp.reshape(-1, 3).cpu().numpy()
    theirs, tm = ref_verts.cpu().numpy(), ref_mask.cpu().numpy()
    assert _same_bits(theirs[8 * P:], ours[8 * P:])                                     # centres
    _o, obnd, osc = tpo.tetra_points(xyz.numpy(), s.numpy(), r.numpy())
    assert _same_bits(ref_sc.cpu().numpy()[:, 0], osc[tm])                              # point scales
    fin = np.isfinite(ours).all(1)
    assert (np.abs(ours[fin] - theirs[fin]) <= 2 * obnd[fin]).all()
    same_corners = int((ours[:8 * P].view(np.uint32) == theirs[:8 * P].view(np.uint32)).all(1).sum())
    mask64, decided = tpo.frustum_decision(ours, tpo.pack_views(views), pos_err=2 * obnd)
    bad = decided & (ours_m != tm)
    print(f"[tetra gpu/reference {kind} P={P} views={n_views}] corners bit-identical {same_corners}/{8 * P}  points {tm.size}  "
          f"in {int(tm.sum())}  undecided {int((~decided).sum())}  disagreeing {int(bad.sum())}  "
          f"mask differs at {int((ours_m != tm).sum())}")
    assert not bad.any()
    assert ref_pts.shape[0] == int(tm.sum()) and torch.equal(ref_pts, ref_verts[ref_mask])


def test_edge_points_and_quirk():
    import gof_extract
    view, pts, exp = ts.edge_scene(device=DEV)
    p = torch.from_numpy(pts).to(DEV)
    assert np.array_equal(gof_extract.get_frustum_mask(p, [view]).cpu().numpy(), exp)
    # a second view of a different size: the reference still bounds it by views[0]'s W and H
    big = ts.Cam(torch.eye(4, device=DEV), 32.0, 32.0, 4096, 4096)
    q = torch.tensor([[-1.5, 0.0, 1.0], [0.0, 0.0, 1.0], [1.2, 0.0, 1.0]], device=DEV)   # u = -16, 32, 70.4 with cx = 32
    assert gof_extract.get_frustum_mask(q, [view, big]).tolist() == [False, True, False]
    assert gof_extract.get_frustum_mask(q, [big, view]).tolist() == [True, True, True]
    ref = ts.ref_frustum_mask()
    if ref is not None:
        assert np.array_equal(ref(p, [view]).cpu().numpy(), exp)
        assert ref(q, [view, big]).tolist() == [False, True, False] and ref(q, [big, view]).tolist() == [True, True, True]
    for near, far in ((0.5, 7.0), (1e-3, 1e3)):
        view, pts, exp = ts.edge_scene(near, far, device=DEV)
        assert np.array_equal(gof_extract.get_frustum_mask(torch.from_numpy(pts).to(DEV), [view], near, far).cpu().numpy(), exp)


def test_degenerate_inputs():
    import gof_extract
    view, _pts, _exp = ts.edge_scene(device=DEV)
    e3, e4 = torch.zeros(0, 3, device=DEV), torch.zeros(0, 4, device=DEV)
    pts, sc = gof_extract.get_tetra_points(e3, e3, e4, [view])
    assert pts.shape == (0, 3) and sc.shape == (0, 1)
    with pytest.raises(ValueError):
        gof_extract.get_tetra_points(e3, e3, e4, [])
    with pytest.raises(ValueError):
        gof_extract.get_frustum_mask(torch.zeros(4, 3, device=DEV), [])
    with pytest.raises(RuntimeError):
        gof_extract.get_tetra_points(torch.zeros(1, 3), torch.ones(1, 3), torch.ones(1, 4), [view])
    with pytest.raises(RuntimeError):
        gof_extract.get_frustum_mask(torch.zeros(4, 3, device=DEV, dtype=torch.float64), [view])
    # centres in front of the single view: a zero quaternion (NaN corners, centre kept), a NaN scale (NaN point scale),
    # a point behind the camera, non-finite centres
    xyz = torch.tensor([[0.0, 0.0, 2.0], [0.1, 0.0, 2.0], [0.0, 0.0, -2.0], [np.inf, 0.0, 2.0], [0.0, np.nan, 2.0]], device=DEV)
    s = torch.full((5, 3), 0.01, device=DEV)
    s[1, 2] = float("nan")
    r = torch.tensor([[0.0, 0.0, 0.0, 0.0], [2.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0]],
                     device=DEV)
    table = gof_extract.pack_views([view], DEV)
    rp, rs, rm = _raw(xyz, s, r, table)
    P = 5
    m = rm.cpu().numpy().astype(bool)
    pts3 = rp.reshape(-1, 3).cpu().numpy()
    assert np.isnan(pts3[0:8]).all() and not m[0:8].any() and m[8 * P + 0]
    assert np.isnan(rs.cpu().numpy()[list(range(8, 16)) + [8 * P + 1]]).all() and np.isnan(pts3[8:16]).all()
    assert not m[8:16].any() and m[8 * P + 1]
    assert not m[16:24].any() and not m[8 * P + 2]
    assert not m[24:40].any() and not m[8 * P + 3] and not m[8 * P + 4]
    _check_against_oracle("degenerate", xyz.cpu().numpy(), s.cpu().numpy(), r.cpu().numpy(), [view], rp.cpu().numpy(), rs.cpu().numpy(),
                          rm.cpu().numpy())


def test_misaligned_rotations_and_many_views():
    import gof_extract
    P = 2000
    xyz, s, r = ts.gaussians(P, 7)
    views = ts.ring_views(1100, 640, 360, device=DEV)
    flat = torch.empty(4 * P + 1, device=DEV)
    flat[1:] = r.reshape(-1).to(DEV)
    r_mis = flat[1:].view(P, 4)
    assert r_mis.data_ptr() & 15
    x, sg = xyz.to(DEV), s.to(DEV)
    a = gof_extract.get_tetra_points(x, sg, r_mis, views)
    b = gof_extract.get_tetra_points(x, sg, r.to(DEV), views)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    table = gof_extract.pack_views(views, DEV)
    rp, rs, rm = _raw(x, sg, r.to(DEV), table)
    _check_against_oracle("1100 views", xyz.numpy(), s.numpy(), r.numpy(), views, rp.cpu().numpy(), rs.cpu().numpy(), rm.cpu().numpy())
    # 1500 views that look away from the edge points, then the one that sees them: the search runs past 1024 views
    view, pts, exp = ts.edge_scene(device=DEV)
    shifted = torch.eye(4, device=DEV)
    shifted[3, 2] = -1e7                           # depth = z - 1e7: every finite point lies behind this camera
    away = ts.Cam(shifted, 32.0, 32.0, 64, 48)
    p = torch.from_numpy(pts).to(DEV)
    assert not gof_extract.get_frustum_mask(p, [away] * 1500).any()
    assert np.array_equal(gof_extract.get_frustum_mask(p, [away] * 1500 + [view]).cpu().numpy(), exp)
    centres = p[exp]
    tp, _tsc = gof_extract.get_tetra_points(centres, torch.full_like(centres, 1e-4), torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(
        centres.shape[0], 4).contiguous(), [away] * 1500 + [view])
    assert tp.shape[0] > 0


def test_determinism_guards_and_refusals():
    import gof_extract
    P = 100_000
    xyz, s, r = (t.to(DEV) for t in ts.gaussians(P, 3))
    views = ts.ring_views(64, 800, 600, device=DEV)
    table = gof_extract.pack_views(views, DEV)
    pad = 4096
    a = _raw(xyz, s, r, table, pad=pad)
    b = _raw(xyz, s, r, table, pad=pad)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8), v.view(torch.uint8))
    assert (a[0][-pad:] == 12345.0).all() and (a[1][-pad:] == 12345.0).all() and (a[2][-pad:] == 7).all()
    assert set(a[2][:-pad].unique().tolist()) <= {0, 1}
    mk = torch.full((9 * P + pad,), 7, dtype=torch.uint8, device=DEV)
    lib = _lib()
    assert lib.gof_frustum_mask(9 * P, a[0].data_ptr(), 64, table.data_ptr(), 0.02, 1e6, mk.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert torch.equal(mk[:-pad], a[2][:-pad]) and (mk[-pad:] == 7).all()

    p, q = xyz.data_ptr(), r.data_ptr()
    assert lib.gof_tetra_points(-1, p, p, q, 64, table.data_ptr(), 0.02, 1e6, p, p, p, None) == -1
    assert lib.gof_tetra_points(477218589, p, p, q, 64, table.data_ptr(), 0.02, 1e6, p, p, p, None) == -1    # 9 P = 2^32 + 5
    assert lib.gof_tetra_points(10, p, p, q, 0, table.data_ptr(), 0.02, 1e6, p, p, p, None) == -1
    assert lib.gof_tetra_points(10, p, p, q + 4, 64, table.data_ptr(), 0.02, 1e6, p, p, p, None) == -1
    assert b"aligned" in lib.gof_last_error()
    assert lib.gof_frustum_mask(-1, p, 64, table.data_ptr(), 0.02, 1e6, p, None) == -1
    assert lib.gof_frustum_mask(10, p, 0, table.data_ptr(), 0.02, 1e6, p, None) == -1


def test_c5_scale():
    """C5: 3 M Gaussians, 64 views at 1920x1080 -- the reference's mask alone would need ~70 GB."""
    import gof_extract
    import gof_synth
    cfg = gof_synth.CONFIGS["C5"]
    P = cfg["P"]
    xyz, s, r = ts.gaussians(P, cfg["seed"])
    views = ts.ring_views(cfg["n_views"], cfg["width"], cfg["height"], device=DEV)
    x, sg, rg = xyz.to(DEV), s.to(DEV), r.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    pts, sc = gof_extract.get_tetra_points(x, sg, rg, views)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated(DEV) - base
    print(f"[tetra C5] P={P} kept {pts.shape[0]}/{9 * P}  peak growth {growth / 2**20:.0f} MiB = {growth / P:.1f} B/Gaussian")
    assert growth <= BYTES_PER_GAUSSIAN * P + (64 << 20)
    assert pts.shape[0] > 0.5 * 9 * P
    del pts, sc
    rp, rs, rm = _raw(x, sg, rg, gof_extract.pack_views(views, DEV))
    idx = np.sort(np.random.default_rng(0).choice(P, 20_000, replace=False))
    rows = np.concatenate([(8 * idx[:, None] + np.arange(8)[None, :]).reshape(-1), 8 * P + idx])
    rows_t = torch.from_numpy(rows).to(DEV)
    sub_pts = torch.zeros(9 * P, 3)
    sub_sc, sub_m = torch.zeros(9 * P), torch.zeros(9 * P, dtype=torch.uint8)
    sub_pts[rows] = rp.reshape(-1, 3)[rows_t].cpu()
    sub_sc[rows] = rs[rows_t].cpu()
    sub_m[rows] = rm[rows_t].cpu()
    _check_against_oracle("C5 sample", xyz.numpy(), s.numpy(), r.numpy(), views, sub_pts.numpy(), sub_sc.numpy(), sub_m.numpy(), idx=idx)
