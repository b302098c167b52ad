"""CPU oracle of the opacity field's voxel-block lattice (DESIGN section 4.15) -- TEST INFRASTRUCTURE ONLY.

numpy float32, bit for bit with csrc/field_grid.cu and the field layout of csrc/tsdf.cu's marching cubes:

* blocks: the frustum test of each Gaussian's centre and its eight 3-sigma box corners exactly as csrc/tetra_points.cuh
  computes them -- the rotation from tetra_points_oracle.frame (bit-exact), the corners' and the view transform's FMA chains
  through fma32, an exactly rounded fused multiply-add -- then the box dilated by one voxel and its block range;
* lattice points: voxel (x, y, z) = key B + (i, j, k) at (f32(x) s, f32(y) s, f32(z) s) in pool order;
* marching cubes: the faces and interpolated vertices are tsdf_oracle's extraction of a volume whose tsdf is the field's values,
  weight 1 everywhere and threshold 0; the edge of every vertex (its two lattice points and their values) is derived here on
  its own, from the meshed cubes, in the extraction's canonical vertex order.
"""
import numpy as np

import tetra_points_oracle as tpo
import tsdf_oracle as T

f32, f64 = np.float32, np.float64
KEY_BIAS = T.KEY_BIAS
BlockRangeError = T.BlockRangeError
MAX_INSTANCES = 1 << 30
MAX_POINTS = 1 << 31


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c), elementwise.  a b is exact in float64; s = fl64(a b + c) with its exact error e
    (TwoSum); rounding s to float32 is then exact unless s is a float32 rounding midpoint, where the sign of e decides."""
    a, b, c = (np.asarray(x, f32).astype(f64) for x in (a, b, c))
    p = a * b
    with np.errstate(all="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        r = s.astype(f32)
        d = s - r.astype(f64)
        nb = np.nextafter(r, np.where(d > 0, f32(np.inf), f32(-np.inf)).astype(f32))
        mid = (r.astype(f64) + nb.astype(f64)) / 2
        fix = (d != 0) & (s == mid) & (e != 0) & (np.sign(e) == np.sign(d))
    return np.where(fix, nb, r).astype(f32)


def corners(xyz, scales, rotation):
    """[P,8,3] float32: the box corners of csrc/tetra_points.cuh's tp_corner (corner k with signs (sx, sy, sz), sz fastest)."""
    R, s3, _ps = tpo.frame(rotation, scales)
    x = np.asarray(xyz, f32)
    out = np.empty((x.shape[0], 8, 3), f32)
    for k in range(8):
        v = tpo.BOX_SIGNS[k][None, :] * s3                           # exact: sign flips
        for i in range(3):
            acc = np.zeros(x.shape[0], f32)
            for j in range(3):
                acc = fma32(R[:, i, j], v[:, j], acc)
            out[:, k, i] = acc + x[:, i]
    return out


def in_view(p, table, near=0.02, far=1e6):
    """[N] bool: tp_first_view(p) >= 0 -- some view's frustum holds p (width and height of views[0])."""
    p = np.asarray(p, f32)
    t = np.asarray(table, f32)
    W, H = t[0, 18], t[0, 19]
    near, far = f32(near), f32(far)
    hit = np.zeros(p.shape[0], bool)
    zero = np.zeros(p.shape[0], f32)
    for vw in t:
        vp = []
        for b in range(3):
            acc = fma32(vw[b], p[:, 0], zero)
            acc = fma32(vw[4 + b], p[:, 1], acc)
            acc = fma32(vw[8 + b], p[:, 2], acc)
            vp.append(fma32(vw[12 + b], f32(1), acc))
        fx, fy, cx, cy = vw[16], vw[17], W * f32(0.5), H * f32(0.5)
        un = fma32(cx, vp[2], fma32(f32(0), vp[1], fma32(fx, vp[0], zero)))
        vn = fma32(cy, vp[2], fma32(fy, vp[1], fma32(f32(0), vp[0], zero)))
        zp = fma32(f32(1), vp[2], fma32(f32(0), vp[1], fma32(f32(0), vp[0], zero)))
        with np.errstate(all="ignore"):
            u, v = un / zp, vn / zp
            hit |= (vp[2] >= near) & (vp[2] <= far) & (u >= 0) & (u <= W - f32(1)) & (v >= 0) & (v <= H - f32(1))
    return hit


def boxes(xyz, scales, rotation, table, voxel_size, near=0.02, far=1e6):
    """(seen [P] bool, lo [P,3], hi [P,3] float32): the Gaussians whose centre some view holds, and their corner extent dilated by
    one voxel s (a NaN corner makes the box NaN)."""
    s = f32(voxel_size)
    P = int(np.asarray(xyz).shape[0])
    if P == 0:
        return np.zeros(0, bool), np.zeros((0, 3), f32), np.zeros((0, 3), f32)
    c = corners(xyz, scales, rotation)
    lo = (np.min(c, axis=1) - s).astype(f32)            # np.min / np.max propagate NaN
    hi = (np.max(c, axis=1) + s).astype(f32)
    return in_view(xyz, table, near, far), lo, hi


def blocks(xyz, scales, rotation, table, voxel_size, block_resolution=8, near=0.02, far=1e6):
    """Sorted unique int64 keys of the blocks the seen Gaussians touch: floor(lo / fl(B s)) .. floor(hi / fl(B s)) per axis."""
    seen, lo, hi = boxes(xyz, scales, rotation, table, voxel_size, near, far)
    bs = f32(f32(block_resolution) * f32(voxel_size))
    with np.errstate(invalid="ignore"):
        a = np.floor(lo[seen] / bs)
        b = np.floor(hi[seen] / bs)
    if a.size and not (np.all(a >= -KEY_BIAS) and np.all(b < KEY_BIAS)):
        raise BlockRangeError("touched block outside [-2^20, 2^20)")
    a, b = a.astype(np.int64), b.astype(np.int64)
    ext = b - a + 1
    if int(np.prod(ext, axis=1).sum()) >= MAX_INSTANCES:
        raise ValueError("2^30 or more (Gaussian, block) instances")
    n = np.prod(ext, axis=1)
    g = np.repeat(np.arange(a.shape[0]), n)                 # every (Gaussian, block) instance, x fastest within its box
    j = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    ex, ey = ext[g, 0], ext[g, 1]
    b3 = np.stack([a[g, 0] + j % ex, a[g, 1] + (j // ex) % ey, a[g, 2] + j // (ex * ey)], 1)
    return np.unique(T.pack_keys(b3))


def voxels(keys, block_resolution):
    """[n B^3, 3] int64 global voxel coordinates of the blocks `keys`, in pool order."""
    B = int(block_resolution)
    lin = np.arange(B ** 3)
    local = np.stack([lin % B, (lin // B) % B, lin // (B * B)], 1)
    return (T.unpack_keys(np.asarray(keys, np.int64))[:, None, :] * B + local[None]).reshape(-1, 3)


def lattice_points(keys, voxel_size, block_resolution=8):
    if len(keys) * int(block_resolution) ** 3 >= MAX_POINTS:
        raise ValueError("the lattice must have fewer than 2^31 points")
    return (voxels(keys, block_resolution).astype(f32) * f32(voxel_size)).astype(f32)


def _lookup(keys, B, g):
    """Pool index of the voxels with global coordinates g [m,3], -1 where their block is not listed."""
    keys = np.asarray(keys, np.int64)
    b = np.floor_divide(g, B)
    ok = np.all(b < KEY_BIAS, axis=1) & np.all(b >= -KEY_BIAS, axis=1)
    k = np.where(ok, T.pack_keys(np.where(ok[:, None], b, 0)), -1)
    pos = np.clip(np.searchsorted(keys, k), 0, max(keys.size - 1, 0))
    found = ok & (keys.size > 0) & (keys[pos] == k) if keys.size else np.zeros(g.shape[0], bool)
    loc = g - b * B
    return np.where(found, pos * B ** 3 + loc[:, 0] + B * loc[:, 1] + B * B * loc[:, 2], -1)


def marching_cubes(keys, values, voxel_size, block_resolution=8):
    """dict(faces [F,3] int64, vertices [V,3] (interpolated, tsdf_oracle's), edge_points [V,2,3], edge_values [V,2]) of the
    field values [n B^3] (pool order) on the lattice of `keys`."""
    keys = np.asarray(keys, np.int64)
    B, s = int(block_resolution), f32(voxel_size)
    n3 = B ** 3
    v = np.asarray(values, f32).reshape(-1)
    vol = T.Volume(voxel_size=s, block_resolution=B)
    vol.keys = keys.copy()
    vol.tsdf = v.reshape(-1, n3).copy()
    vol.weight = np.ones_like(vol.tsdf)
    vol.color = np.zeros((keys.size, 3, n3), f32)
    mesh = vol.extract_triangle_mesh(0.0)
    # the edges: every crossing edge of a cube whose eight corners are listed, owned by its lower voxel
    G = voxels(keys, B)
    idx = np.stack([_lookup(keys, B, G + T.CORNER_OFF[c]) for c in range(8)], 1)     # [N, 8] corner pool indices
    meshed = np.all(idx >= 0, axis=1)
    neg = np.where(idx >= 0, v[np.maximum(idx, 0)] < 0, False)
    owners = []
    for e in range(12):
        a, b = T.EDGE_OWNER[e], T.EDGE_FAR[e]
        cross = meshed & (neg[:, a] != neg[:, b])
        owners.append(idx[cross, a] * 3 + e // 4)
    vid = np.unique(np.concatenate(owners)) if owners else np.zeros(0, np.int64)
    own, axis = vid // 3, vid % 3
    far_g = G[own] + np.eye(3, dtype=np.int64)[axis]
    far = _lookup(keys, B, far_g)
    assert np.all(far >= 0)
    pts_o = (G[own].astype(f32) * s).astype(f32)
    pts_f = (far_g.astype(f32) * s).astype(f32)
    edge_points = np.stack([pts_o, pts_f], 1).reshape(-1, 2, 3)
    edge_values = np.stack([v[own], v[far]], 1).reshape(-1, 2)
    return {"faces": mesh["faces"], "vertices": mesh["vertices"], "edge_points": edge_points, "edge_values": edge_values}


def brute_force_blocks(lo, hi, bs):
    """Reference for blocks() from the boxes alone: every candidate block b with [b bs, (b+1) bs) meeting [lo, hi] on each axis,
    in float64 -- the floor rule's meaning when the quotients are exact (power-of-two voxel sizes)."""
    out = set()
    bs = float(bs)
    for l, h in zip(np.asarray(lo, f64), np.asarray(hi, f64)):
        cand = [range(int(np.floor(l[a] / bs)) - 2, int(np.floor(h[a] / bs)) + 3) for a in range(3)]
        ok = [[b for b in cand[a] if b * bs <= h[a] and (b + 1) * bs > l[a]] for a in range(3)]
        for z in ok[2]:
            for y in ok[1]:
                for x in ok[0]:
                    out.add(int(T.pack_keys([[x, y, z]])[0]))
    return np.array(sorted(out), np.int64)
