"""CPU oracle of the TSDF fusion and marching-cubes extraction (DESIGN section 4.4) -- TEST INFRASTRUCTURE ONLY.

numpy float32, one IEEE operation per step in the order the specification writes it, so that csrc/tsdf.cu (which spells
every step with __fmul_rn / __fadd_rn / __fdiv_rn) agrees with it bit for bit.  Sparse over blocks: the volume keeps its
block keys sorted and one row of B^3 voxels per block, in key order.  The triangle table comes from the same generator
as the CUDA header (tools/gen_mc_table.py).
"""
import importlib.util
import os

import numpy as np

f32 = np.float32
KEY_BITS = 21
KEY_BIAS = 1 << 20            # block coordinates live in [-2^20, 2^20)
TOUCH_STRIDE = 4

_spec = importlib.util.spec_from_file_location(
    "gen_mc_table", os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools", "gen_mc_table.py"))
_gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_gen)
MC_TABLE = _gen.table()
EDGE_OWNER = np.array([_gen.EDGES[e][0] for e in range(12)], np.int64)
EDGE_FAR = np.array([_gen.EDGES[e][1] for e in range(12)], np.int64)
CORNER_OFF = np.array([_gen.corner_offset(c) for c in range(8)], np.int64)   # (dx, dy, dz)


class BlockRangeError(ValueError):
    pass


def pack_keys(b):
    """[n,3] int block coordinates (bx, by, bz) -> [n] int64 keys, z-major."""
    b = np.asarray(b, np.int64).reshape(-1, 3)
    if b.size and (b.min() < -KEY_BIAS or b.max() >= KEY_BIAS):
        raise BlockRangeError("block coordinate outside [-2^20, 2^20)")
    u = b + KEY_BIAS
    return (u[:, 2] << (2 * KEY_BITS)) | (u[:, 1] << KEY_BITS) | u[:, 0]


def unpack_keys(k):
    k = np.asarray(k, np.int64)
    m = (1 << KEY_BITS) - 1
    return np.stack([k & m, (k >> KEY_BITS) & m, k >> (2 * KEY_BITS)], axis=-1) - KEY_BIAS


def _rigid(extrinsic):
    E = np.asarray(extrinsic, f32)
    if E.shape not in ((3, 4), (4, 4)):
        raise ValueError("extrinsic must be [3,4] or [4,4]")
    return E[:3, :3], E[:3, 3]


class Volume:
    def __init__(self, voxel_size=0.002, block_resolution=16, trunc_voxel_multiplier=8.0):
        self.s = f32(voxel_size)
        self.B = int(block_resolution)
        self.tau = f32(f32(trunc_voxel_multiplier) * self.s)
        self.bs = f32(f32(self.B) * self.s)
        n3 = self.B ** 3
        self.keys = np.zeros(0, np.int64)
        self.tsdf = np.zeros((0, n3), f32)
        self.weight = np.zeros((0, n3), f32)
        self.color = np.zeros((0, 3, n3), f32)

    # ---- 1. touch ----------------------------------------------------------------------------------------------
    def touch(self, depth, fx, fy, cx, cy, extrinsic, depth_max=6.0):
        depth = np.asarray(depth, f32)
        H, W = depth.shape
        R, t = _rigid(extrinsic)
        fx, fy, cx, cy, dmax = f32(fx), f32(fy), f32(cx), f32(cy), f32(depth_max)
        v, u = np.mgrid[0:H:TOUCH_STRIDE, 0:W:TOUCH_STRIDE]
        d = depth[v, u]
        m = (d > 0) & (d < dmax)
        u, v, d = u[m].astype(f32), v[m].astype(f32), d[m]
        pc = [((u - cx) * d) / fx, ((v - cy) * d) / fy, d]
        q = [pc[i] - t[i] for i in range(3)]
        pw = [(R[0, i] * q[0] + R[1, i] * q[1]) + R[2, i] * q[2] for i in range(3)]
        lo, hi = [], []
        for i in range(3):
            a = np.floor((pw[i] - self.tau) / self.bs)
            b = np.floor((pw[i] + self.tau) / self.bs)
            if a.size and not (np.all(a >= -KEY_BIAS) and np.all(b < KEY_BIAS)):
                raise BlockRangeError("touched block outside [-2^20, 2^20)")
            lo.append(a.astype(np.int64))
            hi.append(b.astype(np.int64))
        span = max([int((hi[i] - lo[i]).max()) + 1 if lo[i].size else 0 for i in range(3)] + [0])
        out = []
        for dz in range(span):
            for dy in range(span):
                for dx in range(span):
                    b = np.stack([lo[0] + dx, lo[1] + dy, lo[2] + dz], 1)
                    ok = (b[:, 0] <= hi[0]) & (b[:, 1] <= hi[1]) & (b[:, 2] <= hi[2])
                    out.append(pack_keys(b[ok]))
        return np.unique(np.concatenate(out)) if out else np.zeros(0, np.int64)

    # ---- 2. activate ---------------------------------------------------------------------------------------------
    def activate(self, keys):
        new = np.setdiff1d(keys, self.keys)
        if new.size:
            pos = np.searchsorted(self.keys, new)
            self.keys = np.insert(self.keys, pos, new)
            self.tsdf = np.insert(self.tsdf, pos, 0, axis=0)
            self.weight = np.insert(self.weight, pos, 0, axis=0)
            self.color = np.insert(self.color, pos, 0, axis=0)
        return np.searchsorted(self.keys, keys)

    # ---- 3. integrate --------------------------------------------------------------------------------------------
    def integrate(self, depth, color, fx, fy, cx, cy, extrinsic, depth_max=6.0):
        """Touch, activate and integrate one view; returns the view's block keys."""
        depth = np.asarray(depth, f32)
        color = np.asarray(color, f32)
        keys = self.touch(depth, fx, fy, cx, cy, extrinsic, depth_max)
        rows = self.activate(keys)
        if not keys.size:
            return keys
        H, W = depth.shape
        R, t = _rigid(extrinsic)
        fx, fy, cx, cy, dmax, tau, s, B = f32(fx), f32(fy), f32(cx), f32(cy), f32(depth_max), self.tau, self.s, self.B
        lin = np.arange(B ** 3)
        local = np.stack([lin % B, (lin // B) % B, lin // (B * B)], 1)
        vox = unpack_keys(keys)[:, None, :] * B + local[None]            # [n, B^3, 3] int64
        p = [vox[..., i].astype(f32) * s for i in range(3)]
        pc = [((R[r, 0] * p[0] + R[r, 1] * p[1]) + R[r, 2] * p[2]) + t[r] for r in range(3)]
        z = pc[2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = (fx * pc[0]) / z + cx
            v = (fy * pc[1]) / z + cy
        inb = (z > 0) & (u >= 0) & (u <= f32(W - 1)) & (v >= 0) & (v <= f32(H - 1))
        ui = np.where(inb, u, 0).astype(np.int32)
        vi = np.where(inb, v, 0).astype(np.int32)
        d = depth[vi, ui]
        sdf = d - z
        upd = inb & (d > 0) & (d <= dmax) & (sdf >= -tau)
        r_, l_ = np.nonzero(upd)
        g = rows[r_]
        sd = np.minimum(sdf[r_, l_], tau) / tau
        w = self.weight[g, l_]
        w1 = w + f32(1)
        self.tsdf[g, l_] = (w * self.tsdf[g, l_] + sd) / w1
        for c in range(3):
            self.color[g, c, l_] = (w * self.color[g, c, l_] + color[c, vi[r_, l_], ui[r_, l_]]) / w1
        self.weight[g, l_] = w1
        self.last_updates = int(r_.size)
        return keys

    # ---- 4. extract ----------------------------------------------------------------------------------------------
    def _padded(self, row_of, bkey):
        """(B+1)^3 tsdf / weight / colour / existence around the block with coordinates bkey (its +1 neighbours)."""
        B = self.B
        T = np.zeros((B + 1,) * 3, f32)
        Wt = np.zeros((B + 1,) * 3, f32)
        C = np.zeros((3,) + (B + 1,) * 3, f32)
        X = np.zeros((B + 1,) * 3, bool)
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    k = int(pack_keys([bkey + np.array([dx, dy, dz])])[0]) if np.all(bkey + [dx, dy, dz] < KEY_BIAS) else None
                    r = row_of.get(k)
                    if r is None:
                        continue
                    zs = slice(0, B) if dz == 0 else slice(B, B + 1)
                    ys = slice(0, B) if dy == 0 else slice(B, B + 1)
                    xs = slice(0, B) if dx == 0 else slice(B, B + 1)
                    src = (slice(0, B) if dz == 0 else slice(0, 1), slice(0, B) if dy == 0 else slice(0, 1),
                           slice(0, B) if dx == 0 else slice(0, 1))
                    T[zs, ys, xs] = self.tsdf[r].reshape(B, B, B)[src]
                    Wt[zs, ys, xs] = self.weight[r].reshape(B, B, B)[src]
                    C[:, zs, ys, xs] = self.color[r].reshape(3, B, B, B)[(slice(None),) + src]
                    X[zs, ys, xs] = True
        return T, Wt, C, X

    def extract_triangle_mesh(self, weight_threshold=3.0):
        B, s, th = self.B, self.s, f32(weight_threshold)
        n = self.keys.size
        row_of = {int(k): i for i, k in enumerate(self.keys)}
        bco = unpack_keys(self.keys)
        marks = np.zeros((n, B ** 3), np.uint8)
        cubes = []                                                       # per block: (lin, code) of meshed cubes
        pads = []
        ii = np.arange(B)
        K, J, I = np.meshgrid(ii, ii, ii, indexing="ij")                 # [k, j, i] = voxel lin i + B j + B^2 k
        for p in range(n):
            T, Wt, C, X = self._padded(row_of, bco[p])
            pads.append((T, C))
            ok = np.ones((B, B, B), bool)
            code = np.zeros((B, B, B), np.int64)
            for c in range(8):
                dx, dy, dz = CORNER_OFF[c]
                sl = (slice(dz, dz + B), slice(dy, dy + B), slice(dx, dx + B))
                ok &= X[sl] & (Wt[sl] > th)
                code |= (T[sl] < 0).astype(np.int64) << c
            lin = np.nonzero(ok.reshape(-1))[0]
            code = code.reshape(-1)[lin]
            cubes.append((lin, code))
            if not lin.size:
                continue
            ci, cj, ck = I.reshape(-1)[lin], J.reshape(-1)[lin], K.reshape(-1)[lin]
            for e in range(12):
                a, b = EDGE_OWNER[e], EDGE_FAR[e]
                cross = ((code >> a) ^ (code >> b)) & 1 == 1
                if not cross.any():
                    continue
                ox, oy, oz = ci[cross] + CORNER_OFF[a][0], cj[cross] + CORNER_OFF[a][1], ck[cross] + CORNER_OFF[a][2]
                nb = np.stack([ox // B, oy // B, oz // B], 1)
                tgt = np.array([row_of[int(k)] for k in pack_keys(bco[p] + nb)], np.int64)
                np.bitwise_or.at(marks, (tgt, (ox % B) + B * (oy % B) + B * B * (oz % B)), np.uint8(1 << (e // 4)))
        pop = ((marks & 1) + ((marks >> 1) & 1) + ((marks >> 2) & 1)).astype(np.int64).reshape(-1)
        base = (np.cumsum(pop) - pop).reshape(n, B ** 3)
        V = int(pop.sum())
        verts = np.zeros((V, 3), f32)
        cols = np.zeros((V, 3), f32)
        lin_all = np.arange(B ** 3)
        loc = np.stack([lin_all % B, (lin_all // B) % B, lin_all // (B * B)], 1)
        for p in range(n):
            T, C = pads[p]
            for a in range(3):
                sel = np.nonzero((marks[p] >> a) & 1)[0]
                if not sel.size:
                    continue
                vid = base[p, sel] + np.array([bin(int(m) & ((1 << a) - 1)).count("1") for m in marks[p, sel]], np.int64)
                o = loc[sel]
                e = o.copy()
                e[:, a] += 1
                to = T[o[:, 2], o[:, 1], o[:, 0]]
                te = T[e[:, 2], e[:, 1], e[:, 0]]
                r = (f32(0) - to) / (te - to)
                g = bco[p] * B + o                                        # global voxel coordinates of the owners
                for ax in range(3):
                    gx = g[:, ax].astype(f32)
                    verts[vid, ax] = (gx + r) * s if ax == a else gx * s
                one_r = f32(1) - r
                for c in range(3):
                    cols[vid, c] = one_r * C[c, o[:, 2], o[:, 1], o[:, 0]] + r * C[c, e[:, 2], e[:, 1], e[:, 0]]
        faces = []
        for p in range(n):
            lin, code = cubes[p]
            for l_, cd in zip(lin.tolist(), code.tolist()):
                ci, cj, ck = l_ % B, (l_ // B) % B, l_ // (B * B)
                for tri in MC_TABLE[cd]:
                    f = []
                    for e in tri:
                        a = e // 4
                        dx, dy, dz = CORNER_OFF[EDGE_OWNER[e]]
                        ox, oy, oz = ci + dx, cj + dy, ck + dz
                        q = p if (ox < B and oy < B and oz < B) else row_of[int(pack_keys([bco[p] + [ox // B, oy // B, oz // B]])[0])]
                        ol = (ox % B) + B * (oy % B) + B * B * (oz % B)
                        f.append(int(base[q, ol]) + bin(int(marks[q, ol]) & ((1 << a) - 1)).count("1"))
                    faces.append(f)
        faces = np.array(faces, np.int64).reshape(-1, 3)
        return {"vertices": verts, "faces": faces, "colors": cols}

    def state(self):
        return {"keys": self.keys.copy(), "tsdf": self.tsdf.copy(), "weight": self.weight.copy(), "color": self.color.copy()}
