"""Inputs of the opacity-field lattice tests (csrc/field_grid.cu): seeded Gaussians with negative coordinates, zero scales,
boxes ending exactly on block faces and centres outside every view, the views that see them, and the Gaussians at the
+-2^20 block-key limit.  Voxel size 0.25 and B = 4 make a block 1.0 wide, so every block quotient is exact."""
import numpy as np

import _tetra_scenes as TS

f32 = np.float32
S_EXACT, B_EXACT = 0.25, 4
W, H, FOCAL = 64, 48, 40.0


def view(R_rows, t):
    """A Cam whose view coordinates are R p + t (world_view_transform stores [R | t]^T, as the reference does)."""
    M = np.eye(4, dtype=f32)
    M[:3, :3] = np.asarray(R_rows, f32).T
    M[3, :3] = np.asarray(t, f32)
    return TS.Cam(M, FOCAL, FOCAL, W, H)


def views_around(depth=6.0):
    """Two views facing the origin from -z and +z, and one from +x."""
    return [view(np.eye(3), (0, 0, depth)), view([[-1, 0, 0], [0, 1, 0], [0, 0, -1]], (0, 0, depth)),
            view([[0, 0, -1], [0, 1, 0], [1, 0, 0]], (0, 0, depth))]


def gaussians(P, seed, extent=3.0):
    """(xyz, scales, raw rotations) float32: centres in [-extent, extent]^3, log-uniform scales, raw quaternions of norm 0.2..3;
    then four Gaussians with zero scales whose boxes end exactly on block faces (s = 0.25, B = 4) and two far outside every view."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-extent, extent, (P, 3)).astype(f32)
    scales = np.exp(rng.uniform(np.log(0.01), np.log(0.5), (P, 3))).astype(f32)
    q = rng.normal(size=(P, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(0.2, 3.0, (P, 1))).astype(f32)
    face = np.array([[2.75, 0.0, 0.0], [-0.25, -1.25, 0.5], [0.5, 0.75, -2.25], [-1.75, 1.0, 1.75]], f32)
    far = np.array([[50.0, 50.0, 0.0], [0.0, -60.0, 3.0]], f32)
    xyz = np.concatenate([xyz, face, far])
    scales = np.concatenate([scales, np.zeros((4, 3), f32), np.full((2, 3), 0.1, f32)])
    rot = np.concatenate([q, np.tile(np.array([[1, 0, 0, 0]], f32), (6, 1))])
    return xyz, scales, rot


def key_limit_case(x, axis=0):
    """One Gaussian with zero scales at coordinate x on `axis` and a view centred on it."""
    c = np.zeros((1, 3), f32)
    c[0, axis] = x
    t = -c[0].astype(np.float64)
    t[2] += 5.0
    return c, np.zeros((1, 3), f32), np.array([[1, 0, 0, 0]], f32), [view(np.eye(3), t)]


def table(views):
    import tetra_points_oracle as tpo
    return tpo.pack_views(views)
