"""Level-set extraction helpers around GaussianRasterizer.integrate -- the callers of the integrate path in the
reference's extract_mesh.py, restated with view sharding over the GPUs of one box.

* evaluate_alpha    == evaluage_alpha (extract_mesh.py:17-34): alpha = 1 - min over views of the integrated opacity,
                       optionally the colour of the arg-min view.  `min` is associative, so with torch.distributed
                       initialised every rank processes views[rank::world] and the partial minima are merged with one
                       all_reduce(MIN) (colour: the lowest view index attaining the minimum wins, like the reference's
                       strict `<` update in view order).
* opacity_field     -- evaluate_alpha's field with gradients to the points and the Gaussians (DESIGN §4.12), view-sharded
                       like it, in memory that does not grow with the number of views; optionally its colour, with
                       gradients to the Gaussians and their SHs (DESIGN §4.13).
* binary_search     == the 8-step bisection of extract_mesh.py:88-102 on the edge endpoints returned by
                       gof_tetmesh.marching_tetrahedra.
* make_integrate_fn == gaussian_renderer.integrate (gaussian_renderer/__init__.py:118-218) for plain tensors.
* CachedIntegrator  -- the same, with the Gaussian side of every view prepared once and reused by all passes (SURVEY 8(f) rank 3).
* field_gradient    -- evaluate_alpha over a CachedIntegrator together with the field's point gradient, formed in the query's
                       own pass (DESIGN §4.14); extract_level_set(return_normals=True) turns it into vertex normals.
* marching_tetrahedra_sharded / merge_tet_shards -- utils/tetmesh.py's chunk loop (:55-95) spread over ranks (SURVEY 8(e)).
* extract_level_set -- marching_tetrahedra_with_binary_search (extract_mesh.py:37-120) up to the mesh arrays.
* get_tetra_points  == GaussianModel.get_tetra_points (scene/gaussian_model.py:433-463), get_frustum_mask == its module-level
                       get_frustum_mask (:31-72): one CUDA pass (csrc/tetra_points.cu, DESIGN §4.8) in memory linear in the
                       points, where the reference builds ~40 bytes per (view, point).
* extract_level_set_grid -- the same level set without tetrahedra: the field sampled on a sparse voxel-block lattice around
                       the Gaussians, marching cubes, the same bisection, colours and normals (csrc/field_grid.cu, DESIGN §4.15).
"""
import contextlib
import ctypes
import functools
import time

import torch
import torch.distributed as dist


_NO_VIEW = 2 ** 30   # argmin of a point no view lowered below 1


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def _views_of_rank(views, rank, world):
    """The (index, view) pairs of `views` that `rank` of `world` processes in the view-sharded passes: views[rank::world]."""
    views = list(views)
    for vi in range(rank, len(views), world):
        yield vi, views[vi]


def _owns_view(vi, rank, world):
    """Whether view index vi (an int or a tensor of them) is one that _views_of_rank gives `rank`."""
    return vi % world == rank


def _merge_minimum(alpha_min, argmin, rows, group):
    """The ranks' view-sharded running minima, merged into the minimum over all views.  alpha_min [N] becomes the global minimum
    (all_reduce MIN).  With argmin [N] (int32, _NO_VIEW where no view lowered the point below 1), a point's winner is the lowest
    view index that attains that minimum below 1, the view a serial strict `<` update in view order keeps; a second all_reduce
    (MIN) agrees on it.  With rows [N,k] as well, a third all_reduce (SUM) gives every rank the winner's rows, and zeros where no
    view won.  Returns (alpha_min, argmin, rows, won [N] bool), with None for what was not given (won needs argmin)."""
    local = alpha_min.clone() if argmin is not None else None
    dist.all_reduce(alpha_min, op=dist.ReduceOp.MIN, group=group)
    if argmin is None:
        return alpha_min, None, None, None
    cand = torch.where((local == alpha_min) & (local < 1.0), argmin, torch.full_like(argmin, _NO_VIEW))
    argmin = cand.clone()
    dist.all_reduce(argmin, op=dist.ReduceOp.MIN, group=group)
    won = argmin < _NO_VIEW
    if rows is not None:
        rows = torch.where(((cand == argmin) & won).reshape(-1, 1), rows, torch.zeros_like(rows))
        dist.all_reduce(rows, op=dist.ReduceOp.SUM, group=group)
    return alpha_min, argmin, rows, won


@torch.no_grad()
def evaluate_alpha(points, views, integrate_fn, return_color=False, group=None):
    """integrate_fn(points, view) -> (alpha_integrated [N], color_integrated [N,3])."""
    rank, world = _world(group)
    n, dev = points.shape[0], points.device
    final_alpha = torch.ones(n, dtype=torch.float32, device=dev)
    final_color = torch.ones(n, 3, dtype=torch.float32, device=dev) if return_color else None
    best_view = torch.full((n,), _NO_VIEW, dtype=torch.int32, device=dev) if return_color else None
    for vi, view in _views_of_rank(views, rank, world):
        alpha_integrated, color_integrated = integrate_fn(points, view)
        if return_color:
            better = alpha_integrated < final_alpha
            final_color = torch.where(better.reshape(-1, 1), color_integrated, final_color)
            best_view = torch.where(better, torch.full_like(best_view, vi), best_view)
        final_alpha = torch.min(final_alpha, alpha_integrated)
    if world > 1:
        final_alpha, _argmin, contrib, won = _merge_minimum(final_alpha, best_view, final_color, group)
        if return_color:
            final_color = torch.where(won.reshape(-1, 1), contrib, torch.ones_like(contrib))
    alpha = 1 - final_alpha
    return (alpha, final_color) if return_color else alpha


@torch.no_grad()
def binary_search(end_points, end_sdf, eval_alpha, n_steps=8):
    """extract_mesh.py:73-102.  end_points (E,2,3), end_sdf (E,2,1) from marching_tetrahedra; eval_alpha(points)->alpha.
    Returns the refined vertex positions (E,3)."""
    left_points, right_points = end_points[:, 0, :].clone(), end_points[:, 1, :].clone()
    left_sdf, right_sdf = end_sdf[:, 0, :].clone(), end_sdf[:, 1, :].clone()
    points = (left_points + right_points) / 2.
    for _ in range(n_steps):
        mid_points = (left_points + right_points) / 2
        mid_sdf = (eval_alpha(mid_points) - 0.5).reshape(-1, 1)
        ind_low = ((mid_sdf < 0) & (left_sdf < 0)) | ((mid_sdf > 0) & (left_sdf > 0))
        left_sdf[ind_low] = mid_sdf[ind_low]
        right_sdf[~ind_low] = mid_sdf[~ind_low]
        left_points[ind_low.flatten()] = mid_points[ind_low.flatten()]
        right_points[~ind_low.flatten()] = mid_points[~ind_low.flatten()]
        points = (left_points + right_points) / 2
    return points


def make_integrate_fn(means3D, opacities, scales, rotations, shs, sh_degree, settings_for_view):
    """settings_for_view(view) -> GaussianRasterizationSettings.  Returns integrate_fn for evaluate_alpha."""
    from diff_gaussian_rasterization import GaussianRasterizer

    def fn(points, view):
        rs = settings_for_view(view)
        _, alpha_integrated, color_integrated, _ = GaussianRasterizer(rs).integrate(
            points3D=points, means3D=means3D, means2D=torch.zeros_like(means3D), opacities=opacities, shs=shs, scales=scales,
            rotations=rotations)
        return alpha_integrated, color_integrated
    return fn


def _field_inputs(scales, rotations, shs):
    """(colors_precomp, scales, rotations, cov3D_precomp, view2gaussian_precomp, shs) as GaussianRasterizer.integrate passes them
    for shs, scales and rotations: the optional inputs make_integrate_fn's queries leave out, in the reference's empty encoding."""
    import diff_gaussian_rasterization as dgr
    shs, colors, scales, rotations, cov3D, v2g = dgr._normalise_optionals(shs, None, scales, rotations, None, None)
    return colors, scales, rotations, cov3D, v2g, shs


def _field_args(rs, points, means3D, opacities, scales, rotations, shs):
    """The argument tuple of the _C query entry points for GaussianRasterizer(rs).integrate(points3D=points, means3D=means3D,
    opacities=opacities, shs=shs, scales=scales, rotations=rotations): what make_integrate_fn's queries receive."""
    import diff_gaussian_rasterization as dgr
    colors, scales, rotations, cov3D, v2g, shs = _field_inputs(scales, rotations, shs)
    return dgr._integrate_args(rs, points, means3D, colors, opacities, scales, rotations, cov3D, v2g, shs)


class _OpacityField(torch.autograd.Function):
    """alpha = 1 - min over views of alpha_integrated (DESIGN.md 4.12), differentiable with respect to the points and the
    Gaussians; with return_color also the winning view's color_integrated (DESIGN.md 4.13).  The forward keeps a running minimum
    and the winning view per point (8 bytes a point, 20 with the colour, nothing per view); the backward rebuilds one view's query
    state at a time, on the points that view won."""

    @staticmethod
    def forward(ctx, points, means3D, opacities, scales, rotations, shs, views, settings_for_view, group, return_color):
        import diff_gaussian_rasterization as dgr
        from diff_gaussian_rasterization import _C
        rank, world = _world(group)
        n, dev = points.shape[0], points.device
        alpha_min = torch.ones(n, dtype=torch.float32, device=dev)
        argmin = torch.full((n,), _NO_VIEW, dtype=torch.int32, device=dev)
        color = torch.ones(n, 3, dtype=torch.float32, device=dev) if return_color else None
        views = list(views)
        for vi, view in _views_of_rank(views, rank, world):
            rs = settings_for_view(view)
            args = _field_args(rs, points, means3D, opacities, scales, rotations, shs) + (vi, alpha_min, argmin)
            dgr._call_native(_C.integrate_gaussians_to_points_min, args, rs.debug, "snapshot_fw.dump", "forward",
                             **({"color_min": color} if return_color else {}))
        if world > 1:
            alpha_min, argmin, contrib, won = _merge_minimum(alpha_min, argmin, color, group)
            if return_color:
                color = torch.where(won.reshape(-1, 1), contrib, torch.ones_like(contrib))
        ctx.save_for_backward(points, means3D, opacities, scales, rotations, shs, argmin)
        ctx.views, ctx.settings_for_view, ctx.group = views, settings_for_view, group
        if not return_color:
            return 1 - alpha_min
        ctx.set_materialize_grads(False)
        return 1 - alpha_min, color

    @staticmethod
    def backward(ctx, grad_alpha, grad_color=None):
        import diff_gaussian_rasterization as dgr
        from diff_gaussian_rasterization import _C
        points, means3D, opacities, scales, rotations, shs, argmin = ctx.saved_tensors
        rank, world = _world(ctx.group)
        need = ctx.needs_input_grad
        gaussians = any(need[1:6])
        n, P, dev = points.shape[0], means3D.shape[0], points.device
        if grad_alpha is None:
            grad_alpha = torch.zeros(n, dtype=torch.float32, device=dev)
        with_color = grad_color is not None
        # d alpha / d alpha_min = -1, at each point's winning view only; the colour's gradient goes to the same view
        dA = -grad_alpha.to(torch.float32).contiguous()
        dC = grad_color.to(torch.float32).contiguous() if with_color else None
        if world > 1:
            # a rank runs the backward of the views it owns only, so it needs every rank's dL/dalpha (and dL/dcolour): the
            # gradients are those of the sum of the ranks' losses
            if with_color:
                dAC = torch.cat([dA.view(-1, 1), dC.view(-1, 3)], 1)
                dist.all_reduce(dAC, op=dist.ReduceOp.SUM, group=ctx.group)
                dA, dC = dAC[:, 0].contiguous(), dAC[:, 1:].contiguous()
            else:
                dA = dA.clone()
                dist.all_reduce(dA, op=dist.ReduceOp.SUM, group=ctx.group)
        # one flat buffer: a single all-reduce carries every gradient across ranks
        n_sh = shs.numel() if with_color and need[5] else 0
        sizes = (3 * n, 3 * P, P, 3 * P, 4 * P, n_sh)
        flat = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        g_pts, g_means, g_op, g_scales, g_rot, g_sh = torch.split(flat, sizes)
        g_pts, g_means, g_scales, g_rot = g_pts.view(n, 3), g_means.view(P, 3), g_scales.view(P, 3), g_rot.view(P, 4)
        if n and P:
            colors, scales_, rotations_, cov3D, v2g, shs_ = _field_inputs(scales, rotations, shs)
            mine = torch.nonzero((argmin != _NO_VIEW) & _owns_view(argmin, rank, world)).flatten()
            order = mine[torch.argsort(argmin[mine], stable=True)]
            won, counts = torch.unique_consecutive(argmin[order], return_counts=True)
            start = 0
            for vi, c in zip(won.tolist(), counts.tolist()):
                sel = order[start:start + c]
                start += c
                rs = ctx.settings_for_view(ctx.views[vi])
                p = points[sel]
                args = dgr._integrate_args(rs, p, means3D, colors, opacities, scales_, rotations_, cov3D, v2g, shs_)
                R, _color, _a, _c, radii, geom, binning, img, pts, pbin = dgr._call_native(
                    _C.integrate_gaussians_to_points_state, args, rs.debug, "snapshot_fw.dump", "forward")
                del _color, _a, _c
                bargs = dgr._integrate_backward_args(rs, p, means3D, radii, colors, scales_, rotations_, cov3D, v2g, shs_, dA[sel], R,
                                                     geom, binning, img, pts, pbin)
                del geom, binning, img, pts, pbin
                dp, dop, dm, dsc, drot, _dcov, _dv2g, _dcol, dsh = dgr._call_native(
                    _C.integrate_gaussians_to_points_backward, bargs, rs.debug, "snapshot_bw.dump", "backward",
                    points_grad=need[0], dL_dcolor=dC[sel] if with_color else None)
                del bargs   # the state goes back to the scratch pool before the next view
                if n_sh:
                    g_sh += dsh.view(-1)
                if dp is not None:
                    g_pts[sel] = dp
                if gaussians:
                    g_means += dm
                    g_op += dop.view(-1)
                    g_scales += dsc
                    g_rot += drot
        if world > 1:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=ctx.group)
        pick = lambda g, i, like: g.view_as(like) if need[i] else None   # noqa: E731
        return (pick(g_pts, 0, points), pick(g_means, 1, means3D), pick(g_op, 2, opacities), pick(g_scales, 3, scales),
                pick(g_rot, 4, rotations), g_sh.view_as(shs) if n_sh else None, None, None, None, None)


def opacity_field(points, means3D, opacities, scales, rotations, shs, sh_degree, views, settings_for_view, group=None,
                  return_color=False):
    """The multi-view opacity field alpha [N] = 1 - min over views of alpha_integrated: the tensor
    evaluate_alpha(points, views, make_integrate_fn(means3D, opacities, scales, rotations, shs, sh_degree, settings_for_view),
    group=group) returns, bit for bit, but differentiable with respect to points, means3D, opacities, scales and rotations
    (DESIGN.md 4.12).  As in make_integrate_fn, the SH degree the query uses is settings_for_view(view).sh_degree.

    The gradient of a point goes through the view attaining its minimum (the lowest view index on a tie); a point that no view
    lowered below 1 gets zeros.  Memory does not grow with the number of views: the forward keeps 8 bytes a point, and the
    backward rebuilds the query state of one view at a time on the points that view won.

    With torch.distributed initialised, each rank queries views[rank::world] and the ranks merge as evaluate_alpha does, so
    every rank holds the whole field.  The backward is a collective: every rank of `group` must call backward() through the
    field.  The gradients are those of the SUM of the ranks' losses: the backward all-reduces dL/dalpha before it runs each
    rank's views, and all-reduces the gradients after, so every rank's .grad is the single-GPU gradient of that sum, up to
    summation order.  A rank without a loss of its own backpropagates zeros (e.g. (alpha * 0).sum()); a loss computed
    identically on every rank counts once per rank (divide it by the world size, or compute it on one rank only).

    return_color=True returns (alpha, colour [N,3]): the colour evaluate_alpha(..., return_color=True) returns, bit for bit --
    the winning view's color_integrated, (1, 1, 1) where no view lowered the minimum (DESIGN.md 4.13).  Its gradient reaches
    means3D, opacities, scales, rotations and shs through the winning view only; the points get nothing from it (the colour
    is piecewise constant in the point).  With a group, dL/dcolour is all-reduced together with dL/dalpha."""
    return _OpacityField.apply(points, means3D, opacities, scales, rotations, shs, views, settings_for_view, group, return_color)


class CachedIntegrator:
    """integrate_fn for evaluate_alpha / binary_search that prepares the Gaussian side of a view ONCE
    (`_C.integrate_prepare`: preprocess, depth sort, instance emission, tile sort) and afterwards runs only the point side
    (`_C.integrate_points_cached`).  The reference repeats the whole Gaussian side in each of its 9-10 passes over the same
    views (extract_mesh.py:56,92,107).  Results are bit-identical to GaussianRasterizer.integrate.  Memory: 64 B/Gaussian +
    4 B/tile instance per cached view (3 M Gaussians: ~0.23 GB/view; 64 views = 14.4 GB on one 80 GB GPU, or 8 per GPU on 8)."""

    def __init__(self, means3D, opacities, scales, rotations, shs, sh_degree, settings_for_view):
        self.gs = (means3D, opacities, scales, rotations, shs)
        self.sh_degree, self.settings_for_view = sh_degree, settings_for_view
        self._cache = {}     # id(view) -> (view, settings, IntegrateCache)

    def prepare(self, view):
        from diff_gaussian_rasterization import _C
        key = id(view)
        hit = self._cache.get(key)
        if hit is not None:
            return hit
        rs = self.settings_for_view(view)
        means3D, opacities, scales, rotations, shs = self.gs
        e = torch.Tensor([])
        c = _C.integrate_prepare(rs.bg, means3D, e, opacities, scales, rotations, rs.scale_modifier, e, e, rs.viewmatrix, rs.projmatrix,
                                 rs.tanfovx, rs.tanfovy, rs.kernel_size, rs.subpixel_offset, rs.image_height, rs.image_width, shs,
                                 self.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        self._cache[key] = (view, rs, c)
        return self._cache[key]

    def __call__(self, points, view):
        from diff_gaussian_rasterization import _C
        _view, rs, c = self.prepare(view)
        _color, alpha_integrated, color_integrated = _C.integrate_points_cached(c, rs.bg, points, rs.viewmatrix, rs.tanfovx, rs.tanfovy,
                                                                                rs.debug)
        return alpha_integrated, color_integrated

    def min_update(self, points, view, vi, alpha_min, argmin, color_min=None, grad_min=None):
        """Folds view `view` (index vi) into the running minimum over views in place (_C.integrate_points_cached_min)."""
        from diff_gaussian_rasterization import _C
        _view, rs, c = self.prepare(view)
        _C.integrate_points_cached_min(c, rs.bg, points, rs.viewmatrix, rs.tanfovx, rs.tanfovy, vi, alpha_min, argmin,
                                       color_min=color_min, grad_min=grad_min, debug=rs.debug)

    @property
    def cached_bytes(self):
        return sum(c.nbytes for _v, _rs, c in self._cache.values())

    def clear(self):
        self._cache.clear()


@torch.no_grad()
def field_gradient(points, views, integrate_fn, return_color=False, group=None):
    """evaluate_alpha's field and its gradient with respect to the points, in one pass over the cached views (DESIGN.md 4.14).
    integrate_fn must be a CachedIntegrator.  Returns (alpha [N], grad [N,3]) or, with return_color, (alpha, grad, colour [N,3]):
    alpha and colour are evaluate_alpha(points, views, integrate_fn, return_color=...)'s, bit for bit; grad is d alpha / d point
    through the winning view (the lowest view index on a tie), the points.grad that opacity_field(points, ...).sum().backward()
    leaves, bit for bit.  A point that no view lowers below 1 gets zeros.  With torch.distributed initialised each rank folds
    views[rank::world], and the ranks merge as evaluate_alpha does; the winner's rank contributes the gradient and colour rows."""
    if not isinstance(integrate_fn, CachedIntegrator):
        raise TypeError(f"field_gradient: integrate_fn must be a CachedIntegrator, got {type(integrate_fn).__name__}")
    rank, world = _world(group)
    n, dev = points.shape[0], points.device
    alpha_min = torch.ones(n, dtype=torch.float32, device=dev)
    argmin = torch.full((n,), _NO_VIEW, dtype=torch.int32, device=dev)
    grad_min = torch.zeros(n, 3, dtype=torch.float32, device=dev)
    color = torch.ones(n, 3, dtype=torch.float32, device=dev) if return_color else None
    for vi, view in _views_of_rank(views, rank, world):
        integrate_fn.min_update(points, view, vi, alpha_min, argmin, color_min=color, grad_min=grad_min)
    if world > 1:
        # the winner's gradient and colour rows in one [N,6] block, summed in a single all-reduce
        rows = torch.cat([grad_min, color], 1) if return_color else grad_min
        alpha_min, argmin, rows, won = _merge_minimum(alpha_min, argmin, rows, group)
        grad_min = rows[:, :3]
        if return_color:
            color = torch.where(won.reshape(-1, 1), rows[:, 3:], torch.ones_like(color))
    alpha, grad = 1 - alpha_min, -grad_min
    return (alpha, grad, color.contiguous()) if return_color else (alpha, grad.contiguous())


# ---- marching tetrahedra sharded by tet chunk (SURVEY 8(e); utils/tetmesh.py:55-95 is the single-GPU chunk loop) ---------
def _edge_keys(interp_v):
    return (interp_v[:, 0].to(torch.int64) << 32) | interp_v[:, 1].to(torch.int64)


def merge_tet_shards(vertices, sdf, scales, shard_keys, shard_faces):
    """Merges per-shard marching-tetrahedra results the way utils/tetmesh.py:84-95 merges its chunks: the union of the shards'
    crossing edges in lexicographic (first vertex, second vertex) order defines the mesh-vertex numbering, every shard's faces
    are renumbered into it and concatenated in shard order.  shard_keys[i]: int64 (lo << 32 | hi) of shard i's edges in ITS
    numbering; shard_faces[i]: (F_i, 3) int64 into that numbering.  Returns what marching_tetrahedra returns for one batch
    element: ((edge_pos (E,2,3), edge_sdf (E,2,1)), edge_scales (E,2,1), faces (F,3), interp_v (E,2))."""
    allk = torch.cat(shard_keys) if shard_keys else torch.zeros(0, dtype=torch.int64, device=vertices.device)
    union = torch.unique(allk)     # sorted: lexicographic in (lo, hi) because lo is the high word
    faces = []
    for k, f in zip(shard_keys, shard_faces):
        if f.numel():
            faces.append(torch.searchsorted(union, k)[f])
    faces = torch.cat(faces) if faces else torch.zeros((0, 3), dtype=torch.int64, device=vertices.device)
    interp_v = torch.stack([union >> 32, union & 0xFFFFFFFF], dim=1)
    v = vertices.reshape(-1, 3)
    edge_pos = v[interp_v.reshape(-1)].reshape(-1, 2, 3)
    edge_sdf = sdf.reshape(-1)[interp_v.reshape(-1)].reshape(-1, 2, 1)
    edge_scales = scales.reshape(-1)[interp_v.reshape(-1)].reshape(-1, 2, 1)
    return (edge_pos, edge_sdf), edge_scales, faces, interp_v


def shard_tet_range(num_tets, rows, rank, world):
    """Tets [begin, end) of `rank`: whole chunks of `rows` tets (the rows per chunk of the UNSHARDED call), as evenly as
    possible, so that shard boundaries are chunk boundaries and the merged faces come out in the unsharded order."""
    chunks = (num_tets + rows - 1) // rows
    c0, c1 = chunks * rank // world, chunks * (rank + 1) // world
    return min(c0 * rows, num_tets), min(c1 * rows, num_tets)


@torch.no_grad()
def marching_tetrahedra_sharded(vertices, tets, sdf, scales, group=None, chunk_tets=None, extract_fn=None):
    """`gof_tetmesh.marching_tetrahedra` for ONE batch element with the tets sharded by chunk over the ranks of `group`:
    each rank extracts its chunks, ONE all-gather exchanges the crossing-edge keys and the faces, merge_tet_shards merges them,
    and every rank ends with the complete mesh -- bit-identical to the unsharded call (faces are ordered per chunk, so shards
    are whole chunks of the unsharded split; with fewer chunks than ranks some ranks idle).  vertices (N,3), tets (T,4), sdf (N,),
    scales (N,1).  World size 1: the plain call.  `extract_fn(vertices, tets, sdf, scales, rows=...)` defaults to the CUDA
    implementation (tests pass the oracle)."""
    import gof_tetmesh
    if extract_fn is None:
        extract_fn = lambda v, t, s, sc, rows: gof_tetmesh._unbatched_marching_tetrahedra(v, t, s, sc, rows=rows)   # noqa: E731
    rank, world = _world(group)
    T = int(tets.shape[0])
    rows = gof_tetmesh.chunk_rows(T, int(chunk_tets or gof_tetmesh.CHUNK_TETS))
    if world == 1:
        return extract_fn(vertices, tets, sdf, scales, rows)
    b, e = shard_tet_range(T, rows, rank, world)
    dev = vertices.device
    if e > b:
        (_p, _s), _sc, faces, interp_v = extract_fn(vertices, tets[b:e], sdf, scales, rows)
    else:
        faces, interp_v = torch.zeros((0, 3), dtype=torch.int64, device=dev), torch.zeros((0, 2), dtype=torch.int64, device=dev)
    keys = _edge_keys(interp_v)
    sizes = torch.tensor([keys.numel(), faces.shape[0]], dtype=torch.int64, device=dev)
    all_sizes = [torch.zeros_like(sizes) for _ in range(world)]
    dist.all_gather(all_sizes, sizes, group=group)
    nk, nf = max(int(s[0]) for s in all_sizes), max(int(s[1]) for s in all_sizes)
    # one padded all-gather carries both the keys and the faces: a shard's faces index its own keys, which travel with them
    payload = torch.full((nk + 3 * nf,), -1, dtype=torch.int64, device=dev)
    payload[:keys.numel()] = keys
    payload[nk:nk + faces.numel()] = faces.reshape(-1)
    gathered = [torch.empty_like(payload) for _ in range(world)]
    dist.all_gather(gathered, payload, group=group)
    shard_keys = [g[:int(s[0])] for g, s in zip(gathered, all_sizes)]
    shard_faces = [g[nk:nk + 3 * int(s[1])].reshape(-1, 3) for g, s in zip(gathered, all_sizes)]
    return merge_tet_shards(vertices, sdf, scales, shard_keys, shard_faces)


def _stopwatch(timings, cuda):
    """stage(name): a context that adds its seconds to timings[name], after a device synchronise when `cuda`; nothing without
    `timings`."""
    @contextlib.contextmanager
    def stage(name):
        t0 = time.perf_counter()
        yield
        if timings is not None:
            if cuda:
                torch.cuda.synchronize()
            timings[name] = timings.get(name, 0.0) + (time.perf_counter() - t0)
    return stage


def _refine(end_points, end_sdf, views, integrate_fn, n_steps, group, return_color, return_normals, stage):
    """The vertices of both extractions: `n_steps` bisection steps of every edge (end_points (E,2,3), end_sdf (E,2,1)) onto the
    0.5 level set, then, with return_normals, the unit normals and the colours from one field_gradient pass, or with
    return_color alone evaluate_alpha's colours.  Returns (vertices (E,3), colours (E,3) or None, normals (E,3) or None)."""
    with stage("binary_search_s"):
        verts = binary_search(end_points, end_sdf, lambda p: evaluate_alpha(p, views, integrate_fn, group=group), n_steps=n_steps)
    colors = normals = None
    if return_normals:
        with stage("field_gradient_s"):
            _a, grad, *rest = field_gradient(verts, views, integrate_fn, return_color=return_color, group=group)
            colors = rest[0] if return_color else None
            norm = grad.norm(dim=1, keepdim=True)
            # alpha = 1 - (the opacity min_v alpha_integrated) rises from ~0 inside the surface to ~1 outside it, so grad alpha points out
            normals = torch.where(norm > 0, grad / torch.where(norm > 0, norm, torch.ones_like(norm)), torch.zeros_like(grad))
    elif return_color:
        with stage("evaluate_alpha_colors_s"):
            _a, colors = evaluate_alpha(verts, views, integrate_fn, return_color=True, group=group)
    return verts, colors, normals


@torch.no_grad()
def extract_level_set(points, points_scale, tets, views, integrate_fn, n_binary_steps=8, group=None, chunk_tets=None,
                      return_color=False, timings=None, return_normals=False):
    """marching_tetrahedra_with_binary_search (extract_mesh.py:37-120) up to the mesh arrays: opacity field on the tetrahedra
    vertices (view-sharded evaluate_alpha), marching tetrahedra on alpha - 0.5 (tet-chunk sharded), `n_binary_steps`
    bisection steps of every crossing edge, optional vertex colours and the reference's `distance <= scale` vertex mask.
    Returns dict(vertices (E,3), faces (F,3) int64, mask (E,) bool, colors (E,3) or None).
    return_normals=True (integrate_fn a CachedIntegrator) also returns "normals" (E,3): the field's outward unit normal at each
    vertex, grad alpha / |grad alpha| = -grad o / |grad o| for the opacity o = 1 - alpha, (0, 0, 0) where the gradient is zero,
    from one field_gradient pass that also gives the colours (DESIGN.md 4.14)."""
    stage = _stopwatch(timings, points.is_cuda)
    with stage("evaluate_alpha_vertices_s"):
        alpha = evaluate_alpha(points, views, integrate_fn, group=group)
    with stage("marching_tetrahedra_s"):
        (end_points, end_sdf), end_scales, faces, _iv = marching_tetrahedra_sharded(points, tets, alpha - 0.5, points_scale, group=group,
                                                                                 chunk_tets=chunk_tets)
    distance = torch.norm(end_points[:, 0, :] - end_points[:, 1, :], dim=-1)
    scale = end_scales[:, 0, 0] + end_scales[:, 1, 0]
    verts, colors, normals = _refine(end_points, end_sdf, views, integrate_fn, n_binary_steps, group, return_color, return_normals,
                                     stage)
    out = {"vertices": verts, "faces": faces, "mask": distance <= scale, "colors": colors}
    if return_normals:
        out["normals"] = normals
    return out


# ---- the entry points of the tetrahedra points and the field grid (csrc/tetra_points.cu, csrc/field_grid.cu) -------------
class _GridParams(ctypes.Structure):
    _fields_ = [("voxel_size", ctypes.c_float), ("block_resolution", ctypes.c_int)]


@functools.cache
def _tetra_lib():
    """(_C, its library) with the signatures of the tetra-point and field-grid entry points declared, on first use: gof_extract
    itself imports without the library."""
    from diff_gaussian_rasterization import _C
    lib, v, i32, i64, f, a = _C._lib, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, _C._ALLOC_FN
    P, i64p = ctypes.POINTER(_GridParams), ctypes.POINTER(ctypes.c_int64)
    for name, args in (
            ("gof_tetra_points", [i32, v, v, v, i32, v, f, f, v, v, v, v]),
            ("gof_frustum_mask", [i64, v, i32, v, f, f, v, v]),
            ("gof_field_grid_blocks_count", [P, i32, v, v, v, i32, v, f, f, a, v, a, v, i64p, v]),
            ("gof_field_grid_blocks_emit", [P, i32, v, v, i64, v, v]),
            ("gof_field_grid_points", [P, i64, v, v, v]),
            ("gof_field_grid_extract_count", [P, i64, v, v, a, v, i64p, i64p, v]),
            ("gof_field_grid_extract_emit", [P, i64, v, v, v, i64, i64, v, v, v, v])):
        getattr(lib, name).restype = ctypes.c_int
        getattr(lib, name).argtypes = args
    return _C, lib


def _gaussian_inputs(xyz, scales_with_filter, rotation, who):
    """get_tetra_points' inputs as the kernels read them: contiguous CUDA float32 xyz [P,3], scales [P,3], rotation [P,4]."""
    from gof_params import _f32
    x, s, q = _f32(xyz), _f32(scales_with_filter), _f32(rotation)
    P = int(x.shape[0])
    if tuple(x.shape) != (P, 3) or tuple(s.shape) != (P, 3) or tuple(q.shape) != (P, 4):
        raise ValueError(f"{who}: expected xyz [P,3], scales [P,3], rotation [P,4]; got {tuple(x.shape)}, "
                         f"{tuple(s.shape)}, {tuple(q.shape)}")
    return x, s, q


# ---- the tetrahedra points and their multi-view frustum mask (csrc/tetra_points.cu) ---------------------------------------
def pack_views(views, device):
    """[n,20] float32 table of gof_tetra_points / gof_frustum_mask from objects with the reference Camera's attributes
    (world_view_transform, focal_x, focal_y, image_width, image_height; scene/cameras.py).  The scalars are rounded to float32
    as the reference's `torch.Tensor([...])` rounds them."""
    views = list(views)
    if not views:
        raise ValueError("at least one view is needed (the reference reads views[0])")
    wvt = torch.stack([torch.as_tensor(v.world_view_transform).detach().to(device=device, dtype=torch.float32).reshape(16) for v in views])
    extra = torch.tensor([[v.focal_x, v.focal_y, v.image_width, v.image_height] for v in views], dtype=torch.float32)
    return torch.cat([wvt, extra.to(device)], dim=1).contiguous()


@torch.no_grad()
def get_tetra_points(xyz, scales_with_filter, rotation, views, near=0.02, far=1e6):
    """== GaussianModel.get_tetra_points (scene/gaussian_model.py:433-463) with xyz = gaussians.get_xyz,
    scales_with_filter = gaussians.get_scaling_with_3D_filter and rotation = gaussians._rotation (the raw quaternions;
    they are normalised here as build_rotation does).  Returns (points [M,3], points_scale [M,1]): the 8 corners of every
    Gaussian's 3-sigma box, then the centres, kept where some view's frustum holds them.  Width and height come from views[0]
    for every view, as in the reference."""
    _C, lib = _tetra_lib()
    x, s, q = _gaussian_inputs(xyz, scales_with_filter, rotation, "get_tetra_points")
    P = int(x.shape[0])
    table = pack_views(views, x.device)
    pts = torch.empty((9 * P, 3), dtype=torch.float32, device=x.device)
    sc = torch.empty((9 * P, 1), dtype=torch.float32, device=x.device)
    mask = torch.empty(9 * P, dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        _C._check(lib.gof_tetra_points(P, x.data_ptr(), s.data_ptr(), q.data_ptr(), int(table.shape[0]), table.data_ptr(), float(near),
                                       float(far), pts.data_ptr(), sc.data_ptr(), mask.data_ptr(), _C._stream()))
    return pts[mask], sc[mask]


@torch.no_grad()
def get_frustum_mask(points, cameras, near=0.02, far=1e6):
    """== get_frustum_mask (scene/gaussian_model.py:31-72): bool [N], True where the frustum of some camera holds the point
    (near <= depth <= far, 0 <= u <= W-1, 0 <= v <= H-1, with W and H of cameras[0])."""
    from gof_params import _f32
    _C, lib = _tetra_lib()
    p = _f32(points)
    N = int(p.shape[0])
    if tuple(p.shape) != (N, 3):
        raise ValueError(f"get_frustum_mask: expected points [N,3], got {tuple(p.shape)}")
    table = pack_views(cameras, p.device)
    mask = torch.empty(N, dtype=torch.bool, device=p.device)
    with torch.cuda.device(p.device):
        _C._check(lib.gof_frustum_mask(N, p.data_ptr(), int(table.shape[0]), table.data_ptr(), float(near), float(far), mask.data_ptr(),
                                       _C._stream()))
    return mask


# ---- the level set on a sparse voxel-block lattice, without tetrahedra (csrc/field_grid.cu, DESIGN §4.15) -----------------
_GOF_E_INVALID = -1
_MAX_LATTICE_POINTS = 2 ** 31


def _grid_check(_C, rc):
    """A refusal of the lattice's limits (GOF_E_INVALID) as ValueError with the library's message; other failures as _C._check."""
    if rc == _GOF_E_INVALID:
        _C._ALLOC_ERROR.exc = None
        raise ValueError(f"field grid: {_C._lib.gof_last_error().decode()}")
    _C._check(rc)


def _grid_params(voxel_size, block_resolution):
    import numpy as np
    B = int(block_resolution)
    s = float(np.float32(voxel_size))
    if not 1 <= B <= 64:
        raise ValueError(f"field grid: block_resolution must be in 1..64, got {block_resolution}")
    if not s > 0 or s == float("inf"):
        raise ValueError(f"field grid: voxel_size must be a finite float32 > 0, got {voxel_size}")
    return _GridParams(s, B)


@torch.no_grad()
def field_grid_blocks(xyz, scales_with_filter, rotation, views, voxel_size, block_resolution=8, near=0.02, far=1e6):
    """Sorted unique int64 keys [n] of the voxel blocks (B^3 voxels of size voxel_size) touched by the Gaussians whose centre some
    view's frustum holds (get_tetra_points' test): on each axis the blocks from floor((lo - s) / (B s)) to floor((hi + s) / (B s)),
    lo / hi the extent of the Gaussian's eight 3-sigma box corners.  Keys pack block coordinates as the TSDF volume's
    (gof_tsdf, DESIGN §4.4).  Inputs as get_tetra_points'."""
    _C, lib = _tetra_lib()
    par = _grid_params(voxel_size, block_resolution)
    x, s, q = _gaussian_inputs(xyz, scales_with_filter, rotation, "field_grid_blocks")
    P = int(x.shape[0])
    table = pack_views(views, x.device)
    gs, inst = _C._Scratch(x.device, "field_grid_gauss"), _C._Scratch(x.device, "field_grid_inst")
    n = ctypes.c_int64(0)
    with torch.cuda.device(x.device):
        _grid_check(_C, lib.gof_field_grid_blocks_count(ctypes.byref(par), P, x.data_ptr(), s.data_ptr(), q.data_ptr(),
                                                         int(table.shape[0]), table.data_ptr(), float(near), float(far), gs.cb, None,
                                                         inst.cb, None, ctypes.byref(n), _C._stream()))
        keys = torch.empty(n.value, dtype=torch.int64, device=x.device)
        if n.value:
            _grid_check(_C, lib.gof_field_grid_blocks_emit(ctypes.byref(par), P, gs.tensor.data_ptr(), inst.tensor.data_ptr(), n.value,
                                                            keys.data_ptr(), _C._stream()))
    return keys


def _grid_keys(keys, who):
    """Block keys as the kernels read them: a 1-D int64 tensor (they are read 8 bytes a key)."""
    if not isinstance(keys, torch.Tensor) or keys.dtype != torch.int64 or keys.dim() != 1:
        raise ValueError(f"{who}: keys must be a 1-D int64 tensor, got "
                         f"{keys.dtype if isinstance(keys, torch.Tensor) else type(keys).__name__} "
                         f"{tuple(keys.shape) if isinstance(keys, torch.Tensor) else ''}")
    return keys


def _grid_on_cuda(t, name, who, device=None):
    """Refuses, before any launch, a tensor the kernels cannot read: on the host, or on another device than `device`."""
    if not t.is_cuda:
        raise RuntimeError(f"gof_b200 {who}: {name} must be a CUDA tensor (no CPU path), got one on {t.device}")
    if device is not None and t.device != device:
        raise RuntimeError(f"gof_b200 {who}: {name} on {t.device}, keys on {device}")


def _check_lattice_size(num_blocks, block_resolution):
    n = int(num_blocks) * int(block_resolution) ** 3
    if n >= _MAX_LATTICE_POINTS:
        raise ValueError(f"field grid: {num_blocks} blocks of {int(block_resolution) ** 3} voxels make {n} lattice points; the "
                         f"opacity-field query takes fewer than 2^31 points (raise voxel_size)")


@torch.no_grad()
def field_grid_points(keys, voxel_size, block_resolution=8):
    """The lattice points [n B^3, 3] of the blocks `keys` (CUDA int64 [n], as field_grid_blocks returns them), in pool order
    (block, then voxel i + B j + B^2 k): voxel (x, y, z) = key B + (i, j, k) at (float(x) s, float(y) s, float(z) s), as the TSDF
    volume places it."""
    _C, lib = _tetra_lib()
    par = _grid_params(voxel_size, block_resolution)
    _grid_keys(keys, "field_grid_points")
    _check_lattice_size(keys.numel(), par.block_resolution)
    _grid_on_cuda(keys, "keys", "field_grid_points")
    pts = torch.empty((keys.numel() * par.block_resolution ** 3, 3), dtype=torch.float32, device=keys.device)
    if keys.numel():
        k = keys.contiguous()
        with torch.cuda.device(keys.device):
            _grid_check(_C, lib.gof_field_grid_points(ctypes.byref(par), k.numel(), k.data_ptr(), pts.data_ptr(), _C._stream()))
    return pts


@torch.no_grad()
def field_grid_marching_cubes(keys, values, voxel_size, block_resolution=8):
    """Marching cubes of `values` (float32 [n B^3], pool order, the level already subtracted) on the lattice of `keys` (CUDA int64
    [n], sorted, as field_grid_blocks returns them; values on the same device), with the TSDF extraction's table, winding
    (normals towards increasing value) and canonical order; a cube is meshed iff its eight corners lie in listed blocks.  Returns (edge_points [V,2,3], edge_values [V,2], faces [F,3] int64): every vertex as its lattice edge, the
    owner voxel's point and value first, then those of owner + axis."""
    _C, lib = _tetra_lib()
    par = _grid_params(voxel_size, block_resolution)
    who = "field_grid_marching_cubes"
    _grid_keys(keys, who)
    n, dev = int(keys.numel()), keys.device
    _check_lattice_size(n, par.block_resolution)
    if not isinstance(values, torch.Tensor) or tuple(values.shape) != (n * par.block_resolution ** 3,) or values.dtype != torch.float32:
        raise ValueError(f"{who}: values must be a float32 tensor [{n * par.block_resolution ** 3}], got "
                         f"{getattr(values, 'dtype', type(values).__name__)} {tuple(getattr(values, 'shape', ()))}")
    _grid_on_cuda(keys, "keys", who)
    _grid_on_cuda(values, "values", who, device=dev)
    k, v = keys.contiguous(), values.contiguous()
    scratch = _C._Scratch(dev)
    nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
    with torch.cuda.device(dev):
        _grid_check(_C, lib.gof_field_grid_extract_count(ctypes.byref(par), n, k.data_ptr() if n else None, v.data_ptr() if n else None,
                                                          scratch.cb, None, ctypes.byref(nv), ctypes.byref(nf), _C._stream()))
        ep = torch.empty((nv.value, 2, 3), dtype=torch.float32, device=dev)
        ev = torch.empty((nv.value, 2), dtype=torch.float32, device=dev)
        faces = torch.empty((nf.value, 3), dtype=torch.int64, device=dev)
        if nv.value or nf.value:
            _grid_check(_C, lib.gof_field_grid_extract_emit(ctypes.byref(par), n, k.data_ptr(), v.data_ptr(), scratch.tensor.data_ptr(),
                                                             nv.value, nf.value, ep.data_ptr(), ev.data_ptr(), faces.data_ptr(),
                                                             _C._stream()))
    return ep, ev, faces


@torch.no_grad()
def extract_level_set_grid(xyz, scales_with_filter, rotation, views, integrate_fn, voxel_size, block_resolution=8, n_binary_steps=8,
                           near=0.02, far=1e6, group=None, return_color=False, return_normals=False, timings=None):
    """The 0.5 level set of evaluate_alpha's field (1 - min over views of the integrated opacity) as a mesh, without Delaunay
    tetrahedra: the field is sampled on the voxel lattice (size voxel_size, blocks of block_resolution^3 voxels) of the blocks the
    Gaussians' 3-sigma boxes touch (field_grid_blocks), meshed by marching cubes on alpha - 0.5 (field_grid_marching_cubes), and
    every vertex is bisected `n_binary_steps` times on its lattice edge (binary_search), as extract_level_set does on the
    tetrahedra's edges.  Inputs: get_tetra_points' (get_xyz, get_scaling_with_3D_filter, the raw _rotation), the views, and the
    integrate_fn (a CachedIntegrator for return_normals) that extract_level_set takes.

    Returns dict(vertices (E,3), faces (F,3) int64, colors (E,3) or None); return_color: evaluate_alpha's colour at the vertices;
    return_normals: also "normals" (E,3), grad alpha / |grad alpha| from field_gradient ((0, 0, 0) where the gradient is zero),
    outward for GOF's field, with the colours from the same pass.  With torch.distributed initialised the field is view-sharded
    over the ranks of `group` as evaluate_alpha shards it; the blocks and marching cubes are deterministic and run on every rank,
    so every rank returns the same mesh.  ValueError for a bad voxel_size or block_resolution, a block outside [-2^20, 2^20) per
    axis, 2^30 or more (Gaussian, block) pairs, or a lattice of 2^31 points or more.  `timings` (dict): seconds per stage."""
    stage = _stopwatch(timings, xyz.is_cuda)
    with stage("blocks_s"):
        keys = field_grid_blocks(xyz, scales_with_filter, rotation, views, voxel_size, block_resolution, near, far)
    with stage("lattice_s"):
        points = field_grid_points(keys, voxel_size, block_resolution)
    with stage("evaluate_alpha_lattice_s"):
        sdf = evaluate_alpha(points, views, integrate_fn, group=group) - 0.5
        del points
    with stage("marching_cubes_s"):
        end_points, end_sdf, faces = field_grid_marching_cubes(keys, sdf, voxel_size, block_resolution)
        del sdf
    verts, colors, normals = _refine(end_points, end_sdf.unsqueeze(-1), views, integrate_fn, n_binary_steps, group, return_color,
                                     return_normals, stage)
    out = {"vertices": verts, "faces": faces, "colors": colors}
    if return_normals:
        out["normals"] = normals
    return out
