"""Level-set extraction helpers around GaussianRasterizer.integrate -- the callers of the integrate path in the
reference's extract_mesh.py, restated with view sharding over the GPUs of one box.

* evaluate_alpha    == evaluage_alpha (extract_mesh.py:17-34): alpha = 1 - min over views of the integrated opacity,
                       optionally the colour of the arg-min view.  `min` is associative, so with torch.distributed
                       initialised every rank processes views[rank::world] and the partial minima are merged with one
                       all_reduce(MIN) (colour: the lowest view index attaining the minimum wins, like the reference's
                       strict `<` update in view order).
* binary_search     == the 8-step bisection of extract_mesh.py:88-102 on the edge endpoints returned by
                       gof_tetmesh.marching_tetrahedra.
* make_integrate_fn == gaussian_renderer.integrate (gaussian_renderer/__init__.py:118-218) for plain tensors.
* CachedIntegrator  -- the same, with the Gaussian side of every view prepared once and reused by all passes (SURVEY 8(f) rank 3).
* marching_tetrahedra_sharded / merge_tet_shards -- utils/tetmesh.py's chunk loop (:55-95) spread over ranks (SURVEY 8(e)).
* extract_level_set -- marching_tetrahedra_with_binary_search (extract_mesh.py:37-120) up to the mesh arrays.
"""
import torch
import torch.distributed as dist


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


@torch.no_grad()
def evaluate_alpha(points, views, integrate_fn, return_color=False, group=None):
    """integrate_fn(points, view) -> (alpha_integrated [N], color_integrated [N,3])."""
    rank, world = _world(group)
    n, dev = points.shape[0], points.device
    final_alpha = torch.ones(n, dtype=torch.float32, device=dev)
    final_color = torch.ones(n, 3, dtype=torch.float32, device=dev) if return_color else None
    best_view = torch.full((n,), 2 ** 30, dtype=torch.int32, device=dev) if return_color else None
    views = list(views)
    for vi in range(rank, len(views), world):
        alpha_integrated, color_integrated = integrate_fn(points, views[vi])
        if return_color:
            better = alpha_integrated < final_alpha
            final_color = torch.where(better.reshape(-1, 1), color_integrated, final_color)
            best_view = torch.where(better, torch.full_like(best_view, vi), best_view)
        final_alpha = torch.min(final_alpha, alpha_integrated)
    if world > 1:
        local_alpha = final_alpha.clone()
        dist.all_reduce(final_alpha, op=dist.ReduceOp.MIN, group=group)
        if return_color:
            # the winner is the lowest view index whose alpha equals the global minimum (and is < 1, the initial value)
            cand = torch.where((local_alpha == final_alpha) & (local_alpha < 1.0), best_view, torch.full_like(best_view, 2 ** 30))
            win = cand.clone()
            dist.all_reduce(win, op=dist.ReduceOp.MIN, group=group)
            mine = (cand == win) & (win < 2 ** 30)
            contrib = torch.where(mine.reshape(-1, 1), final_color, torch.zeros_like(final_color))
            dist.all_reduce(contrib, op=dist.ReduceOp.SUM, group=group)
            final_color = torch.where((win < 2 ** 30).reshape(-1, 1), contrib, torch.ones_like(contrib))
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

    @property
    def cached_bytes(self):
        return sum(c.nbytes for _v, _rs, c in self._cache.values())

    def clear(self):
        self._cache.clear()


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


def _reference_chunk_rows(num_tets, chunk_tets):
    if chunk_tets <= 0 or num_tets <= chunk_tets:
        return max(int(num_tets), 1)
    n = num_tets // chunk_tets + 1
    return -(-num_tets // n)


@torch.no_grad()
def marching_tetrahedra_sharded(vertices, tets, sdf, scales, group=None, chunk_tets=None, extract_fn=None):
    """`gof_tetmesh.marching_tetrahedra` for ONE batch element with the tets sharded by chunk over the ranks of `group`:
    each rank extracts its chunks, ONE all-gather exchanges the crossing-edge keys and the faces (as edge keys), every rank
    ends with the complete mesh -- bit-identical to the unsharded call (faces are ordered per chunk, so shards are whole
    chunks of the unsharded split; with fewer chunks than ranks some ranks idle).  vertices (N,3), tets (T,4), sdf (N,),
    scales (N,1).  World size 1: the plain call.  `extract_fn(vertices, tets, sdf, scales, rows=...)` defaults to the CUDA
    implementation (tests pass the oracle)."""
    if extract_fn is None:
        import gof_tetmesh
        extract_fn = lambda v, t, s, sc, rows: gof_tetmesh._unbatched_marching_tetrahedra(v, t, s, sc, rows=rows)   # noqa: E731
    chunk = int(chunk_tets or 32 * 1024 * 1024)    # utils/tetmesh.py:55
    rank, world = _world(group)
    T = int(tets.shape[0])
    rows = _reference_chunk_rows(T, chunk)
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
    # one padded all-gather carries both the keys and the faces (as global keys: renumbering then needs no second exchange)
    face_keys = keys[faces.reshape(-1)] if faces.numel() else torch.zeros(0, dtype=torch.int64, device=dev)
    payload = torch.full((nk + 3 * nf,), -1, dtype=torch.int64, device=dev)
    payload[:keys.numel()] = keys
    payload[nk:nk + face_keys.numel()] = face_keys
    gathered = [torch.empty_like(payload) for _ in range(world)]
    dist.all_gather(gathered, payload, group=group)
    shard_keys = [g[:int(s[0])] for g, s in zip(gathered, all_sizes)]
    union = torch.unique(torch.cat(shard_keys))
    faces_all = torch.cat([torch.searchsorted(union, g[nk:nk + 3 * int(s[1])]).reshape(-1, 3) for g, s in zip(gathered, all_sizes)])
    interp = torch.stack([union >> 32, union & 0xFFFFFFFF], dim=1)
    v = vertices.reshape(-1, 3)
    edge_pos = v[interp.reshape(-1)].reshape(-1, 2, 3)
    edge_sdf = sdf.reshape(-1)[interp.reshape(-1)].reshape(-1, 2, 1)
    edge_scales = scales.reshape(-1)[interp.reshape(-1)].reshape(-1, 2, 1)
    return (edge_pos, edge_sdf), edge_scales, faces_all, interp


@torch.no_grad()
def extract_level_set(points, points_scale, tets, views, integrate_fn, n_binary_steps=8, group=None, chunk_tets=None,
                      return_color=False, timings=None):
    """marching_tetrahedra_with_binary_search (extract_mesh.py:37-120) up to the mesh arrays: opacity field on the tetrahedra
    vertices (view-sharded evaluate_alpha), marching tetrahedra on alpha - 0.5 (tet-chunk sharded), `n_binary_steps`
    bisection steps of every crossing edge, optional vertex colours and the reference's `distance <= scale` vertex mask.
    Returns dict(vertices (E,3), faces (F,3) int64, mask (E,) bool, colors (E,3) or None)."""
    import time as _time

    def tick(name, t0):
        if timings is not None:
            torch.cuda.synchronize() if points.is_cuda else None
            timings[name] = timings.get(name, 0.0) + (_time.perf_counter() - t0)

    t0 = _time.perf_counter()
    alpha = evaluate_alpha(points, views, integrate_fn, group=group)
    tick("evaluate_alpha_vertices_s", t0)
    t0 = _time.perf_counter()
    (end_points, end_sdf), end_scales, faces, _iv = marching_tetrahedra_sharded(points, tets, alpha - 0.5, points_scale, group=group,
                                                                             chunk_tets=chunk_tets)
    tick("marching_tetrahedra_s", t0)
    distance = torch.norm(end_points[:, 0, :] - end_points[:, 1, :], dim=-1)
    scale = end_scales[:, 0, 0] + end_scales[:, 1, 0]
    t0 = _time.perf_counter()
    verts = binary_search(end_points, end_sdf, lambda p: evaluate_alpha(p, views, integrate_fn, group=group), n_steps=n_binary_steps)
    tick("binary_search_s", t0)
    colors = None
    if return_color:
        t0 = _time.perf_counter()
        _a, colors = evaluate_alpha(verts, views, integrate_fn, return_color=True, group=group)
        tick("evaluate_alpha_colors_s", t0)
    return {"vertices": verts, "faces": faces, "mask": distance <= scale, "colors": colors}
