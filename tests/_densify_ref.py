"""A plain restatement of GaussianModel.densify_and_prune (scene/gaussian_model.py:631-707 with densify_and_clone,
densify_and_split, densification_postfix, cat_tensors_to_optimizer, prune_points and _prune_optimizer, :549-681) in torch,
written from the semantics, for the tests of gof_densify (csrc/densify.cu).

It runs the reference's three steps in the reference's order, with boolean masks and torch.cat over every per-row tensor:
  clone   Gaussians with (|grad| >= max_grad or |grad_abs| >= Q) and max scale <= percent_dense * extent get one new row,
          position R(q) (s * e) + x with e = noise[0] of the parent, everything else copied;
  split   over the n rows after the clone, with both gradients zero-padded from P to n (:634-640), the selected Gaussians
          with max scale > percent_dense * extent get two new rows (first all first children, then all second children),
          positions R(q) (s * e) + x with e = noise[1] / noise[2] of the parent, raw scaling log(s / (0.8 * 2)); the parents
          are then removed;
  prune   rows with sigmoid(opacity) < min_opacity, and, when max_screen_size is truthy, rows whose max_radii2D exceeds it
          (all zero here: densification_postfix has just reset them) or whose max scale exceeds 0.1 * extent.
New rows carry zero Adam moments.  Besides the tensors, every row carries its source Gaussian and its kind (0 kept original,
1 clone, 2 / 3 first / second split child), so the result can be held against gof_densify's src_index / kind.

torch.normal(0, std) is the one call not restated: the samples are std * the given standard-normal `noise` ([3, P, 3]: clone,
first child, second child, indexed by the parent), the same samples gof_densify's `noise=` path consumes.

Two modes.  fp64=False: every operation in float32 on the inputs' device with torch's own exp / log / sigmoid / division /
quantile, exactly the operations the reference issues -- the reference for every decision, the row order and every gathered
tensor, bit for bit.  fp64=True: the same decisions (they are the reference's float32 decisions by definition), but the new
rows' positions and raw scalings evaluated in float64 from the float32 inputs as well, returned beside the float32 result
as "xyz64" / "scaling64" (every row; the kept and cloned rows' values are their float32 inputs, widened).

Two deliberate departures, both where the reference cannot run as written: P = 0 (torch.quantile refuses an empty input; the
result here is empty, as gof_densify's), and a single surviving row when max_screen_size is falsy (the reference's
`.squeeze()` makes the prune mask 0-d there, and indexing with a 0-d mask adds a dimension; the mask here stays 1-d)."""
import torch

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def build_rotation(q):
    """utils/general_utils.py:78-99: the rotation matrix of the normalised quaternion (r, x, y, z), in q's dtype."""
    q = q / torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])[:, None]
    r, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def grads_and_threshold(accum, accum_abs, denom, max_grad):
    """(grads [P, 1], grads_abs [P, 1], Q): the mean gradients with NaN -> 0 and the quantile of :684-690 (P > 0)."""
    grads = accum.reshape(-1, 1) / denom.reshape(-1, 1)
    grads[grads.isnan()] = 0.0
    grads_abs = accum_abs.reshape(-1, 1) / denom.reshape(-1, 1)
    grads_abs[grads_abs.isnan()] = 0.0
    ratio = (torch.norm(grads, dim=-1) >= max_grad).float().mean()
    return grads, grads_abs, torch.quantile(grads_abs.reshape(-1), 1 - ratio)


def densify_and_prune(params, exp_avg, exp_avg_sq, accum, accum_abs, denom, max_grad, min_opacity, extent, max_screen_size,
                      noise, percent_dense=0.01, fp64=False):
    """Returns dict(params, exp_avg, exp_avg_sq, src_index (int64), kind (uint8), counts) in gof_densify's layout, and with
    fp64 also xyz64 / scaling64; counts = (kept originals, clones, first children, second children) of the final rows."""
    P = int(params["xyz"].shape[0])
    dev = params["xyz"].device
    rows = {}
    for k in GROUPS:
        rows[k], rows["m_" + k], rows["v_" + k] = params[k], exp_avg[k], exp_avg_sq[k]
    rows["src"], rows["kind"] = torch.arange(P, device=dev), torch.zeros(P, dtype=torch.uint8, device=dev)
    if fp64:
        rows["xyz64"], rows["scaling64"] = params["xyz"].double(), params["scaling"].double()

    def select(mask):
        return {k: t[mask] for k, t in rows.items()}

    def postfix(new):                              # densification_postfix + cat_tensors_to_optimizer
        for k in GROUPS:
            new["m_" + k] = torch.zeros_like(new[k])
            new["v_" + k] = torch.zeros_like(new[k])
        for k in rows:
            rows[k] = torch.cat((rows[k], new[k]), dim=0)

    def prune(mask):                               # prune_points + _prune_optimizer
        for k in rows:
            rows[k] = rows[k][~mask]

    def scaling():
        return torch.exp(rows["scaling"])

    def positions(sel, e, reps):
        """R(q) (std * e) + x of the selected rows, each repeated `reps` times; and its fp64 twin."""
        stds = scaling()[sel].repeat(reps, 1)
        new = torch.bmm(build_rotation(rows["rotation"][sel]).repeat(reps, 1, 1), (stds * e).unsqueeze(-1)).squeeze(-1)
        new = new + rows["xyz"][sel].repeat(reps, 1)
        if not fp64:
            return new, None
        s64 = torch.exp(rows["scaling64"][sel]).repeat(reps, 1)
        R64 = build_rotation(rows["rotation"][sel].double()).repeat(reps, 1, 1)
        return new, torch.bmm(R64, (s64 * e.double()).unsqueeze(-1)).squeeze(-1) + rows["xyz64"][sel].repeat(reps, 1)

    if P:
        grads, grads_abs, Q = grads_and_threshold(accum, accum_abs, denom, max_grad)
        # densify_and_clone
        sel = (torch.norm(grads, dim=-1) >= max_grad) | (torch.norm(grads_abs, dim=-1) >= Q)
        sel = sel & (torch.max(scaling(), dim=1).values <= percent_dense * extent)
        new = select(sel)
        new["xyz"], x64 = positions(sel, noise[0][rows["src"][sel]], 1)
        if fp64:
            new["xyz64"] = x64
        new["kind"] = torch.full_like(new["kind"], 1)
        postfix(new)
        # densify_and_split, the gradients zero-padded to the rows after the clone
        n = rows["xyz"].shape[0]
        pg, pga = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        pg[:P], pga[:P] = grads.reshape(-1), grads_abs.reshape(-1)
        sel = (pg >= max_grad) | (pga >= Q)
        sel = sel & (torch.max(scaling(), dim=1).values > percent_dense * extent)
        parents = rows["src"][sel]
        new = {k: torch.cat([t[sel]] * 2) for k, t in rows.items()}
        new["xyz"], x64 = positions(sel, torch.cat([noise[1][parents], noise[2][parents]]), 2)
        new["scaling"] = torch.log(scaling()[sel].repeat(2, 1) / (0.8 * 2))
        if fp64:
            new["xyz64"] = x64
            new["scaling64"] = torch.log(torch.exp(rows["scaling64"][sel]).repeat(2, 1) / (0.8 * 2))
        m = int(sel.sum())
        new["kind"] = torch.cat([torch.full((m,), 2, dtype=torch.uint8, device=dev), torch.full((m,), 3, dtype=torch.uint8, device=dev)])
        postfix(new)
        prune(torch.cat((sel, torch.zeros(2 * m, device=dev, dtype=torch.bool))))
        # the final prune
        n = rows["xyz"].shape[0]
        max_radii2D = torch.zeros(n, device=dev)
        mask = (torch.sigmoid(rows["opacity"]) < min_opacity).reshape(-1)
        if max_screen_size:
            mask = mask | (max_radii2D > max_screen_size) | (scaling().max(dim=1).values > 0.1 * extent)
        prune(mask)

    kind = rows["kind"]
    out = dict(params={k: rows[k] for k in GROUPS}, exp_avg={k: rows["m_" + k] for k in GROUPS},
               exp_avg_sq={k: rows["v_" + k] for k in GROUPS}, src_index=rows["src"], kind=kind,
               counts=tuple(int((kind == k).sum()) for k in range(4)))
    if fp64:
        out["xyz64"], out["scaling64"] = rows["xyz64"], rows["scaling64"]
    return out
