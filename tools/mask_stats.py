#!/usr/bin/env python
"""Lane-utilisation statistics of the blend kernels from the forward's blend masks and alpha-support boxes (GPU box).

For one view of a config it answers: how many (pixel block, Gaussian) visits do the forward (box hits) and the backward
(blocks with >= 1 blended pixel) make for block shapes 8x4 (a warp today), 4x4, 4x2 and 2x2 -- and how many warp iterations
result if the sub-blocks of a warp walk INDEPENDENT lists in lockstep (max over the sub-blocks, per group of 32 list
entries or per batch of 256).  Developer tool; prints one JSON line and writes tool_out/mask_stats_<cfg>.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
import _util  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import _C as ours  # noqa: E402


def popc(x):
    x = x.to(torch.int64) & 0xFFFFFFFF
    x = x - ((x >> 1) & 0x55555555)
    x = (x & 0x33333333) + ((x >> 2) & 0x33333333)
    x = (x + (x >> 4)) & 0x0F0F0F0F
    return ((x * 0x01010101) & 0xFFFFFFFF) >> 24


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "C3"
    view = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(name, view=view)
    fa = _util.fwd_args(cam, gs, dev)
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    R, color, radii, geom, binning, img = ours.rasterize_gaussians(*fa)
    torch.cuda.synchronize()
    st = ours.export_state(P, W, H, R, geom, binning, img, radii, masks=True)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tiles = gx * gy
    ranges = st["ranges"].to(torch.int64)                       # [tiles,2]
    lens = ranges[:, 1] - ranges[:, 0]
    ngroups = (lens + 31) // 32
    G = int(ngroups.sum())
    tile_of_group = torch.repeat_interleave(torch.arange(tiles, device=dev), ngroups)
    first_group = torch.cumsum(ngroups, 0) - ngroups
    g_in_tile = torch.arange(G, device=dev) - first_group[tile_of_group]
    gstart = ranges[tile_of_group, 0] + 32 * tile_of_group + 32 * g_in_tile      # word offset of lane 0
    vm = st["blend_masks"]                                                       # [8, R + 32*tiles]
    idx = gstart[:, None] + torch.arange(32, device=dev)[None, :]                # [G,32]
    words = vm[:, idx]                                                          # [8,G,32]
    # validity: group g of (tile, warp) was written iff 32*g < warp_last (max last_contributor of the warp's 32 pixels)
    last = st["n_contrib"][0].to(torch.int64)                                    # [H,W]
    pad = torch.zeros(gy * 16, gx * 16, dtype=torch.int64, device=dev)
    pad[:H, :W] = last
    blk = pad.view(gy, 4, 4, gx, 2, 8)                                           # tile_y, warp_row, y_in, tile_x, warp_col, x_in
    pix_last = blk.permute(0, 3, 1, 4, 2, 5).reshape(tiles, 8, 32)               # [tile, warp, lane]
    warp_last = pix_last.amax(dim=2)                                             # [tiles,8]
    valid = (32 * g_in_tile)[None, :] < warp_last[tile_of_group].t()            # [8,G]
    words = torch.where(valid[:, :, None], words, torch.zeros_like(words))
    # entries beyond the tile's list length cannot be set; bits for lanes outside the image are zero by construction
    lane = torch.arange(32, device=dev)
    lx, ly = lane & 7, lane >> 3
    out = {"config": name, "view": view, "R": int(R), "visible": int((radii > 0).sum()), "groups": G,
           "pairs_blended": int(popc(words).sum())}

    def or_over(mask_lanes):
        sel = words[:, :, mask_lanes]
        acc = sel[:, :, 0]
        for k in range(1, sel.shape[2]):
            acc = acc | sel[:, :, k]
        return acc                                                               # [8,G]

    # batch id: (tile, g_in_tile // 8)
    batch_id = tile_of_group * 64 + (g_in_tile // 8)
    uniq, inv = torch.unique(batch_id, return_inverse=True)
    shapes = {"8x4": [lane >= 0], "4x4": [lx < 4, lx >= 4], "4x2": [(lx < 4) & (ly < 2), (lx >= 4) & (ly < 2), (lx < 4) & (ly >= 2), (lx >= 4) & (ly >= 2)],
              "2x2": [((lx // 2) == a) & ((ly // 2) == b) for a in range(4) for b in range(2)]}
    bw = {}
    for sname, subs in shapes.items():
        cnts = torch.stack([popc(or_over(torch.nonzero(m).flatten())) for m in subs], 0)   # [S,8,G]
        visits = int(cnts.sum())
        lock_group = int(cnts.amax(dim=0).sum())
        per_batch = torch.zeros(len(subs), 8, uniq.numel(), dtype=torch.int64, device=dev)
        per_batch.index_add_(2, inv, cnts)
        lock_batch = int(per_batch.amax(dim=0).sum())
        bw[sname] = {"block_visits": visits, "warp_iters_lockstep_group32": lock_group, "warp_iters_lockstep_batch256": lock_batch,
                     "lanes_active_per_visit": out["pairs_blended"] / max(visits, 1) }
    out["backward"] = bw

    # ---- forward: alpha-support box hits per block shape, up to the block's saturation point -------------------------
    rec = geom[:P * 64].view(torch.int32).view(P, 16)
    pl = st["point_list"].to(torch.int64)
    box_lo, box_hi = rec[:, 14], rec[:, 15]
    x0 = ((box_lo << 16) >> 16).to(torch.int64); y0 = (box_lo >> 16).to(torch.int64)
    x1 = ((box_hi << 16) >> 16).to(torch.int64); y1 = (box_hi >> 16).to(torch.int64)
    ent_tile = torch.repeat_interleave(torch.arange(tiles, device=dev), lens)
    ent_pos = torch.arange(int(lens.sum()), device=dev) - ranges[ent_tile, 0]     # 0-based position in the tile list
    ex0, ey0, ex1, ey1 = x0[pl], y0[pl], x1[pl], y1[pl]
    tx, ty = (ent_tile % gx) * 16, (ent_tile // gx) * 16
    fw = {}
    pix_last_t = pad.view(gy, 16, gx, 16).permute(0, 2, 1, 3).reshape(tiles, 16, 16)        # [tile, y, x]
    ent_group = ent_tile * 4096 + ent_pos // 32
    ent_batch = ent_tile * 4096 + ent_pos // 256
    ug, invg = torch.unique(ent_group, return_inverse=True)
    ub, invb = torch.unique(ent_batch, return_inverse=True)
    for sname, (bwid, bhei) in {"8x4": (8, 4), "4x4": (4, 4), "4x2": (4, 2), "2x2": (2, 2)}.items():
        nbx, nby = 16 // bwid, 16 // bhei
        blast = pix_last_t.view(tiles, nby, bhei, nbx, bwid).amax(dim=(2, 4))      # [tiles, nby, nbx]: the block's last blended entry (1-based)
        hits_total = 0
        warps = 8
        per_warp_sub = (nbx * nby) // warps                                         # sub-blocks per warp
        cnt_g = torch.zeros(nbx * nby, ug.numel(), dtype=torch.int64, device=dev)
        cnt_b = torch.zeros(nbx * nby, ub.numel(), dtype=torch.int64, device=dev)
        for by in range(nby):
            for bx in range(nbx):
                wx0, wy0 = tx + bx * bwid, ty + by * bhei
                hit = (ex0 <= wx0 + bwid - 1) & (ex1 >= wx0) & (ey0 <= wy0 + bhei - 1) & (ey1 >= wy0)
                # the block keeps walking until all its pixels are done: approximated by its last blended entry + the
                # (unknown) tail up to saturation; entries beyond blast only count when the block never saturated -> use blast
                # for saturated blocks is a lower bound; report both bounds
                alive = ent_pos < blast[ent_tile, by, bx]
                h = (hit & alive).to(torch.int64)
                hits_total += int(h.sum())
                cnt_g[by * nbx + bx].index_add_(0, invg, h)
                cnt_b[by * nbx + bx].index_add_(0, invb, h)
        # group the sub-blocks of one warp: 8x4 warp footprint = consecutive sub-blocks inside it
        def lock(cnt):
            # sub-block (by,bx) belongs to warp ((by*bhei)//4)*2 + (bx*bwid)//8
            wid = torch.tensor([((by * bhei) // 4) * 2 + (bx * bwid) // 8 for by in range(nby) for bx in range(nbx)], device=dev)
            tot = 0
            for w in range(8):
                tot += int(cnt[wid == w].amax(dim=0).sum())
            return tot
        fw[sname] = {"block_visits_until_last_blend": hits_total, "warp_iters_lockstep_group32": lock(cnt_g),
                     "warp_iters_lockstep_batch256": lock(cnt_b)}
    out["forward_box_hits"] = fw
    print(json.dumps(out))
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "tool_out", f"mask_stats_{name}.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
