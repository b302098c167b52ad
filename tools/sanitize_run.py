#!/usr/bin/env python
"""Small end-to-end pass over every CUDA entry point, meant to run under compute-sanitizer (GPU box):

    compute-sanitizer --tool memcheck|racecheck|initcheck|synccheck python tools/sanitize_run.py [parts...]

parts: render (forward + backward, SH and precomputed-colour paths, multi-batch tile lists), integrate, tetmesh, loss,
params, filter, tsdf (touch / activate with pool growth / integrate / marching cubes), knn (distCUDA2 on clouds of
1-4097 points, coincident and non-finite rows included), sort (the multi-word sort, key runs and scan at n = 1 and 4097, three
words), appearance (the weight-gradient kernel of the appearance network, several tiles per CTA).  Sizes are tiny on purpose (the tools slow kernels down 100-1000x).  Exit code 0 = every call returned."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("gaussian-opacity-fields_b200", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import _util  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import _C  # noqa: E402


def render(dev):
    # (a) ordinary scene, image size not a tile multiple; (b) big splats: tile lists longer than one 256-entry batch
    for cfg, view, sigma in ((dict(P=3000, width=136, height=88, seed=11), 3, 2.0), (dict(P=1500, width=64, height=48, seed=12, sigma_px=14.0), 5, 14.0)):
        cam, gs = gof_synth.make_scene(cfg, view=view)
        fa = _util.fwd_args(cam, gs, dev, bg=(0.2, 0.1, 0.3))
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
        grad = torch.randn(9, cam.image_height, cam.image_width, device=dev)
        _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
        _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))     # twice on the same buffers
        torch.cuda.synchronize()
        print("render", cfg, "R =", R, "visible =", int((radii > 0).sum()), flush=True)
    cols = torch.rand(3000, 3)
    cam, gs = gof_synth.make_scene(dict(P=3000, width=136, height=88, seed=11), view=3)
    fa = _util.fwd_args(cam, gs, dev, colors_precomp=cols)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, torch.randn(9, 88, 136, device=dev)))
    _C.mark_visible(gs["means3D"].to(dev), cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev))
    torch.cuda.synchronize()


def integrate(dev):
    cam, gs = gof_synth.make_scene(dict(P=3000, width=136, height=88, seed=11), view=3)
    fa = _util.fwd_args(cam, gs, dev)
    pts = ((torch.rand(20_000, 3) * 2 - 1) * 1.6).to(dev)
    out = _C.integrate_gaussians_to_points(fa[0], pts, *fa[1:])
    torch.cuda.synchronize()
    print("integrate R =", out[0], "alpha mean", float(out[2].mean()), flush=True)


def tetmesh(dev):
    import gof_tetmesh
    z = np.load(os.path.join(ROOT, "tests", "golden", "tetmesh_noisy.npz"))
    t = lambda k: torch.from_numpy(z[k]).to(dev)
    (pos, esdf), esc, faces, iv = gof_tetmesh._unbatched_marching_tetrahedra(t("vertices"), t("tets"), t("sdf"), t("scales"))
    torch.cuda.synchronize()
    print("tetmesh faces", tuple(faces.shape), flush=True)
    (pos, esdf), esc, faces, iv = gof_tetmesh._unbatched_marching_tetrahedra(t("vertices"), t("tets"), t("sdf"), t("scales"), chunk_tets=1000)
    torch.cuda.synchronize()


def loss(dev):
    import gof_loss
    cam, _ = gof_synth.make_scene(dict(P=10, width=100, height=70, seed=1), view=4)
    img = torch.rand(9, 70, 100, device=dev, requires_grad=True)
    gt = torch.rand(3, 70, 100, device=dev)
    l, _terms = gof_loss.view_loss(img, gt, cam.world_view_transform, cam.tanfovx, cam.tanfovy, 0.2, 0.05, 100.0)
    l.backward()
    torch.cuda.synchronize()
    print("loss", float(l), flush=True)


def params(dev):
    import gof_params
    P = 2001
    raw = [torch.randn(P, 3), torch.randn(P, 4), torch.randn(P, 1), torch.rand(P, 1) * 0.01, torch.randn(P, 1, 3), torch.randn(P, 15, 3)]
    raw = [r.to(dev).requires_grad_(i != 3) for i, r in enumerate(raw)]
    outs = gof_params.activate(*raw)
    sum(o.sum() for o in outs).backward()
    p = torch.randn(P * 3, device=dev)
    gof_params.adam_step(p, torch.zeros_like(p), torch.zeros_like(p), torch.randn_like(p), 1e-3, 1)
    torch.cuda.synchronize()
    print("params ok", flush=True)


def filt(dev):
    import gof_params
    z = np.load(os.path.join(ROOT, "tests", "golden", "filter3d_a.npz"))
    out = gof_params.compute_3d_filter(torch.from_numpy(z["xyz"]).to(dev), torch.from_numpy(z["cams"]).to(dev), float(z["cams"][:, 12].max()))
    torch.cuda.synchronize()
    print("filter mean", float(out.mean()), flush=True)


def tsdf(dev):
    import gof_tsdf
    # a few 64x48 views with B = 8: noisy depth around a plane (ambiguous cubes, blocks shared between views), one view with no
    # depth, a pool that starts at one block and grows; then the whole extraction
    rng = np.random.default_rng(5)
    vol = gof_tsdf.TSDFVolume(voxel_size=0.05, block_resolution=8, block_count=1, device=dev)
    for i in range(6):
        d = (3.0 + 0.15 * rng.standard_normal((48, 64))).astype(np.float32)
        if i == 3:
            d[:] = 0
        E = np.eye(4, dtype=np.float32)
        E[:3, 3] = rng.normal(0, 0.05, 3)
        vol.integrate(torch.from_numpy(d).to(dev), torch.rand(3, 48, 64, device=dev), 40.0, 40.0, 31.5, 23.5, E)
    mesh = vol.extract_triangle_mesh(3.0)
    torch.cuda.synchronize()
    print("tsdf blocks", vol.num_blocks, "V", tuple(mesh["vertices"].shape), "F", tuple(mesh["faces"].shape), flush=True)


def knn(dev):
    from simple_knn._C import distCUDA2
    for kind, P in (("colmap", 4097), ("nonfinite", 1025), ("lattice", 33), ("uniform", 1)):
        out = distCUDA2(torch.from_numpy(gof_synth.make_point_cloud(kind, P, seed=3)).to(dev))
        torch.cuda.synchronize()
        print("knn", kind, P, "finite", int(torch.isfinite(out).sum()), flush=True)


def sort(dev):
    # the sort, run and scan primitives through their test entry points: one item, a chunk and a key, three words (w[0] == ka)
    from test_gpu_sort_primitives import _bind, _words_arg
    lib = _bind(_C._lib)
    st = _C._stream()
    g = torch.Generator().manual_seed(7)
    for n in (1, 4097):
        bits = (32, 31, 9)
        words = [torch.randint(-2**31, 2**31, (n,), dtype=torch.int32, generator=g).to(dev) for _ in bits]
        kb, va, vb, head, run = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(5))
        ka = words[0]
        hist = torch.empty(int(lib.gof_probe_scratch_bytes(0, n)), dtype=torch.uint8, device=dev)
        tmp = torch.empty(int(lib.gof_probe_scratch_bytes(1, n)), dtype=torch.uint8, device=dev)
        total = torch.empty(1, dtype=torch.int32, device=dev)
        wp, bp = _words_arg([w.data_ptr() for w in words], bits)
        _C._check(lib.gof_probe_sort_words_u32(3, wp, bp, n, ka.data_ptr(), kb.data_ptr(), va.data_ptr(), vb.data_ptr(), hist.data_ptr(), 1, st))
        _C._check(lib.gof_probe_key_runs_u32(3, wp, bp, vb.data_ptr(), n, head.data_ptr(), run.data_ptr(), tmp.data_ptr(), total.data_ptr(), st))
        _C._check(lib.gof_probe_exclusive_scan_u32(run.data_ptr(), head.data_ptr(), tmp.data_ptr(), total.data_ptr(), n, st))
        torch.cuda.synchronize()
        print("sort n =", n, "scan total", int(total.item()) & 0xFFFFFFFF, flush=True)


def appearance(dev):
    # the appearance network's weight gradient (conv_wgrad.cu) for every channel pair: W % 4 == 0 (cp.async double buffer) with
    # 1 024+ tiles, i.e. at least 3 per CTA of the persistent grid on an H100, so that the prefetch, the buffer swap and the refill
    # barrier run; the scalar fill (odd W); and an image smaller than one tile
    import gof_appearance
    lib = gof_appearance._wgrad_lib()
    g = torch.Generator().manual_seed(3)
    for (co, ci), (H, W) in (((16, 16), (264, 1024)), ((3, 16), (264, 1024)), ((16, 8), (264, 1024)), ((16, 16), (257, 1021)), ((3, 16), (5, 20))):
        x = torch.randn(ci, H, W, generator=g).to(dev)
        gy = torch.randn(co, H, W, generator=g).to(dev)
        dW, db = torch.zeros(co, ci, 3, 3, device=dev), torch.zeros(co, device=dev)
        _C._check(lib.gof_conv3x3_wgrad(co, ci, H, W, x.data_ptr(), gy.data_ptr(), dW.data_ptr(), db.data_ptr(), _C._stream()))
        torch.cuda.synchronize()
        print("appearance", (co, ci), (H, W), "|dW|max", float(dW.abs().max()), flush=True)


PARTS = {"render": render, "integrate": integrate, "tetmesh": tetmesh, "loss": loss, "params": params, "filter": filt, "tsdf": tsdf,
         "knn": knn, "sort": sort, "appearance": appearance}

if __name__ == "__main__":
    dev = torch.device("cuda")
    for name in (sys.argv[1:] or list(PARTS)):
        PARTS[name](dev)
    print("SANITIZE_RUN_DONE", flush=True)
