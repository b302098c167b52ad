#!/usr/bin/env python
"""bench.py -- training views/sec (rasterizer fwd+bwd) at 1080p on a synthetic 1M-Gaussian scene (BASELINE.json).

One "step" = one view per GPU: rasterize forward (9-channel image) + backward (all parameter gradients), and at
N > 1 the NCCL all-reduce of the per-Gaussian parameter gradients (59 floats/Gaussian) plus the densification
statistics.  Workload: config C3 of BASELINE.md (1 000 000 random Gaussians, 1920x1080, sh_degree 3, seed 2; the
camera moves around a 64-view ring, one new view per step and rank).  `value` is measured with CUDA events with
all inputs resident in HBM; `e2e` goes through the public drop-in API (GaussianRasterizer + autograd) with the
step's host inputs (camera + ground-truth image) copied from pinned memory and the loss read back every step.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config C3] [--dump-outputs DIR]

--impl reference times the UNMODIFIED reference extension (oracle/_ref, built from the original project for sm_90a by
oracle/build_ref.sh) on the same GPU through its own entry points; if that build is absent it times the CPU
restatement of the reference (oracle/) on a bounded sample and says so in `cpu_baseline.kind`.
--dump-outputs DIR writes what the last timed step computed as DIR/<name>.npy (see dump_outputs), so that two builds
can be compared output for output on identical, seeded inputs.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import gof_synth  # noqa: E402


# --------------------------------------------------------------------------------------------------------------
class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region: one streaming
    `nvidia-smi -lms 50` process whose lines are collected by this thread."""

    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.proc = index, [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.proc = None

    def run(self):
        if self.proc is None:
            return
        for line in self.proc.stdout:
            parts = [x.strip() for x in line.strip().split(",")]
            if len(parts) >= 6:
                self.samples.append(parts)

    def stop(self):
        if self.proc is not None:
            time.sleep(0.06)
            self.proc.terminate()
            self.join(timeout=3)
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        sm = sorted(int(s[0]) for s in self.samples if s[0].isdigit())
        mx = [int(s[1]) for s in self.samples if s[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for k, n in enumerate(names) if any(s[2 + k].lower().startswith("active") for s in self.samples)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "samples": len(self.samples)}


def dist_setup(n):
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_DEBUG", "INFO")                       # which algorithm / transport NCCL picked goes into the JSON line
        os.environ.setdefault("NCCL_DEBUG_SUBSYS", "INIT,GRAPH")
        os.environ.setdefault("NCCL_DEBUG_FILE", "/tmp/gof_nccl_%p.log")
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        torch.cuda.set_device(0)
    return rank, world, local


def nccl_info():
    """A few lines of NCCL's own INFO log of this process (which transports / algorithms it set up: NVLS, P2P, rings)."""
    path = os.environ.get("NCCL_DEBUG_FILE", "").replace("%p", str(os.getpid()))
    try:
        keep = []
        for ln in open(path, errors="replace"):
            if any(k in ln for k in ("NVLS", "nvls", "Channel 00", "Connected all", "comm 0x", "via P2P")):
                keep.append(ln.strip()[-160:])
        seen, out = set(), []
        for ln in keep:
            key = ln.split("] ")[-1][:60]
            if key not in seen:
                seen.add(key); out.append(ln)
        return out[:8]
    except Exception:
        return None


def barrier_sync(world):
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def max_over_ranks(x, world, dev):
    if world == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


# --------------------------------------------------------------------------------------------------------------
class Workload:
    """Device-resident Gaussians + per-view camera tensors for one rank."""

    def __init__(self, cfg_name, dev, rank, world, n_views=64):
        self.cfg = dict(gof_synth.CONFIGS[cfg_name])
        self.dev, self.rank, self.world, self.n_views = dev, rank, world, n_views
        W, H = self.cfg["width"], self.cfg["height"]
        cam0 = gof_synth.make_camera(W, H, view=0)
        gs = gof_synth.make_gaussians(self.cfg["P"], self.cfg["seed"], cam0.focal_x)
        self.gs = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
        self.cams = [gof_synth.make_camera(W, H, view=v) for v in range(n_views)]
        self.W, self.H, self.P = W, H, self.cfg["P"]
        g = torch.Generator().manual_seed(1234)
        self.dL_host = torch.randn(9, H, W, generator=g).pin_memory()
        self.dL = self.dL_host.to(dev)
        self.gt_host = torch.rand(3, H, W, generator=g).pin_memory()
        self.bg = torch.zeros(3, device=dev)
        self.subpix = torch.zeros((H, W, 2), dtype=torch.float32, device=dev)
        self.empty = torch.Tensor([])
        self.cam_dev = [(c.world_view_transform.to(dev), c.full_proj_transform.to(dev), c.camera_center.to(dev)) for c in self.cams]
        self.cam_host = [torch.cat([c.world_view_transform.flatten(), c.full_proj_transform.flatten(), c.camera_center]).pin_memory()
                         for c in self.cams]

    def view(self, step):
        return (step * self.world + self.rank) % self.n_views

    def fwd_args(self, v, cam_tensors=None):
        c = self.cams[v]
        vm, pm, cp = cam_tensors if cam_tensors is not None else self.cam_dev[v]
        g = self.gs
        return (self.bg, g["means3D"], self.empty, g["opacities"], g["scales"], g["rotations"], 1.0, self.empty, self.empty,
                vm, pm, c.tanfovx, c.tanfovy, 0.0, self.subpix, self.H, self.W, g["shs"], 3, cp, False, False)


def bwd_args(fa, radii, geom, R, binning, img, grad):
    (bg, means3D, colors, opacity, scales, rotations, sm, cov3D, v2g, vm, pm, tfx, tfy, ks, subpix, H, W, sh, deg, campos,
     pre, dbg) = fa
    return (bg, means3D, radii, colors, scales, rotations, sm, cov3D, v2g, vm, pm, tfx, tfy, ks, subpix, grad, sh, deg,
            campos, geom, R, binning, img, dbg)


DUMP_ROWS = 65536
DUMP_LIMIT = 64 << 20


def dump_outputs(out_dir, arrays):
    """Writes each array as out_dir/<name>.npy, float32 (float64 stays float64).  An array with more than DUMP_ROWS rows is cut
    to a fixed sample of its rows, seeded by the row count, so that arrays of the same length are sampled alike and two
    builds run with the same arguments write comparable files."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    total = 0
    for name, t in arrays.items():
        t = t.detach().reshape(1) if t.dim() == 0 else t.detach()
        n = t.shape[0]
        if n > DUMP_ROWS:
            idx = np.sort(np.random.default_rng(n).choice(n, DUMP_ROWS, replace=False))
            t = t.index_select(0, torch.from_numpy(idx).to(t.device))
        a = t.cpu().numpy()
        a = a.astype(np.float64 if a.dtype == np.float64 else np.float32)
        total += a.nbytes
        assert total <= DUMP_LIMIT, f"--dump-outputs: more than {DUMP_LIMIT >> 20} MB"
        np.save(os.path.join(out_dir, name + ".npy"), a)


def image_rows(img):
    """(C, H, W) -> (H*W, C): rows are pixels, so that dump_outputs samples pixels."""
    return img.permute(1, 2, 0).reshape(-1, img.shape[0])


GRAD_NAMES = ("dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dview2gaussian")


def algorithmic_bytes(P, V, R, N):
    """SURVEY.md section 8(d): bytes one fwd+bwd view must move, and the share of the backward blend kernel."""
    step = 52 * P + 962 * V + 188 * R + 120 * N
    render_bwd = 80 * R + 60 * N + 136 * V      # bwd gather + per-pixel reads + one RMW of the 17 accumulators
    render_fwd = 72 * R + 60 * N
    return step, render_fwd, render_bwd



WORKLOAD_FMT = "{cfg}: {P} Gaussians, {W}x{H}, sh_degree 3, seed {seed}, 64-view ring, 1 view/step/GPU"
E2E_API = ("GaussianRasterizer.forward + autograd backward + L1/normal/depth/distortion loss (torch ops); this step's camera + "
           "ground-truth image prefetched from pinned host memory on a copy stream (double buffer), loss read back through a pinned "
           "slot one step late -- the SAME harness (bench.run_e2e_harness) drives both arms")


def run_e2e_harness(args, wl, world, dev, rasterizer_cls, settings_cls, app=None, bucket=None):
    """End-to-end steps through a package's public drop-in API (`GaussianRasterizer(settings)(...)` + autograd), used
    unchanged for this repo's package and for the reference's own package (--impl reference), so that the two `e2e`
    numbers differ only in the rasterizer.  Input pipeline as a training loop runs it: this step's camera + ground-truth
    image travel from pinned host memory on a copy stream into one of two device buffers while the previous step computes;
    the loss goes back through a pinned slot and is read by the host one step later.  Every copy is issued, and completes,
    inside the timed region.  Returns (milliseconds for args.steps steps, max over ranks; H2D bytes per step).
    N > 1: the per-Gaussian gradients are summed over the ranks every step -- by one NCCL all-reduce of the concatenated .grad
    tensors, or, when the package offers it (`bucket`: this repo's gof_dp.GradBucket, handed to its GaussianRasterizer), by the
    package's own exchange."""
    params = {k: wl.gs[k].detach().clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    h2d = wl.cam_host[0].numel() * 4 + wl.gt_host.numel() * 4
    copy_stream = torch.cuda.Stream()
    cam_buf = [torch.empty(35, device=dev) for _ in range(2)]
    gt_buf = [torch.empty(3, wl.H, wl.W, device=dev) for _ in range(2)]
    ready = [torch.cuda.Event() for _ in range(2)]
    consumed = [torch.cuda.Event() for _ in range(2)]
    loss_pin = [torch.zeros(1).pin_memory() for _ in range(2)]
    loss_done = [torch.cuda.Event() for _ in range(2)]
    losses = []

    def prefetch(step):
        b = step & 1
        v = wl.view(step)
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[b])                      # the step that used this buffer has finished with it
            cam_buf[b].copy_(wl.cam_host[v], non_blocking=True)       # H2D: this step's camera
            gt_buf[b].copy_(wl.gt_host, non_blocking=True)            # H2D: this step's ground-truth image
            ready[b].record(copy_stream)

    def step_e2e(step, last):
        b = step & 1
        if not last:
            prefetch(step + 1)
        main = torch.cuda.current_stream()
        main.wait_event(ready[b])
        c = wl.cams[wl.view(step)]
        rs = settings_cls(
            image_height=wl.H, image_width=wl.W, tanfovx=c.tanfovx, tanfovy=c.tanfovy, kernel_size=0.0, subpixel_offset=wl.subpix,
            bg=wl.bg, scale_modifier=1.0, viewmatrix=cam_buf[b][:16].view(4, 4), projmatrix=cam_buf[b][16:32].view(4, 4), sh_degree=3,
            campos=cam_buf[b][32:35], prefiltered=False, debug=False)
        means2D = torch.zeros_like(params["means3D"], requires_grad=True)
        for p in params.values():
            p.grad = None
        rasterizer = rasterizer_cls(rs) if bucket is None else rasterizer_cls(rs, grad_bucket=bucket)
        img, radii = rasterizer(means3D=params["means3D"], means2D=means2D, opacities=params["opacities"],
                                        shs=params["shs"], scales=params["scales"], rotations=params["rotations"])
        l_rgb = app.loss(img[:3], gt_buf[b], wl.view(step)) if app is not None else (img[:3] - gt_buf[b]).abs().mean()
        loss = l_rgb + 0.05 * (img[3:6] ** 2).mean() + 0.01 * img[6].mean() + 100.0 * img[8].mean()
        if app is not None:
            for p in app.params:
                p.grad = None
            app.emb.grad = None
        loss.backward()
        consumed[b].record(main)
        if world > 1 and bucket is not None:
            if app is not None:
                torch.cat([p.grad.flatten() for p in app.params] + [app.emb.grad[wl.view(step)]], out=bucket.views["extra"])
            bucket.all_reduce()
        elif world > 1:
            flat = torch.cat([params[k].grad.flatten() for k in ("means3D", "shs", "opacities", "scales", "rotations")] +
                             ([p.grad.flatten() for p in app.params] + [app.emb.grad[wl.view(step)]] if app is not None else []))
            dist.all_reduce(flat)
        loss_done[b ^ 1].synchronize()                                # D2H of the PREVIOUS step's loss has landed
        losses.append(float(loss_pin[b ^ 1][0]))
        loss_pin[b].copy_(loss.detach().reshape(1), non_blocking=True)   # D2H: this step's loss
        loss_done[b].record(main)

    def run(first, n):
        for ev in consumed + loss_done:
            ev.record(torch.cuda.current_stream())
        prefetch(first)
        for s in range(n):
            step_e2e(first + s, last=(s == n - 1))
        torch.cuda.synchronize()
        losses.append(float(loss_pin[(first + n - 1) & 1][0]))

    run(0, max(2, args.warmup // 2))
    barrier_sync(world)
    t0 = time.perf_counter()
    run(args.warmup, args.steps)
    barrier_sync(world)
    e2e_ms = max_over_ranks((time.perf_counter() - t0) * 1e3, world, dev)
    assert all(math.isfinite(x) for x in losses), "non-finite loss in the end-to-end loop"
    return e2e_ms, h2d


APPEARANCE_NOTE = "; decoupled appearance on (AppearanceNetwork(67,3) + 64-float view embedding, L1_loss_appearance on the rgb channels)"


def metric_name(wl):
    m = "training views/sec (fwd+bwd) @1080p, %s Gaussians" % ("1M" if wl.P == 1_000_000 else f"{wl.P / 1e6:g}M")
    return m + (", decoupled appearance" if wl.cfg.get("appearance") else "")


class AppearanceStep:
    """Config C4: the appearance part of a training step (train.py:157-159) for either arm -- `which` = "ours" uses
    gof_appearance, "reference" the reference's own AppearanceNetwork class and L1_loss_appearance text (staged, tests/_refpy)."""

    def __init__(self, wl, dev, which):
        import types
        torch.manual_seed(7)
        if which == "ours":
            import gof_appearance
            self.net = gof_appearance.AppearanceNetwork(67, 3).to(dev)
            self.loss = lambda img, gt, idx: gof_appearance.l1_loss_appearance(img, gt, self.net, self.emb[idx])
        else:
            import importlib.util
            import _refpy
            spec = importlib.util.spec_from_file_location("gof_ref_appearance_network", _refpy.staged("scene", "appearance_network.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            self.net = mod.AppearanceNetwork(67, 3).to(dev)
            fn = _refpy.ref_function("train.py", "L1_loss_appearance", {"torch": torch, "l1_loss": _refpy.ref_utils("loss_utils").l1_loss})
            stub = types.SimpleNamespace(get_apperance_embedding=lambda idx: self.emb[idx], appearance_network=self.net)
            self.loss = lambda img, gt, idx: fn(img, gt, stub, idx)
        self.emb = (torch.randn(2048, 64, device=dev) * 1e-4).requires_grad_(True)          # scene/gaussian_model.py:113-116
        self.params = list(self.net.parameters())
        self.numel = sum(p.numel() for p in self.params) + 64
        self.gt = wl.gt_host.to(dev)
        self.dL_rest = wl.dL[3:].contiguous()
        self.ev = []

    def loss_grad(self, color, view, extra_out):
        """d loss / d render (9,H,W) for this view; packs the network / embedding-row gradients into `extra_out` (flat)."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rgb = color[:3].detach().requires_grad_(True)
        loss = self.loss(rgb, self.gt, view)
        grads = torch.autograd.grad(loss, [rgb, self.emb] + self.params)
        off = 0
        for g in grads[2:]:
            extra_out[off:off + g.numel()].copy_(g.reshape(-1)); off += g.numel()
        extra_out[off:off + 64].copy_(grads[1][view])
        dL = torch.cat([grads[0], self.dL_rest], dim=0)
        e1.record()
        self.ev.append((e0, e1))
        return dL

    def timed_ms(self):
        torch.cuda.synchronize()
        ts = [a.elapsed_time(b) for a, b in self.ev[-20:]]
        return sum(ts) / max(len(ts), 1)


# --------------------------------------------------------------------------------------------------------------
def run_ours(args, rank, world, dev):
    from diff_gaussian_rasterization import _C, GaussianRasterizer, GaussianRasterizationSettings
    import gof_dp

    wl = Workload(args.config, dev, rank, world)
    app = AppearanceStep(wl, dev, "ours") if wl.cfg.get("appearance") else None
    # N > 1: the SH gradient travels factored (3 floats of dL_dRGB per Gaussian and view instead of 48 of dL_dsh, expanded on
    # every rank by csrc/sh_views.cu) unless --no-factor-sh asks for the plain 64-float bucket
    factored = world > 1 and not args.no_factor_sh
    bucket = gof_dp.GradBucket(wl.P, 16, dev, extra_sum=app.numel if app else 0, factor_sh=factored)
    exchange_note = None
    exchange_tuning = None
    if world > 1 and args.exchange == "auto":
        # every mode is adopted only after a collective self-test on the live mapping, timed, and the fastest kept (same decision
        # on every rank: the times are max-reduced)
        exchange_tuning = bucket.autotune_exchange()
    elif world > 1 and args.exchange != "nccl":
        try:
            bucket.enable_nvls_exchange() if args.exchange == "nvls" else bucket.enable_peer_exchange()
        except Exception as e:   # noqa: BLE001 -- symmetric on all ranks: e.g. no multicast / no peer access on this box
            exchange_note = f"{args.exchange} unavailable ({type(e).__name__}: {str(e)[:160]}); NCCL all-reduce used"

    def step_device(step):
        v = wl.view(step)
        fa = wl.fwd_args(v)
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
        # (no bucket.zero_(): the backward writes every element of its outputs, zeros included)
        # config C4 (decoupled appearance, train.py:157-159): d loss / d rgb comes from the appearance loss of this view, the
        # network's and the embedding row's gradients join the Gaussian gradients in the bucket
        dL = app.loss_grad(color, v, bucket.views["extra"]) if app else wl.dL
        grads = _C.rasterize_gaussians_backward(*bwd_args(fa, radii, geom, R, binning, img, dL), _out=bucket.views)
        if world > 1:
            bucket.all_reduce()      # gradients (SUM) and this step's densification statistics (SUM | MAX tail) in ONE exchange
        return color, radii, grads

    # ---- kernel-path throughput: inputs resident in HBM, CUDA events, max over ranks --------------------------
    for s in range(args.warmup):
        step_device(s)
    exchange_check = None
    if world > 1:   # untimed: the exchanged bucket equals the combination of the per-rank single-GPU results
        # ONE backward per rank into the exchanged bucket (two runs would differ in the last bits: float atomics in the blend
        # kernel); a factored bucket additionally receives this view's own full dL_dsh (checks only) ...
        fa = wl.fwd_args(wl.view(0))
        R0, _c0, radii0, geom0, bin0, img0 = _C.rasterize_gaussians(*fa)
        bucket.zero_()
        views = dict(bucket.views)
        full = None
        if bucket.factored:
            full = torch.empty(wl.P, 16, 3, device=dev)
            views["_dsh_full"] = full
        _C.rasterize_gaussians_backward(*bwd_args(fa, radii0, geom0, R0, bin0, img0, wl.dL), _out=views)
        names = ("dmeans3D", "dsh", "dopacity", "dscales", "drot", "dens_sum", "dens_max")
        single = {n: (full if (n == "dsh" and bucket.factored) else bucket.views[n].clone()) for n in names}    # ... kept per rank ...
        bucket.all_reduce(means3D=fa[1])                                                                        # ... and exchanged
        err, ok_max, errs = 0.0, True, {}
        for name in names:
            mine = single[name].contiguous()
            parts = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(parts, mine)
            got = bucket.views[name]
            if name == "dens_max":
                ok_max = bool(torch.equal(got, torch.stack(parts).amax(0)))
            else:
                st = torch.stack(parts).double()
                want, mag = st.sum(0), st.abs().sum(0)
                errs[name] = float(((got.double() - want).abs() / (1e-6 * mag + 1e-30)).max())      # <= 1: within 1e-6 of the magnitude sum
                err = max(err, errs[name])
            del parts
        ok_sum = err <= 1.0
        same = torch.tensor([float(bucket.flat[:bucket.n_reduce].double().sum()) + float(bucket.views["dsh"].double().sum())],
                            dtype=torch.float64, device=dev)
        lo, hi = same.clone(), same.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        flag = torch.tensor([1.0 if (ok_sum and ok_max and float(lo) == float(hi)) else 0.0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        exchange_check = "ok" if float(flag.item()) == 1.0 else f"FAILED (sum err {err:.3g} {errs}, max ok {ok_max}, identical on ranks {float(lo) == float(hi)})"
        del single, full, views, geom0, bin0, img0
    barrier_sync(world)
    launches0 = _C.launch_count()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier_sync(world)
    e0.record()
    for s in range(args.steps):
        out = step_device(args.warmup + s)
        last = out if args.dump_outputs and s == args.steps - 1 else None      # only the dumped step's outputs outlive it
        del out
    e1.record()
    barrier_sync(world)
    clocks = sampler.stop()
    ms = max_over_ranks(e0.elapsed_time(e1), world, dev)
    launches = _C.launch_count() - launches0
    if args.dump_outputs and rank == 0:
        color, radii, grads = last
        dump_outputs(args.dump_outputs, {"color": image_rows(color), "radii": radii, **dict(zip(GRAD_NAMES, grads))})
    del last
    # per-kernel durations: a separate short pass with the library's CUDA-event brackets around every launch
    # (kept out of the timed region above: the brackets add host work between launches)
    prof_steps = min(args.steps, 5)
    _C.profile_reset()
    _C.profile_enable(True)
    for s in range(prof_steps):
        step_device(args.warmup + s)
    torch.cuda.synchronize()
    _C.profile_enable(False)
    prof = _C.profile_report()
    N = wl.W * wl.H
    # Workload statistics (SURVEY 8(d)) of ONE named view -- rank 0's first timed view, the same in both arms: visible
    # Gaussians, tile instances and tile-list lengths from one extra, untimed forward.
    stats_view = wl.view(args.warmup)
    R, radii_s, geom_s, bin_s, img_s = (lambda o: (o[0], o[2], o[3], o[4], o[5]))(_C.rasterize_gaussians(*wl.fwd_args(stats_view)))
    V = int((radii_s > 0).sum())
    tile_stats = {}
    try:
        st2 = _C.export_state(wl.P, wl.W, wl.H, R, geom_s, bin_s, img_s, radii_s)
        lens = (st2["ranges"][:, 1] - st2["ranges"][:, 0]).to(torch.float64)
        tile_stats = {"tile_list_mean": float(lens.mean()), "tile_list_max": int(lens.max())}
        del st2
    except Exception:
        tile_stats = {}
    del geom_s, bin_s, img_s

    # ---- end to end through the public API with host inputs (the same harness times the reference arm) --------
    e2e_ms, h2d = run_e2e_harness(args, wl, world, dev, GaussianRasterizer, GaussianRasterizationSettings, app,
                                  bucket=bucket if world > 1 else None)

    # the exchange step alone (N > 1): one all-reduce of the 59-float/Gaussian gradient bucket, CUDA events, max over ranks
    allreduce_ms = None
    if world > 1:
        for _ in range(3):
            bucket.all_reduce()
        barrier_sync(world)
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record()
        for _ in range(10):
            bucket.all_reduce()
        a1.record()
        barrier_sync(world)
        allreduce_ms = max_over_ranks(a0.elapsed_time(a1) / 10, world, dev)

    step_bytes, fwd_bytes, bwd_bytes = algorithmic_bytes(wl.P, V, R, N)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))
    dom = max(("render_bwd", "render_fwd"), key=lambda k: prof.get(k, (0, 0.0))[1])
    dom_cnt, dom_ms = prof.get(dom, (1, 0.0))
    dom_bytes = bwd_bytes if dom == "render_bwd" else fwd_bytes
    achieved = (dom_bytes / (dom_ms / max(dom_cnt, 1) * 1e-3) / 1e9) if dom_ms > 0 else None

    line = {
        "metric": metric_name(wl), "value": world * args.steps / (ms * 1e-3),
        "unit": "views/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD_FMT.format(cfg=args.config, P=wl.P, W=wl.W, H=wl.H, seed=wl.cfg["seed"]) + (APPEARANCE_NOTE if app else ""),
                   "visible": V, "num_rendered": R, "stats_view": stats_view, **tile_stats,
                   "parallelism": f"view-parallel dp{world}" if world > 1 else "single GPU",
                   "l2": "no explicit flush: a step touches >400 MB (> 50 MB L2) and every step renders a new view"},
        "e2e": {"value": world * args.steps / (e2e_ms * 1e-3), "unit": "views/s", "h2d_bytes_per_step": h2d,
                "d2h_bytes_per_step": 4, "ms_per_step": e2e_ms / args.steps,
                "api": E2E_API},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "roofline": {"bound": "hbm", "kernel": dom, "achieved": achieved, "peak": peak,
                     "unit": "GB/s", "frac": (achieved / peak) if achieved else None,
                     "peak_source": "MEASURED_PEAKS.json hbm_gbs (of measured)" if peaks else "H100 SXM data sheet, 3350 GB/s HBM3",
                     "algorithmic_bytes_per_launch": dom_bytes, "launch_ms": dom_ms / max(dom_cnt, 1),
                     "step_algorithmic_bytes": step_bytes,
                     "step_frac": step_bytes / ((ms / args.steps) * 1e-3) / 1e9 / peak},
        "kernels_ms_per_step": {k: v[1] / prof_steps for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])},
    }
    if app:
        line["appearance"] = {"ms_per_step": app.timed_ms(), "params": app.numel,
                              "what": "AppearanceNetwork(67,3) forward + backward on the 1056x1920 crop and L1 (gof_appearance, torch/cuDNN convolutions, "
                                      "TF32 like the reference's default), CUDA events, inside the step"}
    if allreduce_ms is not None:
        per = "11 gradient + 5 statistics f32 per Gaussian reduced, 3 f32 of dL_dRGB per Gaussian and view exchanged as records and expanded to " \
              "dL_dsh (48 f32) on every rank by csrc/sh_views.cu" if bucket.factored else "59 gradient + 5 statistics f32 per Gaussian"
        what = {"p2p": per + "; reduction by the library's kernel over NVLink peer memory (csrc/exchange.cu), records read in place from the "
                       "peers' buckets, two NCCL barriers",
                "nvls": per + "; reduction inside the NVSwitch by the library's multimem kernel (csrc/exchange.cu: multimem.ld_reduce + "
                        "multimem.st on a symmetric-memory bucket), records read in place from the peers' buckets, two NCCL barriers",
                "nccl": per + "; NCCL all-reduce(SUM), all-reduce(MAX)" + (" and all-gather of the records" if bucket.factored else "")}[bucket.exchange]
        line["exchange"] = {"impl": bucket.exchange, "what": what, "bytes": int(bucket.nbytes), "factored_sh": bool(bucket.factored),
                            "ms": allreduce_ms}
        line["exchange_check"] = exchange_check
        if exchange_tuning:
            line["exchange"]["autotune_ms"] = exchange_tuning
        info = nccl_info()
        if info:
            line["exchange"]["nccl_info"] = info
        if exchange_note:
            line["exchange"]["note"] = exchange_note
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        line["cpu_baseline"] = cpu_baseline(args.config, full=False)
    return line


def cpu_baseline(cfg_name, full):
    """The reference algorithm on the host cores (oracle/ port, OpenMP): preprocess + binning + sort on the full
    workload ("the reference's CPU preprocess/sort path"), and one complete fwd+bwd view on a bounded sample."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import numpy as np
    import gof_oracle
    cfg = dict(gof_synth.CONFIGS[cfg_name])
    cam, gs = gof_synth.make_scene(cfg_name, view=1)
    sc = gof_oracle.scene_from_synth(cam, gs)
    t0 = time.perf_counter()
    g = gof_oracle.preprocess(sc)
    t1 = time.perf_counter()
    R, plist, ranges = gof_oracle.bin_tiles(sc.W, sc.H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    t2 = time.perf_counter()
    out = {"kind": "port", "cores": gof_oracle.num_threads(), "host_cpus": os.cpu_count(),
           "preprocess_s": t1 - t0, "bin_sort_s": t2 - t1, "gaussians_per_s": cfg["P"] / (t1 - t0), "instances_per_s": R / max(t2 - t1, 1e-9)}
    # bounded sample for the headline unit: the top `rows` pixel rows of the same view, forward + backward
    rows = cfg["height"] if full else min(cfg["height"], 128)
    H = sc.H
    ranges_s = ranges.copy()
    gx = (sc.W + 15) // 16
    ranges_s[(rows // 16) * gx:] = 0          # tiles below the sample are empty
    t3 = time.perf_counter()
    img, final_T, ncontrib = gof_oracle.render_forward(sc, g, plist, ranges_s)
    dl = np.random.default_rng(0).standard_normal(img.shape).astype(np.float32)
    dl[:, rows:, :] = 0
    d = gof_oracle.render_backward(sc, g, plist, ranges_s, final_T, ncontrib, dl)
    gof_oracle.preprocess_backward(sc, g["radii"], g["clamped"], d["dL_dcolors"], d["dL_dv2g"])
    t4 = time.perf_counter()
    frac = rows / H
    view_s = (t1 - t0) + (t2 - t1) + (t4 - t3) / frac
    out.update({"value": 1.0 / view_s, "unit": "views/s",
                "sample": f"preprocess+bin/sort of the full {cfg_name} view; blend fwd+bwd on the top {rows} of {H} pixel rows "
                          f"({t4 - t3:.1f} s), extrapolated by rows"})
    return out



def _reference_api_shim(ref):
    """GaussianRasterizer / GaussianRasterizationSettings over the reference extension's entry points, with the call structure
    of the reference's own Python wrapper (only used when baseline/_ref/gof_ref_py is absent)."""
    import types
    from typing import NamedTuple

    class Settings(NamedTuple):
        image_height: int
        image_width: int
        tanfovx: float
        tanfovy: float
        kernel_size: float
        subpixel_offset: torch.Tensor
        bg: torch.Tensor
        scale_modifier: float
        viewmatrix: torch.Tensor
        projmatrix: torch.Tensor
        sh_degree: int
        campos: torch.Tensor
        prefiltered: bool
        debug: bool

    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, rs):
            e = torch.Tensor([])
            fa = (rs.bg, means3D, e, opacities, scales, rotations, rs.scale_modifier, e, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                  rs.tanfovy, rs.kernel_size, rs.subpixel_offset, rs.image_height, rs.image_width, sh, rs.sh_degree, rs.campos, False, False)
            R, color, radii, geom, binning, img = ref.rasterize_gaussians(*fa)
            ctx.fa, ctx.R = fa, R
            ctx.save_for_backward(radii, geom, binning, img)
            ctx.mark_non_differentiable(radii)
            return color, radii

        @staticmethod
        def backward(ctx, g, _r=None):
            radii, geom, binning, img = ctx.saved_tensors
            d = ref.rasterize_gaussians_backward(*bwd_args(ctx.fa, radii, geom, ctx.R, binning, img, g))
            return d[3], d[0], d[5], d[2], d[6], d[7], None

    class Rasterizer(torch.nn.Module):
        def __init__(self, rs):
            super().__init__()
            self.rs = rs

        def forward(self, means3D, means2D, opacities, shs, scales, rotations):
            return Fn.apply(means3D, means2D, shs, opacities, scales, rotations, self.rs)

    return types.SimpleNamespace(GaussianRasterizer=Rasterizer, GaussianRasterizationSettings=Settings)


def run_reference(args, rank, world, dev):
    import _util
    ref = _util.load_ref()
    if ref is None:
        cb = cpu_baseline(args.config, full=False)
        return {"metric": "training views/sec (fwd+bwd) @1080p, 1M Gaussians", "impl": "reference", "value": cb["value"],
                "unit": "views/s", "n_gpus": 1, "steps": 1, "warmup": 0, "higher_is_better": True, "scaling": "weak",
                "ms_per_step": 1e3 / cb["value"], "dtype": "f32", "data": "synthetic", "vs_baseline": None,
                "config": {"workload": args.config, "note": "reference CUDA extension not built here; CPU restatement timed"},
                "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "views/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    wl = Workload(args.config, dev, rank, world)
    st = {}
    app = AppearanceStep(wl, dev, "reference") if wl.cfg.get("appearance") else None
    app_flat = torch.zeros(app.numel, device=dev) if app else None

    def step_device(step):
        v = wl.view(step)
        fa = wl.fwd_args(v)
        R, color, radii, geom, binning, img = ref.rasterize_gaussians(*fa)
        dL = app.loss_grad(color, v, app_flat) if app else wl.dL
        grads = ref.rasterize_gaussians_backward(*bwd_args(fa, radii, geom, R, binning, img, dL))
        if world > 1:
            flat = torch.cat([grads[i].flatten() for i in (3, 5, 2, 6, 7)] + ([app_flat] if app else []))
            dist.all_reduce(flat)
        return color, radii, grads

    for s in range(args.warmup):
        step_device(s)
    barrier_sync(world)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(args.steps):
        out = step_device(args.warmup + s)
        last = out if args.dump_outputs and s == args.steps - 1 else None      # only the dumped step's outputs outlive it
        del out
    e1.record()
    barrier_sync(world)
    clocks = sampler.stop()
    ms = max_over_ranks(e0.elapsed_time(e1), world, dev)
    if args.dump_outputs and rank == 0:      # per-rank gradients: the reference arm's exchange sums a copy
        color, radii, grads = last
        dump_outputs(args.dump_outputs, {"color": image_rows(color), "radii": radii, **dict(zip(GRAD_NAMES, grads))})
    del last

    # end to end: the SAME harness as our arm, driving the reference's own public API -- its unmodified Python package
    # (autograd Function + GaussianRasterizer module, staged by baseline/stage_ref.sh) on top of its compiled extension
    import _refpy
    pkg = _refpy.ref_rasterizer_package()
    api_note = "reference's own diff_gaussian_rasterization package (unmodified Python + extension)"
    if pkg is None:   # staged Python missing: same call structure over the extension's entry points
        pkg = _reference_api_shim(ref)
        api_note = "reference extension entry points behind a minimal autograd shim (staged reference Python absent)"
    e2e_ms, h2d = run_e2e_harness(args, wl, world, dev, pkg.GaussianRasterizer, pkg.GaussianRasterizationSettings, app)
    stats_view = wl.view(args.warmup)
    o = ref.rasterize_gaussians(*wl.fwd_args(stats_view))
    st["R"], st["radii"] = o[0], o[2]
    del o
    return {
        "metric": metric_name(wl), "impl": "reference", "value": world * args.steps / (ms * 1e-3),
        "unit": "views/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD_FMT.format(cfg=args.config, P=wl.P, W=wl.W, H=wl.H, seed=wl.cfg["seed"]) + (APPEARANCE_NOTE if app else ""),
                   "visible": int((st["radii"] > 0).sum()), "num_rendered": int(st["R"]), "stats_view": stats_view,
                   "reference": "unmodified diff-gaussian-rasterization of GOF compiled for sm_90a (oracle/build_ref.sh), on the GPU"},
        "cpu_baseline": {"kind": "reference", "cores": 0, "value": world * args.steps / (ms * 1e-3), "unit": "views/s",
                         "sample": "the reference has no CPU path (rasterize_points.cu:75-79 allocates CUDA tensors); this arm "
                                   "runs its own CUDA kernels on the same GPU"},
        "e2e": {"value": world * args.steps / (e2e_ms * 1e-3), "unit": "views/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                "ms_per_step": e2e_ms / args.steps, "api": E2E_API + "; " + api_note},
        "clocks": clocks,
    }


# ==============================================================================================================
# Config C5: opacity-field mesh extraction (BASELINE.json configs[4]): 3 M Gaussians, 27 M query points, 64 views
# ==============================================================================================================
EXTRACT_METRIC = "opacity-field query points/sec (integrate, one 1080p view per step) over 3M Gaussians"
EXTRACT_WORKLOAD_FMT = ("{cfg}: {P} Gaussians, {PN} query points (9 per Gaussian like get_tetra_points + samples in the 3-sigma boxes), "
                        "{W}x{H}, {nv}-view ring, 1 view/step/GPU")


class ExtractWorkload:
    def __init__(self, args, dev, rank, world):
        cfg = dict(gof_synth.CONFIGS[args.config])
        self.P = cfg["P"]
        self.PN = int(args.points or cfg.get("points", 10 * cfg["P"]))
        self.n_views = int(args.views or cfg.get("n_views", 64))
        self.W, self.H, self.dev, self.rank, self.world, self.cfg = cfg["width"], cfg["height"], dev, rank, world, cfg
        cam0 = gof_synth.make_camera(self.W, self.H, view=0)
        gs = gof_synth.make_gaussians(self.P, cfg["seed"], cam0.focal_x)
        self.gs = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
        self.cams = [gof_synth.make_camera(self.W, self.H, view=v, n_views=self.n_views) for v in range(self.n_views)]
        self.points, self.pscale = gof_synth.make_tetra_points(self.gs, self.PN, cfg["seed"] + 100, dev)
        self.bg = torch.zeros(3, device=dev)
        self.subpix = torch.zeros((self.H, self.W, 2), dtype=torch.float32, device=dev)
        self.cam_host = [torch.cat([c.world_view_transform.flatten(), c.full_proj_transform.flatten(), c.camera_center]).pin_memory()
                         for c in self.cams]

    def view(self, step):
        return (step * self.world + self.rank) % self.n_views

    def settings(self, cls, v, cam_buf=None):
        c = self.cams[v]
        vm = c.world_view_transform.to(self.dev) if cam_buf is None else cam_buf[:16].view(4, 4)
        pm = c.full_proj_transform.to(self.dev) if cam_buf is None else cam_buf[16:32].view(4, 4)
        cp = c.camera_center.to(self.dev) if cam_buf is None else cam_buf[32:35]
        return cls(image_height=self.H, image_width=self.W, tanfovx=c.tanfovx, tanfovy=c.tanfovy, kernel_size=0.0,
                   subpixel_offset=self.subpix, bg=self.bg, scale_modifier=1.0, viewmatrix=vm, projmatrix=pm, sh_degree=3, campos=cp,
                   prefiltered=False, debug=False)


def extract_e2e(args, wl, world, dev, rasterizer_cls, settings_cls):
    """End to end through a package's public API: GaussianRasterizer(settings).integrate(points3D=...) for this step's view,
    camera copied from pinned host memory every step, the smallest integrated alpha read back (4 bytes).  The query points
    are the step-invariant operand of an extraction pass (extract_mesh.py evaluates the same points for all views) and
    stay resident.  Same function for both arms."""
    g = wl.gs
    cam_buf = torch.empty(35, device=dev)
    res_pin = torch.zeros(1).pin_memory()
    m2d = torch.zeros_like(g["means3D"])

    def step(i):
        v = wl.view(i)
        cam_buf.copy_(wl.cam_host[v], non_blocking=True)
        rs = wl.settings(settings_cls, v, cam_buf)
        with torch.no_grad():
            _img, alpha, _col, _rad = rasterizer_cls(rs).integrate(points3D=wl.points, means3D=g["means3D"], means2D=m2d,
                                                                   opacities=g["opacities"], shs=g["shs"], scales=g["scales"],
                                                                   rotations=g["rotations"])
        res_pin.copy_(alpha.min().reshape(1), non_blocking=True)
        torch.cuda.synchronize()
        return float(res_pin[0])

    for i in range(max(2, args.warmup // 2)):
        step(i)
    barrier_sync(world)
    t0 = time.perf_counter()
    vals = [step(args.warmup + i) for i in range(args.steps)]
    barrier_sync(world)
    ms = max_over_ranks((time.perf_counter() - t0) * 1e3, world, dev)
    assert all(math.isfinite(x) for x in vals)
    return ms


def run_extract_ours(args, rank, world, dev):
    from diff_gaussian_rasterization import _C, GaussianRasterizer, GaussianRasterizationSettings
    import gof_extract
    wl = ExtractWorkload(args, dev, rank, world)
    g = wl.gs
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3,
                                      lambda v: wl.settings(GaussianRasterizationSettings, v))
    # Gaussian side of this rank's views, once (SURVEY 8(f) rank 3): timed separately
    my_views = sorted({wl.view(s) for s in range(args.warmup + args.steps)})
    torch.cuda.synchronize()
    p0 = time.perf_counter()
    for v in my_views:
        ci.prepare(v)
    torch.cuda.synchronize()
    prepare_ms = (time.perf_counter() - p0) * 1e3 / max(len(my_views), 1)

    def step_device(s):
        return ci(wl.points, wl.view(s))

    for s in range(args.warmup):
        step_device(s)
    barrier_sync(world)
    launches0 = _C.launch_count()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier_sync(world)
    e0.record()
    for s in range(args.steps):
        out = step_device(args.warmup + s)
        last = out if args.dump_outputs and s == args.steps - 1 else None      # only the dumped step's outputs outlive it
        del out
    e1.record()
    barrier_sync(world)
    clocks = sampler.stop()
    ms = max_over_ranks(e0.elapsed_time(e1), world, dev)
    launches = _C.launch_count() - launches0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, dict(zip(("alpha_integrated", "color_integrated"), last)))
    del last
    prof_steps = min(args.steps, 3)
    _C.profile_reset(); _C.profile_enable(True)
    for s in range(prof_steps):
        step_device(args.warmup + s)
    torch.cuda.synchronize(); _C.profile_enable(False)
    prof = _C.profile_report()

    # workload statistics of rank 0's first timed view
    sv = wl.view(args.warmup)
    _vw, rs_sv, cache_sv = ci.prepare(sv)
    img_sv, _a, _c = _C.integrate_points_cached(cache_sv, wl.bg, wl.points, rs_sv.viewmatrix, rs_sv.tanfovx, rs_sv.tanfovy)
    PNv = int(img_sv[8].sum().item())
    Rg, Vg = int(cache_sv.num_rendered), int((cache_sv.radii > 0).sum())
    N = wl.W * wl.H
    del img_sv

    e2e_ms = extract_e2e(args, wl, world, dev, GaussianRasterizer, GaussianRasterizationSettings)

    # the whole extraction once (untimed against the headline): evaluate_alpha on all vertices, marching tetrahedra, 8 bisection steps
    pipeline = None
    if not args.no_pipeline:
        T = int(wl.PN * wl.cfg.get("tets_per_point", 6.5)) if not args.tets else int(args.tets)
        tets = gof_synth.make_local_tets(wl.PN, T, wl.cfg["seed"] + 200, dev)
        views = list(range(wl.n_views))
        tm = {}
        torch.cuda.synchronize(); barrier_sync(world)
        t0 = time.perf_counter()
        out = gof_extract.extract_level_set(wl.points, wl.pscale, tets, views, ci, n_binary_steps=8,
                                            group=None if world == 1 else dist.group.WORLD, timings=tm)
        torch.cuda.synchronize(); barrier_sync(world)
        total_s = max_over_ranks(time.perf_counter() - t0, world, dev)
        pipeline = {"tets": T, "faces": int(out["faces"].shape[0]), "mesh_vertices": int(out["vertices"].shape[0]), "views": wl.n_views,
                    "total_s": total_s, **{k: round(v, 4) for k, v in tm.items()},
                    "tets_per_s": T / max(tm.get("marching_tetrahedra_s", 1e-9), 1e-9),
                    "cached_view_bytes": int(ci.cached_bytes),
                    "what": "gof_extract.extract_level_set: evaluate_alpha on the tetrahedra vertices (view-sharded, one all_reduce(MIN)), "
                            "marching tetrahedra (tet-chunk sharded), 8 bisection steps, Gaussian side of every view cached"}
        del tets, out

    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))
    # SURVEY 8(d), extraction: the query kernel gathers 72 B per tile instance (records of the tile lists), reads 16 B and writes
    # 16 B per projected point, writes the 9-channel image; the point side in front of it reads 12 B/point and writes 24 B/projected point
    k_bytes = 72 * Rg + 32 * PNv + 36 * N
    view_bytes = k_bytes + 12 * wl.PN + 24 * PNv
    cnt, k_ms = prof.get("integrate", (1, 0.0))
    achieved = (k_bytes / (k_ms / max(cnt, 1) * 1e-3) / 1e9) if k_ms > 0 else None
    line = {
        "metric": EXTRACT_METRIC, "value": world * args.steps * wl.PN / (ms * 1e-3), "unit": "points/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": EXTRACT_WORKLOAD_FMT.format(cfg=args.config, P=wl.P, PN=wl.PN, W=wl.W, H=wl.H, nv=wl.n_views),
                   "stats_view": sv, "visible": Vg, "num_rendered": Rg, "points_projected": PNv,
                   "parallelism": f"view-parallel dp{world}" if world > 1 else "single GPU",
                   "gaussian_side": f"prepared once per view and cached ({prepare_ms:.2f} ms/view, outside the timed steps; the e2e "
                                    f"number below repeats it every step like the reference)",
                   "l2": "no explicit flush: a step streams the 27 M points (> 0.5 GB, > 50 MB L2) and every step is a new view"},
        "e2e": {"value": world * args.steps * wl.PN / (e2e_ms * 1e-3), "unit": "points/s", "h2d_bytes_per_step": 35 * 4,
                "d2h_bytes_per_step": 4, "ms_per_step": e2e_ms / args.steps,
                "api": "GaussianRasterizer(settings).integrate(points3D=...) incl. the Gaussian side; camera from pinned host memory every "
                       "step, min(alpha_integrated) read back; query points resident (one extraction pass evaluates the same points for all views)"},
        "gpu_launches": int(launches), "clocks": clocks,
        "roofline": {"bound": "hbm", "kernel": "integrate", "achieved": achieved, "peak": peak, "unit": "GB/s",
                     "frac": (achieved / peak) if achieved else None, "traffic": None,
                     "peak_source": "MEASURED_PEAKS.json hbm_gbs (of measured)" if peaks else "H100 SXM data sheet, 3350 GB/s HBM3",
                     "algorithmic_bytes_per_launch": k_bytes, "launch_ms": k_ms / max(cnt, 1), "step_algorithmic_bytes": view_bytes,
                     "step_frac": view_bytes / ((ms / args.steps) * 1e-3) / 1e9 / peak},
        "kernels_ms_per_step": {k: v[1] / prof_steps for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])},
    }
    if pipeline is not None:
        line["extraction"] = pipeline
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        line["cpu_baseline"] = cpu_baseline_extract(wl)
    return line


def cpu_baseline_extract(wl):
    """The reference's query algorithm on the host cores (oracle/ port, OpenMP) for one view: Gaussian side of the full view,
    point side on a bounded sample -- the top 64 pixel rows' tiles and the query points that project into them."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ctypes
    import numpy as np
    import gof_oracle
    gs_cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in wl.gs.items()}
    cam = wl.cams[1]
    sc = gof_oracle.scene_from_synth(cam, gs_cpu)
    t0 = time.perf_counter()
    g = gof_oracle.preprocess(sc)
    R, plist, ranges = gof_oracle.bin_tiles(sc.W, sc.H, g["radii"], g["means2D"], g["depths"], g["tiles_touched"])
    t1 = time.perf_counter()
    rows = 64
    gx = (sc.W + 15) // 16
    ranges_s = np.ascontiguousarray(ranges, np.uint32).copy()
    ranges_s[(rows // 16) * gx:] = 0
    # points that project into the kept rows (same projection as forward.cu:756-765, float64 here: only used to pick the sample)
    pts = wl.points.cpu().numpy().astype(np.float64)
    vm = cam.world_view_transform.numpy().astype(np.float64)
    pv = pts @ vm[:3, :3] + vm[3, :3]
    fx, fy = sc.W / (2 * cam.tanfovx), sc.H / (2 * cam.tanfovy)
    x = fx * pv[:, 0] / (pv[:, 2] + 1e-7) + sc.W / 2.0
    y = fy * pv[:, 1] / (pv[:, 2] + 1e-7) + sc.H / 2.0
    proj = (pv[:, 2] > 0.2) & (x >= 0) & (x < sc.W) & (y >= 0) & (y < sc.H)
    keep = proj & (y < rows)
    sample = np.ascontiguousarray(pts[keep][:2_000_000], np.float32)
    PNs = int(sample.shape[0])
    out = np.zeros((9, sc.H, sc.W), np.float32)
    final_T = np.zeros((sc.H, sc.W), np.float32)
    n_contrib = np.zeros((sc.H, sc.W), np.uint32)
    alpha_int = np.ones(PNs, np.float32)
    color_int = np.zeros((PNs, 3), np.float32)
    _p = gof_oracle._p
    t2 = time.perf_counter()
    gof_oracle._lib.oracle_integrate(sc.W, sc.H, ctypes.c_float(sc.tan_fovx), ctypes.c_float(sc.tan_fovy), _p(sc.arr["viewmatrix"]), PNs,
                                     _p(sample), _p(ranges_s), _p(np.ascontiguousarray(plist, np.uint32)),
                                     _p(np.ascontiguousarray(g["rgb"], np.float32)), _p(np.ascontiguousarray(g["view2gaussian"], np.float32)),
                                     _p(np.ascontiguousarray(g["conic_opacity"], np.float32)), _p(sc.arr["background"]), _p(out), _p(final_T),
                                     _p(n_contrib), _p(alpha_int), _p(color_int))
    t3 = time.perf_counter()
    n_proj = int(proj.sum())
    view_s = (t1 - t0) + (t3 - t2) * (n_proj / max(PNs, 1))
    return {"kind": "port", "cores": gof_oracle.num_threads(), "host_cpus": os.cpu_count(), "gaussian_side_s": t1 - t0,
            "sample_query_s": t3 - t2, "value": wl.PN / view_s, "unit": "points/s",
            "sample": f"Gaussian side of the full view; point side on the {PNs} query points that project into the top {rows} pixel rows "
                      f"(their tiles only), extrapolated to the {n_proj} projected points of the view"}


def run_extract_reference(args, rank, world, dev):
    import _util
    import _refpy
    ref = _util.load_ref()
    pkg = _refpy.ref_rasterizer_package()
    if ref is None or pkg is None:
        return {"impl": "reference", "unavailable": "reference extension / staged Python not built here (needs the original project at build time)"}
    wl = ExtractWorkload(args, dev, rank, world)
    g = wl.gs
    e = torch.Tensor([])

    def step_device(s):
        c = wl.cams[wl.view(s)]
        vm, pm, cp = (c.world_view_transform.to(dev), c.full_proj_transform.to(dev), c.camera_center.to(dev))
        return ref.integrate_gaussians_to_points(wl.bg, wl.points, g["means3D"], e, g["opacities"], g["scales"], g["rotations"], 1.0, e, e, vm,
                                                 pm, c.tanfovx, c.tanfovy, 0.0, wl.subpix, wl.H, wl.W, g["shs"], 3, cp, False, False)

    for s in range(args.warmup):
        step_device(s)
    barrier_sync(world)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(args.steps):
        out = step_device(args.warmup + s)
        last = out if args.dump_outputs and s == args.steps - 1 else None      # only the dumped step's outputs outlive it
        del out
    e1.record()
    barrier_sync(world)
    clocks = sampler.stop()
    ms = max_over_ranks(e0.elapsed_time(e1), world, dev)
    if args.dump_outputs and rank == 0:      # (num_rendered, out_color, alpha_integrated, color_integrated, ...)
        dump_outputs(args.dump_outputs, {"alpha_integrated": last[2], "color_integrated": last[3]})
    del last
    sv = wl.view(args.warmup)
    o = step_device(args.warmup)
    Rg, PNv, Vg = int(o[0]), int(o[1][8].sum().item()), int((o[4] > 0).sum())
    del o
    e2e_ms = extract_e2e(args, wl, world, dev, pkg.GaussianRasterizer, pkg.GaussianRasterizationSettings)
    val = world * args.steps * wl.PN / (ms * 1e-3)
    return {
        "metric": EXTRACT_METRIC, "impl": "reference", "value": val, "unit": "points/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": EXTRACT_WORKLOAD_FMT.format(cfg=args.config, P=wl.P, PN=wl.PN, W=wl.W, H=wl.H, nv=wl.n_views),
                   "stats_view": sv, "visible": Vg, "num_rendered": Rg, "points_projected": PNv,
                   "reference": "unmodified diff-gaussian-rasterization of GOF compiled for sm_90a (oracle/build_ref.sh), on the GPU"},
        "cpu_baseline": {"kind": "reference", "cores": 0, "value": val, "unit": "points/s",
                         "sample": "the reference has no CPU path; this arm runs its own CUDA kernels on the same GPU"},
        "e2e": {"value": world * args.steps * wl.PN / (e2e_ms * 1e-3), "unit": "points/s", "h2d_bytes_per_step": 35 * 4,
                "d2h_bytes_per_step": 4, "ms_per_step": e2e_ms / args.steps,
                "api": "reference's own GaussianRasterizer(settings).integrate; same harness as our arm (bench.extract_e2e)"},
        "clocks": clocks,
    }


# ==============================================================================================================
# --mode train_step: one whole training iteration around the rasterizer (SURVEY 8(f) ranks 1-2 next to the hot path)
# ==============================================================================================================
TRAIN_METRIC = "training iterations/sec (activations + render + loss + backward + Adam) @1080p"
_LRS = {"_xyz": 1.6e-4, "_features_dc": 2.5e-3, "_features_rest": 2.5e-3 / 20, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001}
_LAMBDAS = (0.2, 0.05, 100.0)      # lambda_dssim, lambda_depth_normal, lambda_distortion (arguments/__init__.py)


def _raw_params(wl, dev):
    g = wl.gs
    return {"_xyz": g["means3D"].clone(), "_scaling": torch.log(g["scales"]), "_rotation": g["rotations"].clone(),
            "_opacity": torch.logit(g["opacities"].clamp(1e-4, 1 - 1e-4)), "_features_dc": g["shs"][:, :1].contiguous(),
            "_features_rest": g["shs"][:, 1:].contiguous()}


def run_train_step(args, rank, world, dev):
    """ours:       gof_params.activate -> GaussianRasterizer -> gof_loss.view_loss -> backward -> [all-reduce] -> gof_params.adam_step
    reference:  torch activations (scene/gaussian_model.py:152-194) -> the reference's rasterizer package -> the reference's own
                l1_loss / ssim / depth_to_normal as train.py:151-188 combines them -> backward -> [all-reduce] -> torch.optim.Adam(eps=1e-15)
    Host inputs per step (camera + ground-truth image) come from pinned memory, the loss is read back: every step is end to end."""
    import types
    import torch.nn.functional as F
    ours = args.impl == "ours"
    wl = Workload(args.config, dev, rank, world)
    filt = (torch.rand(wl.P, 1, generator=torch.Generator().manual_seed(5)) * 0.002).to(dev)
    raw = {k: v.to(dev).requires_grad_(True) for k, v in _raw_params(wl, dev).items()}
    cam_buf = torch.empty(35, device=dev)
    gt_buf = torch.empty(3, wl.H, wl.W, device=dev)
    loss_pin = torch.zeros(1).pin_memory()
    if ours:
        import gof_loss
        import gof_params
        from diff_gaussian_rasterization import GaussianRasterizer, GaussianRasterizationSettings
        state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in raw.items()}
    else:
        import _refpy
        pkg = _refpy.ref_rasterizer_package()
        lu, du = _refpy.ref_utils("loss_utils"), _refpy.ref_utils("depth_utils")
        if pkg is None or lu is None or du is None:
            return {"impl": "reference", "unavailable": "reference extension / staged Python not built here (needs the original project at build time)"}
        GaussianRasterizer, GaussianRasterizationSettings = pkg.GaussianRasterizer, pkg.GaussianRasterizationSettings
        opt = torch.optim.Adam([{"params": [v], "lr": _LRS[k]} for k, v in raw.items()], lr=0.0, eps=1e-15)
    it = [0]

    def step(s):
        it[0] += 1
        v = wl.view(s)
        c = wl.cams[v]
        cam_buf.copy_(wl.cam_host[v], non_blocking=True)
        gt_buf.copy_(wl.gt_host, non_blocking=True)
        wvt = cam_buf[:16].view(4, 4)
        rs = GaussianRasterizationSettings(image_height=wl.H, image_width=wl.W, tanfovx=c.tanfovx, tanfovy=c.tanfovy, kernel_size=0.0,
                                           subpixel_offset=wl.subpix, bg=wl.bg, scale_modifier=1.0, viewmatrix=wvt,
                                           projmatrix=cam_buf[16:32].view(4, 4), sh_degree=3, campos=cam_buf[32:35], prefiltered=False, debug=False)
        means2D = torch.zeros_like(raw["_xyz"], requires_grad=True)
        if ours:
            for p in raw.values():
                p.grad = None
            scales, rots, ops, shs = gof_params.activate(raw["_scaling"], raw["_rotation"], raw["_opacity"], filt, raw["_features_dc"], raw["_features_rest"])
        else:
            opt.zero_grad(set_to_none=True)
            sc = torch.exp(raw["_scaling"])                                   # get_scaling_with_3D_filter, :157-163
            s2 = torch.square(sc)
            scales = torch.sqrt(s2 + torch.square(filt))
            coef = torch.sqrt(s2.prod(dim=1) / (s2 + torch.square(filt)).prod(dim=1))      # get_opacity_with_3D_filter, :173-185
            ops = torch.sigmoid(raw["_opacity"]) * coef[..., None]
            rots = F.normalize(raw["_rotation"])                              # get_rotation, :165-167
            shs = torch.cat((raw["_features_dc"], raw["_features_rest"]), dim=1)   # get_features, :187-191
        img, radii = GaussianRasterizer(rs)(means3D=raw["_xyz"], means2D=means2D, opacities=ops, shs=shs, scales=scales, rotations=rots)
        if ours:
            loss, _terms = gof_loss.view_loss(img, gt_buf, c.world_view_transform, c.tanfovx, c.tanfovy, *_LAMBDAS, rotation=wl.rot9[v])
        else:
            view = types.SimpleNamespace(world_view_transform=wvt, image_width=wl.W, image_height=wl.H, FoVx=2 * math.atan(c.tanfovx),
                                         FoVy=2 * math.atan(c.tanfovy))
            image = img[:3]
            rgb_loss = (1.0 - _LAMBDAS[0]) * lu.l1_loss(image, gt_buf) + _LAMBDAS[0] * (1.0 - lu.ssim(image, gt_buf))      # train.py:156-161
            depth_normal, _ = du.depth_to_normal(view, img[6][None])                                                         # :170-186
            depth_normal = depth_normal.permute(2, 0, 1)
            render_normal = F.normalize(img[3:6], p=2, dim=0)
            c2w = (wvt.T).inverse()
            rnw = (c2w[:3, :3] @ render_normal.reshape(3, -1)).reshape(3, *render_normal.shape[1:])
            loss = rgb_loss + (1 - (rnw * depth_normal).sum(dim=0)).mean() * _LAMBDAS[1] + img[8].mean() * _LAMBDAS[2]
        loss.backward()
        if world > 1:
            flat = torch.cat([p.grad.flatten() for p in raw.values()])
            dist.all_reduce(flat)
            off = 0
            for p in raw.values():
                p.grad = flat[off:off + p.numel()].view_as(p); off += p.numel()
        if ours:
            with torch.no_grad():
                for k, p in raw.items():
                    gof_params.adam_step(p.data, state[k][0], state[k][1], p.grad.contiguous(), _LRS[k], it[0])
        else:
            opt.step()
        loss_pin.copy_(loss.detach().reshape(1), non_blocking=True)
        return loss_pin

    if ours:
        import gof_loss as _gl
        wl.rot9 = [_gl.camera_rotation(c.world_view_transform) for c in wl.cams]
    for s in range(args.warmup):
        step(s)
    barrier_sync(world)
    launches0 = 0
    if ours:
        from diff_gaussian_rasterization import _C
        launches0 = _C.launch_count()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier_sync(world)
    t0 = time.perf_counter()
    e0.record()
    for s in range(args.steps):
        step(args.warmup + s)
    e1.record()
    barrier_sync(world)
    wall_ms = max_over_ranks((time.perf_counter() - t0) * 1e3, world, dev)
    clocks = sampler.stop()
    ms = max_over_ranks(e0.elapsed_time(e1), world, dev)
    final = float(loss_pin[0])
    if args.dump_outputs and rank == 0:      # the parameters after the last step's update, and that step's loss
        dump_outputs(args.dump_outputs, {"loss": loss_pin.clone(), **{k.lstrip("_"): v for k, v in raw.items()}})
    assert math.isfinite(final)
    h2d = 35 * 4 + wl.gt_host.numel() * 4
    line = {"metric": TRAIN_METRIC, "value": world * args.steps / (ms * 1e-3), "unit": "iterations/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic", "mode": "train_step",
            "config": {"workload": WORKLOAD_FMT.format(cfg=args.config, P=wl.P, W=wl.W, H=wl.H, seed=wl.cfg["seed"]),
                       "iteration": ("gof_params.activate -> GaussianRasterizer -> gof_loss.view_loss -> backward -> gof_params.adam_step" if ours else
                                     "torch activations -> reference rasterizer package -> reference l1_loss/ssim/depth_to_normal (train.py:151-188) "
                                     "-> backward -> torch.optim.Adam(eps=1e-15)"),
                       "final_loss": final},
            "e2e": {"value": world * args.steps / (wall_ms * 1e-3), "unit": "iterations/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                    "ms_per_step": wall_ms / args.steps, "api": "the same loop on the host clock: camera + ground-truth image from pinned memory and the loss read back every step"},
            "clocks": clocks}
    if not ours:
        line["impl"] = "reference"
        line["cpu_baseline"] = {"kind": "reference", "cores": 0, "value": line["value"], "unit": "iterations/s",
                                "sample": "the reference has no CPU path; this arm runs its own CUDA kernels + torch on the same GPU"}
    else:
        line["gpu_launches"] = int(_C.launch_count() - launches0)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=None, help="timed steps (default 50; 16 for the extraction config C5)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="C3", choices=sorted(gof_synth.CONFIGS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--mode", default="raster", choices=["raster", "train_step"],
                    help="raster (default): the rasterizer fwd+bwd step of BASELINE.json; train_step: a whole training iteration around it")
    ap.add_argument("--points", type=int, default=0, help="C5: number of query points (default: the config's 27 M)")
    ap.add_argument("--views", type=int, default=0, help="C5: number of views on the ring (default 64)")
    ap.add_argument("--tets", type=int, default=0, help="C5: number of tetrahedra of the pipeline run (default 6.5 per point)")
    ap.add_argument("--no-pipeline", action="store_true", help="C5: skip the one full extraction run (evaluate_alpha + marching tets + bisection)")
    ap.add_argument("--exchange", default="auto", choices=["auto", "nvls", "p2p", "nccl"],
                    help="N>1 gradient exchange: the library's multimem kernel through the NVSwitch (nvls), its NVLink peer-memory kernel "
                         "(p2p), NCCL's all-reduce (nccl), or auto = nvls, else p2p, else nccl -- each mode is adopted only after a "
                         "collective self-test on the live mapping")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed as DIR/<name>.npy (float32, a seeded sample of "
                         "rows where an output is larger; at most 64 MB in all)")
    ap.add_argument("--no-factor-sh", action="store_true", help="N>1: exchange the full dL_dsh (64 floats per Gaussian in the bucket) instead of "
                                                               "the per-view dL_dRGB records (16 reduced + 3 per view)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the rasterizer has no CPU path")
    # keep stdout clean for the ONE JSON line (NCCL prints its version banner to stdout): everything else -> stderr
    sys.stdout.flush()
    saved_stdout = os.dup(1)
    os.dup2(2, 1)
    rank, world, local = dist_setup(args.gpus)
    dev = torch.device("cuda", local if world > 1 else 0)
    extract = "points" in gof_synth.CONFIGS[args.config]
    if args.steps is None:
        args.steps = 16 if extract else 50          # a C5 step is a 27 M-point query: keep the default run within minutes
    if args.mode == "train_step" and not extract:
        line = run_train_step(args, rank, world, dev)
    elif extract:
        line = run_extract_ours(args, rank, world, dev) if args.impl == "ours" else run_extract_reference(args, rank, world, dev)
    else:
        line = run_ours(args, rank, world, dev) if args.impl == "ours" else run_reference(args, rank, world, dev)
    sys.stdout.flush()
    os.dup2(saved_stdout, 1)
    if rank == 0:
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
