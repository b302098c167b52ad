"""View-parallel helpers: one process per GPU, every rank holds all Gaussians and rasterizes a different view;
per-Gaussian parameter gradients are summed with ONE all-reduce of a flat buffer (SURVEY.md section 8(e)).

The reference is single-GPU (its only multi-GPU use is one training job per GPU, scripts/run_mipnerf360.py:20-41),
so this module is new, not a port.  It uses torch.distributed (NCCL on GPUs, gloo in the CPU tests); the
rasterizer backward writes its outputs directly into views of the flat buffer (`_out=` of
`_C.rasterize_gaussians_backward`), so there is no pack/copy step before the collective.

Exchange step: `GradBucket.all_reduce()` is NCCL's all-reduce (SUM over the gradients and the summed statistics, MAX over
the statistics' MAX tail).  `GradBucket.enable_peer_exchange()` switches it to the library's own kernel over NVLink peer
memory (csrc/exchange.cu: every rank maps every rank's bucket through CUDA IPC, reduces its 1/N slice from all of them in rank
order and stores it into all of them), bracketed by two NCCL barriers.  `GradBucket.enable_nvls_exchange()` moves the bucket
into a torch symmetric-memory allocation (plumbing: it binds every rank's copy to one NVSwitch multicast object) and reduces
it with the library's multimem kernel: the switch adds the ranks' copies (multimem.ld_reduce) and broadcasts the result
(multimem.st) -- one bucket of NVLink traffic per GPU and direction instead of 2 (N-1)/N.

Factored SH gradient (`GradBucket(..., factor_sh=True)`): 48 of the 59 gradient floats per Gaussian are dL_dsh, and ONE view's
dL_dsh is an outer product w(dir(mean, camera)) (x) dL_dRGB (backward.cu:45-139).  Every rank holds all means, so the ranks only
need each other's clamp-masked dL_dRGB -- 3 floats per Gaussian and view -- and each expands sum_v w(dir_v) (x) rgb_v itself
(csrc/sh_views.cu), in rank order, bit-identical to adding the views' dL_dsh tensors.  The reduced part of the bucket shrinks from
64 to 16 floats per Gaussian; the per-view records sit behind it ([world] x (64-float header + three colour planes)) and are read in place over
NVLink by the expansion kernel (peer-memory / NVLS exchange) or all-gathered (NCCL / gloo).

The bucket also carries this view's densification statistics (written by the rasterizer backward itself, see
gof_backward_out_t.dens_sum / dens_max): `dens_sum` (P,3) = (|dL_dmean2D.xy|, |dL_dmean2D.z|, visible) reduced with SUM and `dens_max`
(P,2) = (|dL_dmean2D.z|, radius) reduced with MAX -- what GaussianModel.add_densification_stats and train.py:255 accumulate.
"""
import ctypes

import torch
import torch.distributed as dist

from diff_gaussian_rasterization import _C

# per-Gaussian parameter gradients that must be reduced across views: 3 + 48 + 1 + 3 + 4 = 59 floats
_FIELDS = (("dmeans3D", (3,)), ("dsh", None), ("dopacity", (1,)), ("dscales", (3,)), ("drot", (4,)))
_STAT_FIELDS = (("dens_sum", (3,)), ("dens_max", (2,)))       # SUM region ends where dens_max starts
SH_SLOT_HEADER = 64                                           # floats in front of a view record's rgb (include/gof_rasterizer.h)


class GradBucket:
    """Flat fp32 buffer [sum of fields] with one contiguous, correctly shaped view per gradient tensor."""

    def __init__(self, P, M, device, dtype=torch.float32, with_stats=True, extra_sum=0, factor_sh=False, group=None):
        """`extra_sum`: additional floats summed with the gradients (view "extra": e.g. the appearance network's gradients).
        `factor_sh`: exchange dL_dRGB per view instead of dL_dsh (module docstring); needs an initialised process group (the
        number of view records is its world size).  views["dsh"] is then a local tensor that all_reduce() fills, and the
        rasterizer backward is handed views["dsh_rgb"] / views["sh_hdr"] (it finds them in `_out=bucket.views`)."""
        self.P, self.M = int(P), int(M)
        self.factored = bool(factor_sh)
        if self.factored:
            if not (dist.is_available() and dist.is_initialized()):
                raise RuntimeError("GradBucket(factor_sh=True) needs an initialised process group")
            self._n_views, self._view = dist.get_world_size(group), dist.get_rank(group)
            if self._n_views > 16:
                raise RuntimeError("GradBucket(factor_sh=True): at most 16 ranks (csrc/sh_views.cu)")
        shapes = {}
        for name, tail in _FIELDS:
            if name == "dsh" and self.factored:
                continue
            shapes[name] = (self.P, self.M, 3) if name == "dsh" else (self.P,) + tail
        if extra_sum:
            shapes["extra"] = (int(extra_sum),)
        if with_stats:
            for name, tail in _STAT_FIELDS:
                shapes[name] = (self.P,) + tail
        self._offsets, off = _C._layout(shapes)
        self.n_reduce = off                                                    # floats [0, n_reduce) are reduced over the ranks:
        self.n_sum = self._offsets["dens_max"][0] if with_stats else off      #   [0, n_sum) SUM, [n_sum, n_reduce) MAX
        self._slot = 0
        self.dsh = None
        if self.factored:    # [n_reduce, numel): one record per view = SH_SLOT_HEADER floats (camera centre, degree) + rgb [P,3]
            self._plane = _C._sh_plane(self.P)              # the record's three colour planes
            self._slot = SH_SLOT_HEADER + 3 * self._plane
            off += self._n_views * self._slot
            self.dsh = torch.zeros(self.P, self.M, 3, dtype=dtype, device=device)
        self.numel = off
        self.flat = torch.zeros(max(self.numel, 64), dtype=dtype, device=device)
        self.views = self._make_views()
        self._symm = None        # torch symmetric-memory handle (NVLS exchange)

        self._peer_ptrs = None   # addresses (this process) of every rank's bucket, index = rank; own cudaMalloc at [rank]
        self._own_ptr, self._mapped = None, []
        self._sync = None
        self.exchange = "nccl"

    def _make_views(self):
        views = _C._views(self.flat, self._offsets)
        if self.factored:
            rec = self._record(self._view)
            views["sh_hdr"] = rec[:SH_SLOT_HEADER]
            views["dsh_rgb"] = rec[SH_SLOT_HEADER:].view(3, self._plane)
            views["dsh"] = self.dsh
        return views

    def _record(self, v):
        """View v's record inside THIS rank's buffer (valid for v != own rank only after an all-gather)."""
        return self.flat[self.n_reduce + v * self._slot:self.n_reduce + (v + 1) * self._slot]

    def zero_(self):
        self.flat.zero_()
        if self.dsh is not None:
            self.dsh.zero_()

    # ---- factored SH gradient: sum over the views' records ------------------------------------------------------
    def _expand_sh(self, record_ptrs, means3D):
        """dsh = sum_v w(dir(means3D, camera_v)) (x) rgb_v from the records at `record_ptrs` (device addresses valid in this
        process: local or peer memory), by the library's kernel."""
        if means3D is None:
            means3D = self.views.get("_means3D")
        if means3D is None:
            raise RuntimeError("GradBucket.all_reduce: the factored SH gradient needs means3D (run the rasterizer backward with _out=bucket.views "
                               "first, or pass means3D=)")
        if not (means3D.is_cuda and means3D.dtype == torch.float32 and means3D.is_contiguous() and tuple(means3D.shape) == (self.P, 3)):
            raise RuntimeError("GradBucket: means3D must be a contiguous CUDA float32 (P,3) tensor")
        arr = (ctypes.c_void_p * len(record_ptrs))(*record_ptrs)
        with torch.cuda.device(self.flat.device):
            _C._check(_C._lib.gof_sh_grad_from_views(self.P, self.M, len(record_ptrs), means3D.data_ptr(), arr, self.dsh.data_ptr(), _C._stream()))

    def _expand_sh_torch(self, means3D):
        """The same sum with torch ops from the all-gathered local records (CPU buckets of the gloo tests; the reference the CUDA
        kernel is tested against)."""
        if means3D is None:
            means3D = self.views.get("_means3D")
        if means3D is None:
            raise RuntimeError("GradBucket.all_reduce: the factored SH gradient needs means3D")
        self.dsh.copy_(sh_grad_from_views_torch(means3D, [self._record(v) for v in range(self._n_views)], self.P, self.M))

    def _record_ptrs(self):
        """Addresses (valid in this process) of every rank's record IN THAT RANK'S OWN BUFFER, or None when peers' memory is
        not mapped (NCCL / gloo: the records are all-gathered into the local buffer instead)."""
        tail = lambda r: 4 * (self.n_reduce + r * self._slot)   # noqa: E731
        if self.exchange == "p2p":
            return [int(self._peer_ptrs[r]) + tail(r) for r in range(self._n_views)]
        if self.exchange == "nvls":
            off = self.flat.data_ptr() - int(self._symm.buffer_ptrs[self._view])
            return [int(self._symm.buffer_ptrs[r]) + off + tail(r) for r in range(self._n_views)]
        return None

    def enable_peer_exchange(self, group=None):
        """Move the bucket into a CUDA-IPC shareable allocation, map every other rank's bucket into this process (one node,
        NVLink) and switch all_reduce() to the library's peer-memory kernel.  Collective: every rank of `group` must call
        it, before the views are handed to anyone (they are re-created).  Raises if mapping or the self-test fails."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return self
        if not self.flat.is_cuda or self.flat.dtype != torch.float32:
            raise RuntimeError("peer exchange needs a CUDA float32 bucket")
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        if world > 8:
            raise RuntimeError("peer exchange: at most 8 ranks (one NVSwitch domain)")
        lib, dev, n = _C._lib, self.flat.device, self.flat.numel()
        for f in ("gof_peer_alloc", "gof_peer_open", "gof_p2p_allreduce_f32"):
            getattr(lib, f).restype = ctypes.c_int
        lib.gof_peer_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p), ctypes.c_char_p]
        lib.gof_peer_open.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_void_p)]
        lib.gof_p2p_allreduce_f32.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p]
        def agree(ok):   # True only if every rank says so: all ranks leave this function the same way (raise or return)
            t = torch.tensor([1.0 if ok else 0.0], dtype=torch.float32, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            return float(t.item()) == 1.0

        ptr, handle = ctypes.c_void_p(0), ctypes.create_string_buffer(64)
        err = None
        with torch.cuda.device(dev):
            torch.cuda.synchronize()
            try:
                _C._check(lib.gof_peer_alloc(n * 4, ctypes.byref(ptr), handle))
                mine = bytes(handle.raw)
            except Exception as e:   # noqa: BLE001 -- reported below, on every rank
                err, mine = e, None
            handles = [None] * world
            dist.all_gather_object(handles, mine, group=group)
            ptrs = []
            if err is None and all(h is not None for h in handles):
                try:
                    for r in range(world):
                        if r == rank:
                            ptrs.append(ptr.value)
                        else:
                            q = ctypes.c_void_p(0)
                            _C._check(lib.gof_peer_open(handles[r], ctypes.byref(q)))
                            ptrs.append(q.value)
                except Exception as e:   # noqa: BLE001
                    err = e
            elif err is None:
                err = RuntimeError("a peer could not allocate its shareable bucket")
        self._lib = lib
        self._own_ptr = ptr.value
        self._mapped = [q for r, q in enumerate(ptrs) if r != rank]
        if not agree(err is None):
            self._release_peer_memory()
            raise RuntimeError(f"peer exchange: mapping failed on some rank ({err if err is not None else 'another rank'})")

        class _Raw:   # zero-copy torch view of the cudaMalloc'ed bucket
            __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr.value, False), "version": 2}
        self._raw = _Raw()
        self.flat = torch.as_tensor(self._raw, device=dev)
        if self.flat.data_ptr() != ptr.value or self.flat.numel() != n:
            raise RuntimeError("peer exchange: could not wrap the shared allocation")
        self.views = self._make_views()
        self._peer_ptrs = (ctypes.c_void_p * world)(*ptrs)
        self._sync = torch.zeros(1, dtype=torch.float32, device=dev)
        self._lib, self._check, self._world, self._rank = lib, _C._check, world, rank
        self.exchange = "p2p"
        dist.barrier(group=group)
        # self-test on the live mapping: ones must sum to `world` in every bucket
        self.flat.fill_(1.0)
        self.all_reduce(group=group, _expand=False)
        torch.cuda.synchronize(dev)
        good = bool((self.flat[:self.n_sum] == float(world)).all().item()) and bool((self.flat[self.n_sum:self.n_reduce] == 1.0).all().item())
        rec_ok = self._selftest_records(group)       # collective: evaluated on every rank, whatever `good` says
        good = agree(good and rec_ok)
        self.flat.zero_()
        if not good:
            self.close()
            raise RuntimeError("peer exchange self-test failed on some rank")
        return self

    def _release_peer_memory(self):
        lib = getattr(self, "_lib", None)
        if lib is None:
            return
        lib.gof_peer_close.argtypes = [ctypes.c_void_p]
        lib.gof_peer_free.argtypes = [ctypes.c_void_p]
        for q in self._mapped:
            if q:
                lib.gof_peer_close(ctypes.c_void_p(q))
        self._mapped = []
        if self._own_ptr:
            lib.gof_peer_free(ctypes.c_void_p(self._own_ptr))
        self._own_ptr = None

    def close(self, group=None):
        """Leaves peer-exchange mode: unmaps the peers' buckets, frees the shared allocation and falls back to a torch-owned
        buffer + NCCL.  Collective when peer exchange was enabled (every rank must stop using its peers' memory first).
        The views are re-created (their contents are not kept)."""
        if self.exchange == "nvls":
            dev, n = self.flat.device, self.flat.numel()
            if dist.is_available() and dist.is_initialized():
                torch.cuda.synchronize(dev)
                dist.barrier(group=group)
            self.exchange, self._symm = "nccl", None
            self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
            self.views = self._make_views()
            return
        if self.exchange != "p2p" and not self._own_ptr:
            return
        dev = self.flat.device
        if dist.is_available() and dist.is_initialized():
            torch.cuda.synchronize(dev)
            dist.barrier(group=group)
        self.exchange = "nccl"
        n = self.flat.numel()
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.views = self._make_views()
        self._raw, self._peer_ptrs = None, None
        self._release_peer_memory()

    def __del__(self):
        # non-collective last resort (interpreter teardown / bucket re-created after densification without close()):
        # the mappings and the allocation are released; peers that still map this bucket keep it alive in the driver
        try:
            self._release_peer_memory()
        except Exception:   # noqa: BLE001
            pass

    def enable_nvls_exchange(self, group=None):
        """Move the bucket into a torch symmetric-memory allocation -- every rank's copy bound to ONE NVSwitch multicast object
        -- and switch all_reduce() to the library's multimem kernel (csrc/exchange.cu: k_nvls_allreduce).  Collective; the views
        are re-created.  Raises (on every rank alike) when the fabric / driver offers no multicast or the self-test fails."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return self
        if not self.flat.is_cuda or self.flat.dtype != torch.float32:
            raise RuntimeError("NVLS exchange needs a CUDA float32 bucket")
        import torch.distributed._symmetric_memory as symm_mem
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        dev, n = self.flat.device, self.flat.numel()
        lib = _C._lib
        lib.gof_nvls_allreduce_f32.restype = ctypes.c_int
        lib.gof_nvls_allreduce_f32.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p]

        def agree(ok):
            t = torch.tensor([1.0 if ok else 0.0], dtype=torch.float32, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            return float(t.item()) == 1.0

        err, buf, hdl = None, None, None
        try:
            with torch.cuda.device(dev):
                buf = symm_mem.empty(n, dtype=torch.float32, device=dev)
                hdl = symm_mem.rendezvous(buf, group if group is not None else dist.group.WORLD)
            if not int(hdl.multicast_ptr):
                raise RuntimeError("this fabric / driver offers no multicast (multicast_ptr == 0)")
        except Exception as e:   # noqa: BLE001 -- reported below, on every rank alike
            err = e
        if not agree(err is None):
            raise RuntimeError(f"NVLS exchange: symmetric-memory setup failed on some rank ({err if err is not None else 'another rank'})")
        old = (self.flat, self.views, self.exchange)
        self.flat = buf
        self.flat.zero_()
        self.views = self._make_views()
        self._symm, self._mc = hdl, int(hdl.multicast_ptr) + (buf.data_ptr() - int(hdl.buffer_ptrs[rank]))
        self._sync = torch.zeros(1, dtype=torch.float32, device=dev)
        self._lib, self._check, self._world, self._rank = lib, _C._check, world, rank
        self.exchange = "nvls"
        dist.barrier(group=group)
        # self-test on the live mapping: rank r contributes r+1 to the SUM part and r to the MAX tail
        self.flat[:self.n_sum].fill_(float(rank + 1))
        self.flat[self.n_sum:].fill_(float(rank))
        self.all_reduce(group=group, _expand=False)
        torch.cuda.synchronize(dev)
        good = bool((self.flat[:self.n_sum] == float(world * (world + 1) // 2)).all().item()) and \
            bool((self.flat[self.n_sum:self.n_reduce] == float(world - 1)).all().item())
        rec_ok = self._selftest_records(group)       # collective: evaluated on every rank, whatever `good` says
        good = agree(good and rec_ok)
        self.flat.zero_()
        if not good:
            self.flat, self.views, self.exchange = old
            self._symm = None
            raise RuntimeError("NVLS exchange self-test failed on some rank")
        return self

    def autotune_exchange(self, group=None, modes=("nvls", "p2p", "nccl"), iters=5):
        """Measures the exchange with every mode this box supports (each adopted only after its collective self-test) and keeps
        the fastest: which one wins depends on the machine and the world size -- at two ranks a peer-memory kernel moves the
        fewest bytes per rank, while the in-switch reduction saves NVLink traffic as ranks are added.
        Collective; every rank takes the same decision (times are max-reduced).  Returns {mode: ms or the reason it is
        unavailable}; the views are re-created."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return {}
        dev = self.flat.device
        report, best, best_ms = {}, "nccl", float("inf")
        means = None
        if self.factored:     # realistic records: the expansion kernel skips Gaussians whose dL_dRGB is zero
            means = (torch.rand(self.P, 3, generator=torch.Generator().manual_seed(1)) * 4 - 2).to(dev)

        def prime():
            if self.factored:
                rec = self._record(self._view)
                rec[:4] = torch.tensor([0.3 * self._view - 0.5, 0.25, -3.0, 3.0], device=dev)
                rec[SH_SLOT_HEADER:].normal_()
                rec[SH_SLOT_HEADER:].view(3, self._plane)[:, ::7] = 0.0
                self.views["_means3D"] = means
        for mode in modes:
            try:
                if mode == "nvls":
                    self.enable_nvls_exchange(group)
                elif mode == "p2p":
                    self.enable_peer_exchange(group)
            except Exception as e:   # noqa: BLE001 -- symmetric on all ranks
                report[mode] = f"unavailable ({type(e).__name__}: {str(e)[:120]})"
                continue
            prime()
            for _ in range(2):
                self.all_reduce(group=group)
            dist.barrier(group=group)
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                self.all_reduce(group=group)
            e1.record()
            torch.cuda.synchronize(dev)
            t = torch.tensor([e0.elapsed_time(e1) / iters], dtype=torch.float64, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            report[mode] = float(t.item())
            if report[mode] < best_ms:
                best, best_ms = mode, report[mode]
            self.close(group)
        if best == "nvls":
            self.enable_nvls_exchange(group)
        elif best == "p2p":
            self.enable_peer_exchange(group)
        self.zero_()
        return report

    def _selftest_records(self, group=None):
        """Factored bucket, peer-memory / NVLS mode: the expansion kernel reading the peers' records in place gives what torch
        computes from an NCCL all-gather of the same records.  Collective; True when not factored."""
        if not self.factored:
            return True
        dev, rank = self.flat.device, self._view
        gen = torch.Generator().manual_seed(1234)
        means = (torch.rand(self.P, 3, generator=gen) * 4 - 2).to(dev)
        rec = self._record(rank)
        rec.zero_()
        rec[:4] = torch.tensor([0.3 * rank - 0.5, 0.25, -3.0 - 0.1 * rank, 3.0], device=dev)
        rgb = torch.randn(3, self._plane, generator=torch.Generator().manual_seed(77 + rank)).to(dev)
        rgb[:, rank::5] = 0.0
        rec[SH_SLOT_HEADER:] = rgb.reshape(-1)
        torch.cuda.synchronize(dev)
        dist.barrier(group=group)
        self._expand_sh(self._record_ptrs(), means)
        got = self.dsh.clone()
        recs = [torch.empty_like(rec) for _ in range(self._n_views)]
        dist.all_gather(recs, rec.clone(), group=group)
        want = sh_grad_from_views_torch(means, recs, self.P, self.M)
        torch.cuda.synchronize(dev)
        dist.barrier(group=group)
        self.dsh.zero_()
        return bool(torch.allclose(got, want, rtol=1e-4, atol=1e-5))

    def all_reduce(self, group=None, async_op=False, means3D=None, _expand=True):
        """SUM over ranks of floats [0, n_sum), MAX of the statistics tail [n_sum, n_reduce); a factored bucket then fills
        views["dsh"] with the sum over all ranks' views (`means3D`: the Gaussian centres the backward ran on -- remembered from
        the last rasterizer backward into this bucket when not given).  World size 1: no-op."""
        if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
            return None
        expand = self.factored and _expand
        if async_op and expand:
            raise ValueError("GradBucket.all_reduce(async_op=True) is not available for a factored bucket (the SH expansion follows the exchange)")
        if self.exchange in ("p2p", "nvls"):
            if async_op:
                raise ValueError("GradBucket.all_reduce(async_op=True) is not available with the peer-memory / NVLS exchange: "
                                 "the kernel is ordered on the current stream")
            # barrier: every rank's backward has filled its bucket (a 4-byte NCCL all-reduce on the same stream orders it
            # after the local kernels and completes only when every rank has reached it)
            dist.all_reduce(self._sync, group=group)
            stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            with torch.cuda.device(self.flat.device):
                if self.exchange == "p2p":
                    self._check(self._lib.gof_p2p_allreduce_f32(self._peer_ptrs, self._world, self._rank, self.n_sum, self.n_reduce, stream))
                else:
                    self._check(self._lib.gof_nvls_allreduce_f32(ctypes.c_void_p(self._mc), self._world, self._rank, self.n_sum,
                                                                 self.n_reduce, stream))
            if expand:   # the views' records are read where the ranks left them, over NVLink
                self._expand_sh(self._record_ptrs(), means3D)
            # barrier: every slice has been written into every bucket (and every record has been read)
            dist.all_reduce(self._sync, group=group)
            return None
        if self.n_sum == self.flat.numel():
            return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        w1 = dist.all_reduce(self.flat[:self.n_sum], op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        w2 = None
        if self.n_reduce > self.n_sum:
            w2 = dist.all_reduce(self.flat[self.n_sum:self.n_reduce], op=dist.ReduceOp.MAX, group=group, async_op=async_op)
        if expand:
            own = self._record(self._view)
            if self.flat.is_cuda:
                dist.all_gather_into_tensor(self.flat[self.n_reduce:], own, group=group)     # in place: own record already sits at its slot
                self._expand_sh([self.flat.data_ptr() + 4 * (self.n_reduce + v * self._slot) for v in range(self._n_views)], means3D)
            else:
                recs = [torch.empty_like(own) for _ in range(self._n_views)]
                dist.all_gather(recs, own.clone(), group=group)
                for v, r in enumerate(recs):
                    self._record(v).copy_(r)
                self._expand_sh_torch(means3D)
        return (w1, w2) if async_op else None

    @property
    def nbytes(self):
        """Bytes of the exchanged buffer (reduced part + the views' records)."""
        return self.flat.numel() * self.flat.element_size()


_SH_C1 = 0.4886025119029199
_SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
          -0.5900435899266435)


def sh_grad_weights_torch(dirs, degree):
    """d colour / d SH coefficient for unit directions `dirs` [P,3]: [P,(degree+1)^2] (backward.cu:45-139; gof_sh_grad_weights)."""
    x, y, z = dirs[:, 0], dirs[:, 1], dirs[:, 2]
    w = [torch.full_like(x, 0.28209479177387814)]
    if degree > 0:
        w += [-_SH_C1 * y, _SH_C1 * z, -_SH_C1 * x]
    if degree > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        w += [_SH_C2[0] * xy, _SH_C2[1] * yz, _SH_C2[2] * (2 * zz - xx - yy), _SH_C2[3] * xz, _SH_C2[4] * (xx - yy)]
    if degree > 2:
        w += [_SH_C3[0] * y * (3 * xx - yy), _SH_C3[1] * xy * z, _SH_C3[2] * y * (4 * zz - xx - yy), _SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
              _SH_C3[4] * x * (4 * zz - xx - yy), _SH_C3[5] * z * (xx - yy), _SH_C3[6] * x * (xx - 3 * yy)]
    return torch.stack(w, dim=1)


def sh_grad_from_views_torch(means3D, records, P, M):
    """sum_v w(dir(means3D, camera_v)) (x) rgb_v as [P,M,3] from view records (header: camera centre, degree | rgb planes [3][plane])."""
    out = torch.zeros(P, M, 3, dtype=means3D.dtype, device=means3D.device)
    for rec in records:
        cam, degree = rec[:3], int(round(float(rec[3])))
        plane = _C._sh_plane(P)
        rgb = rec[SH_SLOT_HEADER:SH_SLOT_HEADER + 3 * plane].view(3, plane)[:, :P].t()
        d = means3D - cam[None, :]
        d = d / torch.linalg.vector_norm(d, dim=1, keepdim=True)
        w = sh_grad_weights_torch(d, degree)
        out[:, :w.shape[1], :] += w[:, :, None] * rgb[:, None, :]
    return out


def densification_stats(dmeans2D, radii):
    """Per-view densification statistics of the reference (scene/gaussian_model.py:709-714): the norm of the
    signed screen-space gradient, the abs-sum gradient, a visibility count and the radius, as one [P,4]
    tensor so that a view-parallel step reduces 16 B/Gaussian instead of the raw dL_dmean2D of every view."""
    vis = radii > 0
    out = torch.zeros(dmeans2D.shape[0], 4, dtype=torch.float32, device=dmeans2D.device)
    out[:, 0] = torch.where(vis, torch.linalg.vector_norm(dmeans2D[:, :2], dim=-1), out[:, 0])
    out[:, 1] = torch.where(vis, torch.linalg.vector_norm(dmeans2D[:, 2:], dim=-1), out[:, 1])
    out[:, 2] = vis.to(torch.float32)
    out[:, 3] = radii.to(torch.float32)
    return out


def all_reduce_densification_stats(stats, group=None):
    """SUM for the two gradient norms and the visibility count, MAX for the radius."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return stats
    sums = stats[:, :3].contiguous()
    mx = stats[:, 3].contiguous()
    dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=group)
    return torch.cat([sums, mx[:, None]], dim=1)


def view_for(step, rank, world_size, n_views=64):
    """Round-robin view schedule: step s gives rank r view (s*world_size + r) mod n_views."""
    return (step * world_size + rank) % n_views
