#!/usr/bin/env python
"""Developer tool (GPU box, under torchrun with N >= 2 ranks): sweeps the launch parameters of the gradient-bucket exchange
kernels (csrc/exchange.cu probes) on the 256 MB C3 bucket -- NVLS (multimem) and peer-memory variants -- next to NCCL's
all-reduce and torch's own multimem all-reduce, and writes one JSON line per variant to tool_out/exchange_sweep_n<N>.jsonl.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/exchange_sweep.py
"""
import ctypes
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
import gof_dp  # noqa: E402
from diff_gaussian_rasterization import _C  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
lib = _C._lib
lib.gof_nvls_probe.restype = ctypes.c_int
lib.gof_nvls_probe.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t] + [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_void_p]
lib.gof_p2p_probe.restype = ctypes.c_int
lib.gof_p2p_probe.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t] + [ctypes.c_int] * 4 + [ctypes.c_void_p]

P = 1_000_000
out_path = os.path.join(ROOT, "tool_out", f"exchange_sweep_n{world}.jsonl")
sync = torch.zeros(1, device=dev)
sms = torch.cuda.get_device_properties(dev).multi_processor_count
ITERS = 6


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def timed(fn, barriers=True):
    """ms per call (max over ranks): like GradBucket.all_reduce, each call bracketed by two 4-byte NCCL all-reduces."""
    def once():
        if barriers:
            dist.all_reduce(sync)
        fn()
        if barriers:
            dist.all_reduce(sync)
    for _ in range(2):
        once()
    dist.barrier()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        once()
    e1.record()
    torch.cuda.synchronize(dev)
    t = torch.tensor([e0.elapsed_time(e1) / ITERS], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


results = []


def report(**kw):
    if rank == 0:
        results.append(kw)
        print(json.dumps(kw), flush=True)


# ---- library references
bucket = gof_dp.GradBucket(P, 16, dev)
n = bucket.flat.numel()
report(kind="nccl_allreduce_sum_whole_bucket", ms=timed(lambda: dist.all_reduce(bucket.flat), barriers=False), bytes=n * 4)
report(kind="barrier_pair_only", ms=timed(lambda: None))

# ---- NVLS
try:
    bucket.enable_nvls_exchange()
    report(kind="nvls_production", ms=timed(lambda: bucket.all_reduce(), barriers=False))
    mc = ctypes.c_void_p(bucket._mc)
    sink = torch.zeros(16, device=dev)
    try:
        import torch.distributed._symmetric_memory as symm_mem  # noqa: F401
        gname = dist.group.WORLD.group_name
        report(kind="torch_multimem_all_reduce_", ms=timed(lambda: torch.ops.symm_mem.multimem_all_reduce_(bucket.flat, "sum", gname), barriers=False))
    except Exception as e:  # noqa: BLE001
        report(kind="torch_multimem_all_reduce_", error=str(e)[:200])

    def nvls(grid, threads, unroll, layout, mode):
        with torch.cuda.device(dev):
            _C._check(lib.gof_nvls_probe(mc, world, rank, n, grid, threads, unroll, layout, mode, ctypes.c_void_p(sink.data_ptr()), stream()))

    # correctness of one probe configuration before timing anything
    bucket.flat.fill_(float(rank + 1))
    dist.barrier(); torch.cuda.synchronize(dev)
    dist.all_reduce(sync); nvls(sms * 2, 512, 4, 1, 3); dist.all_reduce(sync)
    torch.cuda.synchronize(dev)
    ok = bool((bucket.flat == float(world * (world + 1) // 2)).all().item())
    report(kind="nvls_probe_selftest", ok=ok)
    bucket.flat.zero_()
    for mode in (3, 1, 2):
        for layout in (0, 1):
            for threads, per_sm in ((512, 4), (512, 2), (512, 1), (1024, 2), (1024, 1), (256, 8), (256, 4), (128, 8)):
                for unroll in (1, 2, 4, 8):
                    if mode != 3 and (unroll not in (2, 8) or layout == 0 and threads != 512):
                        continue
                    if threads * unroll > 2048:      # the unrolled variants do not fit 1024-thread CTAs (registers)
                        continue
                    ms = timed(lambda: nvls(sms * per_sm, threads, unroll, layout, mode))
                    report(kind="nvls_probe", mode=mode, layout=layout, threads=threads, ctas_per_sm=per_sm, unroll=unroll, ms=ms)
    # grids that are NOT a multiple of the SM count (few fat CTAs, NCCL-like)
    for grid in (16, 32, 64, 128):
        for unroll in (4, 8):
            ms = timed(lambda: nvls(grid, 512, unroll, 1, 3))
            report(kind="nvls_probe", mode=3, layout=1, threads=512, grid=grid, unroll=unroll, ms=ms)
    bucket.close()
except Exception as e:  # noqa: BLE001
    report(kind="nvls", error=f"{type(e).__name__}: {str(e)[:300]}")

# ---- peer memory
try:
    bucket = gof_dp.GradBucket(P, 16, dev)
    bucket.enable_peer_exchange()
    report(kind="p2p_production", ms=timed(lambda: bucket.all_reduce(), barriers=False))

    def p2p(grid, threads, unroll, layout):
        with torch.cuda.device(dev):
            _C._check(lib.gof_p2p_probe(bucket._peer_ptrs, world, rank, n, grid, threads, unroll, layout, stream()))

    bucket.flat.fill_(float(rank + 1))
    dist.barrier(); torch.cuda.synchronize(dev)
    dist.all_reduce(sync); p2p(sms * 2, 512, 2, 1); dist.all_reduce(sync)
    torch.cuda.synchronize(dev)
    report(kind="p2p_probe_selftest", ok=bool((bucket.flat == float(world * (world + 1) // 2)).all().item()))
    bucket.flat.zero_()
    max_unroll = {2: 8, 4: 4, 8: 2}.get(world, 1)
    if world in (2, 4, 8):
        for layout in (0, 1):
            for threads, per_sm in ((512, 4), (512, 2), (512, 1), (1024, 2), (1024, 1), (256, 8), (256, 4)):
                for unroll in (1, 2, 4, 8):
                    if unroll > max_unroll or threads * unroll * world > 4096:
                        continue
                    ms = timed(lambda: p2p(sms * per_sm, threads, unroll, layout))
                    report(kind="p2p_probe", layout=layout, threads=threads, ctas_per_sm=per_sm, unroll=unroll, ms=ms)
    bucket.close()
except Exception as e:  # noqa: BLE001
    report(kind="p2p", error=f"{type(e).__name__}: {str(e)[:300]}")

if rank == 0:
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        for r in results:
            f.write(json.dumps(r) + "\n")
dist.barrier()
dist.destroy_process_group()
