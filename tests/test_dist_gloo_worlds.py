"""CPU, over gloo at world sizes 3 and 5 (test_dist_gloo.py stops at 2): gof_dp.GradBucket's CPU exchange, plain and with the
factored SH gradient.

With three or more addends the order of a sum shows in its last bits, and gloo's reduction order is its own, so the SUM fields
are held to the bound every fp32 summation order of N addends meets: |got - exact| <= (N-1) 2^-24 sum_r |b_r|, exact = the
fp64 sum.  The MAX tail (dens_max) is exact in any order.  The all-gathered view records must be every rank's own record,
views["dsh"] their expansion by gof_dp.sh_grad_from_views_torch, and every rank must hold the same bits."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gaussian-opacity-fields_b200")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _values(shape, g):
    """Normal floats of mixed sign and exponent (randn 2^k, k in [-20, 20])."""
    return torch.randn(shape, generator=g) * torch.exp2(torch.randint(-20, 21, shape, generator=g).float())


def _worker(rank, world, port, q, factored):
    sys.path.insert(0, PKG)
    import gof_dp
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    P, M = (203, 16) if factored else (257, 16)
    b = gof_dp.GradBucket(P, M, "cpu", factor_sh=factored)
    g = torch.Generator().manual_seed(1000 * world + rank)
    names = [n for n in b.views if n not in ("dsh", "sh_hdr", "dsh_rgb")] + ([] if factored else ["dsh"])
    local = {}
    for n in names:
        v = b.views[n]
        v.copy_(_values(v.shape, g).abs() if n == "dens_max" else _values(v.shape, g))
    if factored:
        rgb = b.views["dsh_rgb"]
        rgb.copy_(torch.randn(rgb.shape, generator=g))
        rgb[:, rank::3] = 0.0                                         # Gaussians this view does not see
        rgb[1:, rank + 1::5] = 0.0                                    # ... and rows with one non-zero channel
        rgb[:, P:] = 0.0
        b.views["sh_hdr"][:4] = torch.tensor([2.5 + rank, -1.0 + 0.25 * rank, 0.5 * rank - 1.0, float(3 - rank % 4)])
        local["record"] = b._record(rank).clone()
    for n in names:
        local[n] = b.views[n].clone()
    means = torch.randn(P, 3, generator=torch.Generator().manual_seed(5)) * 2     # the same Gaussians on every rank
    b.all_reduce(means3D=means if factored else None)
    got = {n: b.views[n].clone() for n in names}
    if factored:
        got["dsh"] = b.views["dsh"].clone()
        got["records"] = [b._record(v).clone() for v in range(world)]
    # plain numpy in the queue: tensors would be shared by fd and the worker exits before the parent reads
    q.put((rank, {k: v.numpy().copy() for k, v in local.items()},
           {k: ([r.numpy().copy() for r in v] if k == "records" else v.numpy().copy()) for k, v in got.items()},
           b.flat.numpy().copy(), means.numpy().copy(), b.n_sum, b.n_reduce))
    dist.destroy_process_group()


def _run(world, factored):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, factored)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in range(world)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def _bits(a):
    return torch.from_numpy(a).view(torch.int32)


@pytest.mark.parametrize("factored", [False, True])
@pytest.mark.parametrize("world", [3, 5])
def test_bucket_allreduce_at_world(world, factored):
    res = _run(world, factored)
    t = torch.from_numpy
    locals_ = [r[1] for r in res]
    for name in (n for n in locals_[0] if n != "record"):
        parts = [t(loc[name]) for loc in locals_]
        got = t(res[0][2][name])
        if name == "dens_max":
            want = parts[0]
            for p in parts[1:]:
                want = torch.maximum(want, p)
            assert torch.equal(got, want), name
        else:
            exact = sum(p.double() for p in parts)
            bound = (world - 1) * 2.0 ** -24 * sum(p.double().abs() for p in parts)
            assert bool(((got.double() - exact).abs() <= bound).all()), name
            assert float(bound.max()) > 0
    for r in range(1, world):                                      # every rank holds the same bits
        assert torch.equal(_bits(res[r][3]), _bits(res[0][3]))
        for name in res[0][2]:
            if name != "records":
                assert torch.equal(_bits(res[r][2][name]), _bits(res[0][2][name])), (r, name)
    if not factored:
        return
    sys.path.insert(0, PKG)
    import gof_dp
    P, M = res[0][2]["dsh"].shape[:2]
    for r in range(world):
        recs = [t(a) for a in res[r][2]["records"]]
        for v in range(world):                                     # the gathered records are the ranks' own
            assert torch.equal(recs[v].view(torch.int32), t(locals_[v]["record"]).view(torch.int32)), (r, v)
        want = gof_dp.sh_grad_from_views_torch(t(res[r][4]), recs, P, M)
        assert torch.equal(t(res[r][2]["dsh"]).view(torch.int32), want.view(torch.int32)), r
    dsh = t(res[0][2]["dsh"])
    assert torch.isfinite(dsh).all() and float(dsh[:, 9:].abs().max()) > 0      # a degree-3 view reaches the top band
