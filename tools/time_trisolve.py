"""Times the device triangular solves (csrc/trisolve.cu) and prints one JSON line per workload.

    python tools/time_trisolve.py [--iters 20] [--only rand1m_lower,chain100k]

Per workload: n, the non-zeros of the solved triangle (diagonal included), the depth of its
dependency graph (tests/trisolve_oracle.py levels), the plan time (host clock around the
blocking plan call), the solve time (CUDA events around solve_dev only, median and min of
`iters` solves after two warm-ups; rhs refilled outside the events), the host-call time
(sprs_b200_trisolve_solve with host rhs: copies included), the oracle's single-thread time,
parity bit for bit on the whole x, and the compulsory bytes 12 nnz + w (n + 1) + 4 n + 16 n
(indices and values, indptr of width w, the diagonal offsets, x read and written) with their
share of 3.35 TB/s.  GPU name, power limit and SM clock are read in the same process.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sprs_b200 as sp  # noqa: E402
import trisolve_oracle as TO  # noqa: E402
from sprs_b200 import generate as G  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def lap2d_lower(ctx, m):
    """Lower triangle of the 5-point Laplacian on an m x m grid: row i = y m + x holds -1 at
    i - m and i - 1 (inside the grid) and 4 on the diagonal (the Gauss-Seidel sweep of
    examples/heat.rs)."""
    dev = G._device(ctx)
    n = m * m
    i = torch.arange(n, device=dev, dtype=torch.int64)
    has_s, has_w = i >= m, (i % m) != 0
    cnt = 1 + has_s.to(torch.int64) + has_w.to(torch.int64)
    ip = torch.zeros(n + 1, device=dev, dtype=torch.int64)
    torch.cumsum(cnt, 0, out=ip[1:])
    nnz = int(ip[-1])
    ind = torch.empty(nnz, device=dev, dtype=torch.int32)
    val = torch.empty(nnz, device=dev, dtype=torch.float64)
    p = ip[:-1].clone()
    ind[p[has_s]] = (i[has_s] - m).to(torch.int32)
    val[p[has_s]] = -1.0
    p += has_s.to(torch.int64)
    ind[p[has_w]] = (i[has_w] - 1).to(torch.int32)
    val[p[has_w]] = -1.0
    p += has_w.to(torch.int64)
    ind[p] = i.to(torch.int32)
    val[p] = 4.0
    G._sync()
    return G.DeviceCsr(ctx, n, n, ip.to(torch.int32), ind, val)


def chain(ctx, n):
    """Lower bidiagonal: x_r depends on x_{r-1} -- depth n."""
    rng = np.random.default_rng(9)
    ip = np.concatenate([[0], np.arange(1, 2 * n, 2)]).astype(np.int32)
    ind = np.empty(2 * n - 1, np.int32)
    val = np.empty(2 * n - 1)
    ind[0], val[0] = 0, 1.5
    ind[1::2], ind[2::2] = np.arange(n - 1), np.arange(1, n)
    val[1::2], val[2::2] = rng.standard_normal(n - 1) * 0.5, 1.0 + rng.random(n - 1)
    dev = G._device(ctx)
    return G.DeviceCsr(ctx, n, n, torch.from_numpy(ip).to(dev), torch.from_numpy(ind).to(dev),
                       torch.from_numpy(val).to(dev))


def measure(ctx, name, t, lower, csc, iters):
    if csc:
        mirror, ip, ind, dat = G._with_views(ctx, t.mirror.to_other_storage())
    else:
        mirror, ip, ind, dat = t.mirror, t.indptr, t.indices, t.data
    n, nnz = t.rows, t.nnz
    form = ("lsolve_" if lower else "usolve_") + ("csc" if csc else "csr")
    hip, hind = ip.cpu().numpy().view(np.uint32), ind.cpu().numpy().view(np.uint32)
    hdat = dat.cpu().numpy()
    depth = TO.levels(hip, hind, upper=not lower, csr=not csc)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    plan = sp.linalg.TriSolvePlan(mirror, lower)
    plan_ms = (time.perf_counter() - t0) * 1e3
    b = G.normal_vector(ctx, n, seed=0x5EED7100)
    x = torch.empty_like(b)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for it in range(iters + 2):
        x.copy_(b)
        e0.record()
        assert G.trisolve_dev(ctx, plan, x) is None
        e1.record()
        e1.synchronize()
        if it == 0:
            got = x.cpu().numpy()
        if it >= 2:
            times.append(e0.elapsed_time(e1))
    hb = b.cpu().numpy()
    hx = hb.copy()
    t0 = time.perf_counter()
    plan.solve(hx)
    host_ms = (time.perf_counter() - t0) * 1e3
    want = hb.copy()
    t0 = time.perf_counter()
    assert TO.solve(form, hip, hind, hdat, want) is None
    oracle_ms = (time.perf_counter() - t0) * 1e3
    parity = TO.first_difference(got, want) is None and TO.first_difference(hx, want) is None
    plan.free()
    w = 4  # every mirror timed here has a u32 indptr
    bytes_ = 12 * nnz + w * (n + 1) + 4 * n + 16 * n
    med = float(np.median(times))
    return dict(workload=name, form=form, n=n, nnz=nnz, depth=depth, plan_ms=round(plan_ms, 3),
                solve_ms_median=round(med, 4), solve_ms_min=round(float(np.min(times)), 4),
                host_call_ms=round(host_ms, 3), oracle_ms=round(oracle_ms, 3),
                speedup_vs_oracle=round(oracle_ms / med, 2), parity_bits=bool(parity),
                compulsory_bytes=bytes_, hbm_share=round(bytes_ / (med * 1e-3) / HBM_BPS, 4),
                iters=iters, gpu=gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    only = set(filter(None, args.only.split(",")))
    ctx = sp.Context.default()

    def want(*names):
        return not only or any(n in only for n in names)

    if want("rand1m_lower", "rand1m_upper", "rand1m_lower_csc"):
        a = G.rand_csr(ctx, 1_000_000, 1_000_000, 32, seed=0x5EED0002)
        for name, lower, csc in (("rand1m_lower", True, False), ("rand1m_upper", False, False),
                                 ("rand1m_lower_csc", True, True)):
            if want(name):
                print(json.dumps(measure(ctx, name, G.triangular(ctx, a, lower), lower, csc,
                                         args.iters)), flush=True)
        del a
    if want("rmat10m_lower", "rmat10m_upper"):
        a = G.rmat_csr(ctx, 10_000_000, 100, seed=0x5EED0005)
        for name, lower in (("rmat10m_lower", True), ("rmat10m_upper", False)):
            if want(name):
                t = G.triangular(ctx, a, lower)
                print(json.dumps(measure(ctx, name, t, lower, False, args.iters)), flush=True)
                del t
                torch.cuda.empty_cache()
        del a
    if want("lap2d_lower"):
        print(json.dumps(measure(ctx, "lap2d_lower", lap2d_lower(ctx, 2000), True, False,
                                 args.iters)), flush=True)
    if want("chain100k"):
        print(json.dumps(measure(ctx, "chain100k", chain(ctx, 100_000), True, False, args.iters)),
              flush=True)


if __name__ == "__main__":
    main()
