"""Time BiCGSTAB steps (csrc/solver.cu) on a generated matrix; prints one JSON line.
The point is the cost of a step next to its two SpMVs (the iteration itself need not converge).
  python tools/time_bicgstab.py [--n 10000000] [--per-row 100] [--steps 10]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--per-row", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = args.n
    a = G.rmat_csr(ctx, n, args.per_row, seed=0x5EED0005)
    # convergence is irrelevant for the cost of a step: the R-MAT matrix is used as it is
    lib = ctx.lib
    x0 = G.normal_vector(ctx, n, 1)
    b = G.normal_vector(ctx, n, 2)
    G._sync()  # new_dev copies x0 / b on the library's stream: torch's must have written them
    h = C.c_void_p()
    ctx.check(lib.sprs_b200_bicgstab_new_dev(ctx.h, a.mirror.h, C.c_void_p(x0.data_ptr()),
                                             C.c_void_p(b.data_ptr()), n, C.byref(h)))
    err = C.c_double()
    for _ in range(2):
        ctx.check(lib.sprs_b200_bicgstab_step(h, C.byref(err)))
    ctx.synchronize()
    y = torch.empty(n, device=x0.device, dtype=torch.float64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        G.spmv(ctx, a, x0, y)
    e0.record()
    for _ in range(10):
        G.spmv(ctx, a, x0, y)
    e1.record()
    torch.cuda.synchronize()
    spmv_ms = e0.elapsed_time(e1) / 10
    l0 = ctx.launches
    t0 = time.perf_counter()
    for _ in range(args.steps):
        ctx.check(lib.sprs_b200_bicgstab_step(h, C.byref(err)))
    ctx.synchronize()
    step_ms = (time.perf_counter() - t0) / args.steps * 1e3
    launches = (ctx.launches - l0) / args.steps
    lib.sprs_b200_bicgstab_free(h)
    print(json.dumps({"workload": "bicgstab_step_rmat", "n": n, "nnz": a.nnz,
                      "step_ms": round(step_ms, 4), "spmv_ms": round(spmv_ms, 4),
                      "vector_part_ms": round(step_ms - 2 * spmv_ms, 4),
                      "launches_per_step": launches, "err": err.value,
                      "vector_bytes_per_step": 128 * n,
                      "note": "wall clock over %d steps incl. 3 scalar syncs per step" % args.steps}))


if __name__ == "__main__":
    main()
