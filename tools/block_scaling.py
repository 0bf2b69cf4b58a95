"""Row blocks of 1/8 .. 1 of the config-5 matrix (full x) on one GPU: how the SpMV rate depends
on the block (rows per non-zero differ 3x between the head and the tail of an R-MAT matrix)."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sprs_b200 as sp  # noqa: E402
from sprs_b200 import generate as G  # noqa: E402
from sprs_b200.dist import nnz_balanced_bounds  # noqa: E402

ctx = sp.Context.default(0)
n = 10_000_000
full = G.make_matrix(ctx, "rmat", n, 100, 0x5EED0005)
x = G.normal_vector(ctx, n)
b = nnz_balanced_bounds(full.indptr, 8, row_cost=30.0)
s_own = torch.cuda.Stream()
sptr = C.c_void_p(s_own.cuda_stream)


FLUSH_LIST = [int(v) for v in os.environ.get("BLOCK_SCALING_FLUSH_MB", "0").split(",")]  # > 0: write that many MB between products
FLUSH_MB = 0
flush = torch.empty(max(max(FLUSH_LIST), 1) << 17, device="cuda", dtype=torch.float64)


def time_block_cold(a, y, stream_ptr, reps=20):
    """each product timed on its own, after FLUSH_MB of plain writes went through L2 (what a
    rank's L2 sees between two steps when its peers deposit their slices of y)"""
    tot = 0.0
    with torch.cuda.stream(s_own):
        for i in range(reps + 3):
            flush[:FLUSH_MB << 17].fill_(float(i))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s_own)
            ctx.check(ctx.lib.sprs_b200_spmv_dev(ctx.h, a.mirror.h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), 0, stream_ptr))
            e1.record(s_own)
            s_own.synchronize()
            if i >= 3:
                tot += e0.elapsed_time(e1)
    return tot / reps


def time_block(r0, r1, persist, stream_ptr, reps=30):
    a = full if (r0, r1) == (0, n) else full.slice_rows(r0, r1)
    y = torch.empty(max(r1 - r0, 1), device="cuda", dtype=torch.float64)
    torch.cuda.synchronize()
    if FLUSH_MB:
        return a.nnz, time_block_cold(a, y, stream_ptr)
    with torch.cuda.stream(s_own):
        for _ in range(5):
            ctx.check(ctx.lib.sprs_b200_spmv_dev(ctx.h, a.mirror.h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), 0, stream_ptr))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s_own)
        for _ in range(reps):
            ctx.check(ctx.lib.sprs_b200_spmv_dev(ctx.h, a.mirror.h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), 0, stream_ptr))
        e1.record(s_own)
    torch.cuda.synchronize()
    return a.nnz, e0.elapsed_time(e1) / reps


for FLUSH_MB in FLUSH_LIST:
    persist = False
    pts = []
    for lo, hi in ((0, 1), (3, 4), (6, 7), (2, 4), (4, 8), (0, 8)):
        nnz, ms = time_block(b[lo], b[hi], persist, sptr)
        pts.append((nnz, ms))
        print(json.dumps({"flush_mb": FLUSH_MB, "prefetch_x": os.environ.get("SPRS_B200_SPMV_PREFETCH_X", "1"), "blocks": [lo, hi], "nnz": nnz, "ms": round(ms, 4),
                          "gnnz_s": round(nnz / ms / 1e6, 1)}), flush=True)
    A = np.array([[1.0, p[0]] for p in pts])
    t = np.array([p[1] for p in pts])
    (a0, b0), *_ = np.linalg.lstsq(A, t, rcond=None)
    print(json.dumps({"persist_x_in_l2": persist, "fit_fixed_ms": round(float(a0), 4),
                      "fit_gnnz_s": round(1.0 / b0 / 1e6, 1)}), flush=True)
