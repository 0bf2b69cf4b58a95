"""Driver of tools/spmv_lab.cu: ceiling-kernel sweep on the bench's own matrices (GPU box only).
    python tools/spmv_lab.py [quick|full] > lab.txt
Prints one line per variant: workload, variant, ms, Gnnz/s, fraction of the HBM roofline the
12 B/nnz stream would reach at that rate."""
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sprs_b200 as sp  # noqa: E402
from sprs_b200 import generate as G  # noqa: E402

lab = C.CDLL(os.path.join(ROOT, "tools", "libspmv_lab.so"))
lab.lab_ceiling.restype = C.c_int
lab.lab_ceiling.argtypes = [C.c_int] * 6 + [C.c_uint32, C.c_uint32] + [C.c_void_p] * 4 + [C.c_uint64, C.c_int, C.c_void_p]

PEAK = 6590.9
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def ceiling(a, x, out, epl, mode, gop, minb, carve=-1, cmode=0, mask=0xFFFFFFFF, iters=5):
    ms = (C.c_float * 2)()
    rc = lab.lab_ceiling(epl, mode, gop, minb, carve, cmode, mask, a.cols, a.indices.data_ptr(),
                         a.data.data_ptr(), x.data_ptr(), out.data_ptr(), a.nnz, iters, ms)
    torch.cuda.synchronize()
    return (ms[0], int(ms[1])) if rc == 0 else (None, rc)


def product_ms(ctx, a, x, y, k=10):
    for _ in range(3):
        G.spmv(ctx, a, x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        G.spmv(ctx, a, x, y)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def report(name, tag, a, ms, occ=None):
    if ms is None:
        print("%-14s %-28s FAILED rc=%s" % (name, tag, occ), flush=True)
        return
    gb = (12.0 * a.nnz + 8.0 * a.rows) / ms / 1e6
    print("%-14s %-28s %8.3f ms %7.1f Gnnz/s  frac %.3f%s" % (
        name, tag, ms, a.nnz / ms / 1e6, gb / PEAK, "" if occ is None else "  occ %d" % occ), flush=True)


def main():
    full = len(sys.argv) > 1 and sys.argv[1] == "full"
    ctx = sp.Context.default(0)
    dev = torch.device("cuda", 0)
    wl = [("rmat_10m_100", "rmat", 10_000_000, 100, 0x5EED0005), ("rand_1m_32", "rand", 1_000_000, 32, 0x5EED0002)]
    for name, gen, n, npr, seed in wl:
        a = G.make_matrix(ctx, gen, n, npr, seed)
        x = G.normal_vector(ctx, n)
        y = torch.empty(n, device=dev, dtype=torch.float64)
        out = torch.empty(ctx.sm_count * 6 * 256 + 4096, device=dev, dtype=torch.float64)
        report(name, "product spmv", a, product_ms(ctx, a, x, y))
        # 1. the grid: EPL x MODE x GOP x MINB, real columns, exact carve-out
        epls = (8, 12, 16)
        modes = (0, 1, 2, 3)
        gops = (0, 1, 2, 3) if full else (0, 1)
        minbs = (2, 3, 4, 6)
        for epl in epls:
            for mode in modes:
                for gop in gops:
                    for minb in minbs:
                        ms, occ = ceiling(a, x, out, epl, mode, gop, minb)
                        report(name, "ceil e%d m%d g%d b%d" % (epl, mode, gop, minb), a, ms, occ)
        # 2. carve-out sweep for the direct modes (L1 size vs gather rate)
        for mode in (0, 2):
            for carve in (0, 25, 50, 75, 100):
                ms, occ = ceiling(a, x, out, 12, mode, 0, 3, carve=carve)
                report(name, "ceil e12 m%d g0 b3 carve%d" % (mode, carve), a, ms, occ)
        # 3. where is the wall: x range shrunk (L2-near / L1-sized), sequential columns
        for mask, lbl in ((0xFFFFF, "x8MB"), (0x1FFFF, "x1MB"), (0x3FFF, "x128KB")):
            ms, occ = ceiling(a, x, out, 12, 0, 0, 3, cmode=1, mask=mask)
            report(name, "ceil e12 m0 g0 b3 " + lbl, a, ms, occ)
            ms, occ = ceiling(a, x, out, 12, 1, 0, 3, cmode=1, mask=mask)
            report(name, "ceil e12 m1 g0 b3 " + lbl, a, ms, occ)
        for mode in (0, 1, 3):
            ms, occ = ceiling(a, x, out, 12, mode, 0, 3, cmode=2)
            report(name, "ceil e12 m%d g0 b3 seq" % mode, a, ms, occ)
        del a, x, y, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
