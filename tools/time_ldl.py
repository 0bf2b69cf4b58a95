"""Times the device LDL^T factorization (csrc/ldl.cu) and prints one JSON line per workload.

    python tools/time_ldl.py [--repeats 5] [--only nd2d_300,chain100k]

Per workload: n, |L|, the factorization's flops (sum over the columns of L of c (c - 1)
multiply-subtract flops for the column updates, plus 3 per entry of L for l_ki and D_k), the
height of the elimination tree (tests/ldl_oracle.py), the symbolic time (host clock around
LdlSymbolic.new_perm: the host walk and the uploads), the numeric time (host clock around the
blocking `update`, which ends in a device synchronise: the pattern check and the factorization
kernel; median of `repeats` after the first `factor`, or that `factor` alone for --repeats 0,
which includes the allocations), the solve time (CUDA events around solve_dev,
median of `repeats` after one warm-up), the oracle's single-thread times of the numeric
factorization and of the solve, and bit parity of L, D and x with the oracle.  GPU name, power
limit and SM clock are read in the same process.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sps
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ldl_oracle as LO  # noqa: E402
import sprs_b200 as sp  # noqa: E402
from sprs_b200 import generate as G  # noqa: E402
from test_gpu_ldl import laplacian, nested_dissection  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def chain(n):
    rng = np.random.default_rng(5)
    off = rng.standard_normal(n - 1)
    return sps.diags([off, 4.0 + rng.random(n), off], [-1, 0, 1], format="csr")


WORKLOADS = {
    "nd2d_100": lambda: (laplacian((100, 100)), nested_dissection((100, 100))),
    "nd2d_300": lambda: (laplacian((300, 300)), nested_dissection((300, 300))),
    "nd2d_1000": lambda: (laplacian((1000, 1000)), nested_dissection((1000, 1000))),
    "nd3d_20": lambda: (laplacian((20, 20, 20)), nested_dissection((20, 20, 20))),
    "natural2d_100": lambda: (laplacian((100, 100)), None),
    "chain100k": lambda: (chain(100_000), None),
}


def measure(name, repeats):
    a, perm = WORKLOADS[name]()
    a = sps.csr_matrix(a)
    a.sort_indices()
    n = a.shape[0]
    mat = sp.CsMat.new((n, n), a.indptr.astype(np.uint32), a.indices.astype(np.uint32), a.data)
    dev = mat.device()
    p = np.arange(n) if perm is None else perm
    t0 = time.perf_counter()
    sym = sp.ldl.LdlSymbolic.new_perm(dev, p, sp.ldl.SymmetryCheck.DontCheckSymmetry)
    t_sym = time.perf_counter() - t0
    print("%s: symbolic %.3f s" % (name, t_sym), file=sys.stderr, flush=True)
    t0 = time.perf_counter()
    num = sym.factor(dev)
    t_factor = time.perf_counter() - t0
    print("%s: factor %.3f s" % (name, t_factor), file=sys.stderr, flush=True)
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        num.update(dev)
        times.append(time.perf_counter() - t0)
    fa = LO.Factor(a.indptr, a.indices, perm)
    t0 = time.perf_counter()
    assert fa.update(a.data) is None
    t_oracle = time.perf_counter() - t0
    cp, li, lv = fa.l()
    c = np.diff(cp.astype(np.int64))
    flops = int(np.sum(c * (c - 1)) + 3 * int(cp[-1]))
    lm = num.l()
    parity_l = LO.first_difference(lm.data, lv) is None and np.array_equal(
        lm.indices.astype(np.uint64), li) and np.array_equal(lm.indptr.astype(np.uint64), cp)
    parity_d = LO.first_difference(num.d(), fa.diag()) is None
    ctx = dev.ctx
    b = np.random.default_rng(1).standard_normal(n)
    db = torch.from_numpy(b).to(G._device(ctx))
    dx = torch.empty_like(db)
    num.solve_dev(db.data_ptr(), dx.data_ptr())
    G._sync()
    t0 = time.perf_counter()
    want = fa.solve(b)
    t_oracle_solve = time.perf_counter() - t0
    parity_x = LO.first_difference(dx.cpu().numpy(), want) is None
    st = []
    for _ in range(max(repeats, 1)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        num.solve_dev(db.data_ptr(), dx.data_ptr())
        e1.record()
        e1.synchronize()
        st.append(e0.elapsed_time(e1) / 1e3)
    t_num = float(np.median(times)) if times else t_factor
    return dict(workload=name, n=n, nnz_a=int(a.nnz), nnz_l=int(cp[-1]), flops=flops,
                etree_height=fa.etree_height(), symbolic_s=round(t_sym, 4),
                factor_s=round(t_factor, 5), numeric_repeats=len(times),
                numeric_s=round(t_num, 5), numeric_gflops=round(flops / t_num / 1e9, 3),
                solve_s=round(float(np.median(st)), 5), oracle_numeric_s=round(t_oracle, 5),
                oracle_solve_s=round(t_oracle_solve, 5), parity_l=bool(parity_l),
                parity_d=bool(parity_d), parity_x=bool(parity_x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    names = args.only.split(",") if args.only else list(WORKLOADS)
    for name in names:
        print(json.dumps(measure(name, args.repeats)), flush=True)


if __name__ == "__main__":
    main()
