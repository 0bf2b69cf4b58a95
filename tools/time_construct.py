"""Times the device construction (csrc/construct.cu) on the project's workloads: one JSON line each.

    python tools/time_construct.py [--calls 10] [--warmup 2] [--only vstack_rmat10m_7,...] [--out DIR]

Workloads (every input built on the device with sprs_b200.generate):
  vstack_rmat10m_7   config 5 (10M x 10M R-MAT, 10^9 non-zeros) cut into 7 uneven row slices,
                     vstack-ed back
  hstack_rand1m      two config-2 CSR matrices (seeds 0x5EED0002, 0x5EED1002) hstack-ed: a CSC
                     result, the two CSR -> CSC conversions included in the call
  bmat_kkt           [[H, J^T], [J, None]]: H = config 2, J a 500k x 1M sprs-rand matrix with 16
                     non-zeros per row and J^T its transpose view (its conversion in the call)
  kron_lap2d_2000    kron(I, T) and kron(T, I), T the 2000 x 2000 second-difference matrix
  kron_rmat500k_x4   kron(config-4 R-MAT, dense random 4x4): every output row 4x an R-MAT row
  kron_x4_rmat500k   kron(dense random 4x4, config-4 R-MAT): the skewed rows in 4 copies

Each line: nnz in and out; the call time (host clock around the blocking call, which ends in a
stream synchronise), median and min over --calls calls after --warmup; the kernel time of one
call in a separate torch.profiler run, all kernels and the construction kernels alone (indptr
and fill: `bmat_*` / `kron_*`); the algorithmic bytes -- stacks: 12 B read and written per
non-zero plus every input and the output indptr; Kron: 12 nnzC + wC (outerC + 1) written plus
the compulsory reads of both operands -- and the construction kernels' share of 3.35 TB/s; the
single-thread oracle time (tests/construct_oracle.cpp) and a parity flag from the bit-exact
comparison of the whole output (vstack_rmat10m_7: against config 5 itself, no oracle); GPU name,
power limit and SM clock read in the same process.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12
NAMES = ("vstack_rmat10m_7", "hstack_rand1m", "bmat_kkt", "kron_lap2d_2000", "kron_rmat500k_x4",
         "kron_x4_rmat500k")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (reported, not fatal)
        return {"gpu": "unknown (%s)" % e}


def host(m):
    """oracle Mat of a DeviceCsr or of a result (mirror, indptr, indices, data)"""
    import construct_oracle as CO
    if isinstance(m, tuple):
        mirror, ip, ind, dat = m
        storage, shape = mirror.storage, (mirror.rows, mirror.cols)
    else:
        storage, shape, ip, ind, dat = "CSR", (m.rows, m.cols), m.indptr, m.indices, m.data
    ip = ip.cpu().numpy()
    ip = ip.view(np.uint32) if ip.dtype == np.int32 else ip
    return CO.mat(storage, shape, ip, ind.cpu().numpy().view(np.uint32), dat.cpu().numpy())


def dense4(sp, ctx):
    rng = np.random.default_rng(0x4A4)
    d = sp.CsMat.new((4, 4), np.arange(0, 17, 4), np.tile(np.arange(4), 4), rng.standard_normal(16))
    d._ctx = ctx
    return d.device()


def second_difference(sp, ctx, n):
    ip = np.concatenate([[0], np.cumsum([2] + [3] * (n - 2) + [2])])
    ind = np.concatenate([[0, 1]] + [[i - 1, i, i + 1] for i in range(1, n - 1)] + [[n - 2, n - 1]])
    dat = np.concatenate([[2., -1.]] + [[-1., 2., -1.]] * (n - 2) + [[-1., 2.]])
    t = sp.CsMat.new((n, n), ip, ind, dat)
    t._ctx = ctx
    e = sp.CsMat.eye(n)
    e._ctx = ctx
    return e.device(), t.device()


def workload(sp, ctx, name):
    """(call, inputs for the byte count, oracle thunk or None, keepalive).  call() returns the
    result mirror(s) of one timed call."""
    from sprs_b200 import construct as K, generate as G
    if name == "vstack_rmat10m_7":
        n = 10_000_000
        a = G.rmat_csr(ctx, n, 100, seed=0x5EED0005)
        cuts = [0, 1, 1_234_567, 3_000_000, 3_000_000, 6_500_001, 9_999_999, n]
        slices = [a.slice_rows(r0, r1) for r0, r1 in zip(cuts[:-1], cuts[1:])]
        return (lambda: [K.bmat_dev(ctx, [[s.mirror] for s in slices])], slices, None, a)
    if name == "hstack_rand1m":
        n = 1_000_000
        a = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
        b = G.rand_csr(ctx, n, n, 32, seed=0x5EED1002)

        def call():
            tv = [K.transpose_view_dev(ctx, m.mirror) for m in (a, b)]
            return [K.transpose_view_dev(ctx, K.bmat_dev(ctx, [[v] for v in tv]))]
        import construct_oracle as CO
        return (call, [a, b], lambda: CO.hstack([host(a), host(b)]), None)
    if name == "bmat_kkt":
        n = 1_000_000
        h = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
        j = G.rand_csr(ctx, n // 2, n, 16, seed=0x5EED2002)

        def call():
            jt = K.transpose_view_dev(ctx, j.mirror)
            return [K.bmat_dev(ctx, [[h.mirror, jt], [j.mirror, None]])]
        import construct_oracle as CO
        return (call, [h, j, j], lambda: CO.bmat([[host(h), CO.transpose_view(host(j))],
                                                  [host(j), None]]), None)
    if name == "kron_lap2d_2000":
        e, t = second_difference(sp, ctx, 2000)
        import construct_oracle as CO
        he = CO.mat("CSR", (2000, 2000), *e.download(np.uint64))
        ht = CO.mat("CSR", (2000, 2000), *t.download(np.uint64))
        return (lambda: [K.kron_dev(ctx, e, t), K.kron_dev(ctx, t, e)], [(e, t), (t, e)],
                lambda: [CO.kronecker_product(he, ht), CO.kronecker_product(ht, he)], None)
    a = G.rmat_csr(ctx, 500_000, 16, seed=0x5EED0004)
    d = dense4(sp, ctx)
    import construct_oracle as CO
    hd = CO.mat("CSR", (4, 4), *d.download(np.uint64))
    if name == "kron_rmat500k_x4":
        return (lambda: [K.kron_dev(ctx, a.mirror, d)], [(a.mirror, d)],
                lambda: [CO.kronecker_product(host(a), hd)], a)
    return (lambda: [K.kron_dev(ctx, d, a.mirror)], [(d, a.mirror)],
            lambda: [CO.kronecker_product(hd, host(a))], a)


def _ipw(m):
    d, ipb = C.c_void_p(), C.c_int()
    m.ctx.check(m.ctx.lib.sprs_b200_csmat_device_arrays(m.h, C.byref(d), C.byref(ipb), C.byref(d),
                                                        C.byref(d)))
    return ipb.value


def _outer(m):
    return m.rows if m.storage == "CSR" else m.cols


def algorithmic_bytes(name, inputs, results):
    out = sum(12 * r.nnz + _ipw(r) * (_outer(r) + 1) for r in results)
    if name.startswith("kron"):
        rd = sum(12 * (x.nnz + y.nnz) + _ipw(x) * (_outer(x) + 1) + _ipw(y) * (_outer(y) + 1)
                 for x, y in inputs)
    else:
        rd = sum(12 * m.nnz + m.indptr.element_size() * (m.rows + 1) for m in inputs)
    return rd + out


def run(sp, ctx, name, args):
    import torch
    from sprs_b200 import generate as G
    call, inputs, oracle, keep = workload(sp, ctx, name)
    G._sync()
    for _ in range(args.warmup):
        for m in call():
            m.free()
    times = []
    for _ in range(args.calls):
        t0 = time.perf_counter()
        res = call()
        times.append((time.perf_counter() - t0) * 1e3)
        for m in res:
            m.free()
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(3):  # a profiler run now and then records none of the call's kernels
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = call()
        kernels = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                kernels[e.name] = kernels.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
        construct_ms = sum(v for k, v in kernels.items() if "bmat_" in k or "kron_" in k)
        if construct_ms or attempt == 2:
            break
        for m in res:
            m.free()
    kernel_ms = sum(kernels.values())
    nbytes = algorithmic_bytes(name, inputs, res)
    views = [G._with_views(ctx, m) for m in res]
    oracle_ms = None
    if oracle is None:  # vstack of config 5's slices: the result is config 5
        ok = all(torch.equal(p.view(torch.int64) if p.dtype == torch.float64 else p,
                             q.view(torch.int64) if q.dtype == torch.float64 else q)
                 for p, q in zip(views[0][1:], (keep.indptr, keep.indices, keep.data)))
        err = None if ok else "differs from config 5"
    else:
        import construct_oracle as CO
        t0 = time.perf_counter()
        want = oracle()
        oracle_ms = (time.perf_counter() - t0) * 1e3
        want = want if isinstance(want, list) else [want]
        err = None
        for v, w in zip(views, want):
            err = err or CO.first_difference(host(v), w, kron=name.startswith("kron"))
    line = {"workload": name, "nnz_in": sum(m.nnz for m in inputs) if not name.startswith("kron")
            else sum(x.nnz + y.nnz for x, y in inputs), "nnz_out": sum(r.nnz for r in res),
            "call_ms_median": round(statistics.median(times), 3), "call_ms_min": round(min(times), 3),
            "calls": args.calls, "kernel_ms": round(kernel_ms, 3),
            "construct_kernel_ms": round(construct_ms, 3),
            "kernels_ms": {k[:80]: round(v, 3) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])},
            "call_fraction_of_3.35TBps": round(nbytes / HBM_BPS * 1e3 / min(times), 3),
            "algorithmic_bytes": nbytes, "roofline_ms": round(nbytes / HBM_BPS * 1e3, 3),
            "construct_fraction_of_3.35TBps": round(nbytes / HBM_BPS * 1e3 / construct_ms, 3)
            if construct_ms else None,
            "oracle_single_thread_ms": round(oracle_ms, 1) if oracle_ms is not None else None,
            "parity": "ok" if err is None else "FAIL: " + err}
    line.update(gpu_info())
    del views, res, inputs, keep
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=",".join(NAMES))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import sprs_b200 as sp
    ctx = sp.Context.default()
    lines = []
    for name in args.only.split(","):
        line = run(sp, ctx, name, args)
        print(json.dumps(line), flush=True)
        lines.append(line)
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_construct.jsonl"), "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)
    return 0 if all(x["parity"] == "ok" for x in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
