"""bench.py legs for the non-headline workloads of BASELINE.json:
  spmm_rand_1m_k64  (config 3)  CSR x dense C-order 1M x 64  -> csr_mulacc_dense_rowmaj
  spgemm_rmat_500k  (config 4)  two 500k x 500k R-MAT, ~16 nnz/row -> smmp::mul_csr_csr
Single GPU (the BASELINE configs are single-GPU); same JSON contract as bench.py."""
import ctypes as C
import json
import os
import statistics
import time

import numpy as np


def ncu_traffic(workload, world, source=False):
    """roofline.traffic: DRAM bytes (read + write) per launch of the dominant kernel as ncu
    measured them (profiles/ncu_traffic.json names the capture each number comes from);
    null when no capture of this workload / GPU count exists."""
    try:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "profiles",
                               "ncu_traffic.json")) as f:
            rec = json.load(f).get(workload)
    except (OSError, ValueError):
        return None
    if not rec or rec.get("n_gpus") != world:
        return None
    return rec["source"] if source else rec["bytes"]


def _cpu_spmm(a, b_t, budget_rows):
    from oracle import oracle as O
    import torch
    r1 = min(a.rows, budget_rows)
    e = int(a.indptr[r1].item())
    hip = a.indptr[:r1 + 1].cpu().numpy().view(np.uint32)
    hind = a.indices[:e].cpu().numpy().view(np.uint32)
    hdat = a.data[:e].cpu().numpy()
    hb = b_t.cpu().numpy()
    out = np.zeros((r1, hb.shape[1]))
    O.csr_mulacc_dense_rowmaj(hip, hind, hdat, hb, out)
    ts = []
    for _ in range(3):
        out[:] = 0
        t = time.perf_counter()
        O.csr_mulacc_dense_rowmaj(hip, hind, hdat, hb, out)
        ts.append(time.perf_counter() - t)
    t = statistics.median(ts)
    return {"value": 2.0 * e * hb.shape[1] / t / 1e9, "unit": "GFLOP/s", "cores": 1,
            "kind": "port", "sample": "first %d rows / %d nnz, 1 thread as in sprs, median of 3"
            % (r1, e), "host_cores": O.num_procs()}


def _cpu_spgemm(A, B, rows):
    from oracle import oracle as O
    r1 = min(A.rows, rows)
    e = int(A.indptr[r1].item())
    a = (A.indptr[:r1 + 1].cpu().numpy().view(np.uint32), A.indices[:e].cpu().numpy().view(np.uint32),
         A.data[:e].cpu().numpy())
    b = B.to_host()
    t = time.perf_counter()
    cip, cind, cd = O.mul_csr_csr((r1, A.cols), a, (B.rows, B.cols), b, threads=0)
    dt = time.perf_counter() - t
    nprod = int(np.sum(np.diff(b[0].astype(np.int64))[a[1]]))
    return {"value": 2.0 * nprod / dt / 1e9, "unit": "GFLOP/s", "cores": O.num_procs(),
            "kind": "port", "sample": "first %d rows of A (n_prod %d, nnzC %d), sprs thread rule "
            "(Automatic: min(rows, (nnzA+nnzB)/8128, ncpu)), 1 run" % (r1, nprod, len(cind))}


def dump_csr_rows(out_dir, ctx, cm, rows, dev, budget, seed):
    """--dump-outputs of the SpGEMM leg: whole rows of the product mirror `cm`, a fixed, seeded
    sample of them within `budget` bytes, in row order, as float64 arrays c_rows (row numbers),
    c_indptr (offsets into the sample) and c_indices / c_data (the rows' entries)."""
    import types
    import torch
    import bench as B
    from sprs_b200 import generate as G
    d_ip, d_ind, d_dat, ipb = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
    ctx.check(ctx.lib.sprs_b200_csmat_device_arrays(cm, C.byref(d_ip), C.byref(ipb), C.byref(d_ind),
                                                    C.byref(d_dat)))
    ip = torch.as_tensor(G._DevArray(d_ip.value, rows + 1, "<i4" if ipb.value == 4 else "<i8"),
                         device=dev)
    nnz = G.u32(ip[-1]) if ipb.value == 4 else int(ip[-1].item())
    c = types.SimpleNamespace(indptr=ip,
                              indices=torch.as_tensor(G._DevArray(d_ind.value, nnz, "<i4"), device=dev),
                              data=torch.as_tensor(G._DevArray(d_dat.value, nnz, "<f8"), device=dev))
    lens = np.diff(ip.cpu().numpy().view(np.uint32 if ipb.value == 4 else np.int64).astype(np.int64))
    order = np.random.default_rng(seed).permutation(rows)
    cost = np.cumsum(16 + 16 * lens[order])  # row number + offset, index + value per entry
    sel = np.sort(order[:int(np.searchsorted(cost, budget, side="right"))])
    sub_ip, ind, dat = B.rows_to_host(c, torch.from_numpy(sel).to(dev))
    os.makedirs(out_dir, exist_ok=True)
    for name, arr in (("c_rows", sel), ("c_indptr", sub_ip), ("c_indices", ind), ("c_data", dat)):
        np.save(os.path.join(out_dir, name + ".npy"), arr.astype(np.float64))


def run(args, ctx, kind, n, npr, gen, seed):
    import torch
    from sprs_b200 import generate as G
    import bench as B
    peaks, peak_src = B.measured_peaks()
    hbm = float(peaks["hbm_gbs"])
    dev = torch.device("cuda", ctx.device)
    sampler = B.ClockSampler(ctx.device)
    warm = max(args.warmup, 3)
    if kind == "spmm":
        k = 64
        a = G.make_matrix(ctx, gen, n, npr, seed)
        b = torch.randn(n, k, device=dev, dtype=torch.float64)
        c = torch.empty(n, k, device=dev, dtype=torch.float64)
        for _ in range(warm):
            G.spmm_rowmaj(ctx, a, b, c)
        torch.cuda.synchronize()
        sampler.start()
        l0 = ctx.launches
        tw0 = time.time()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            G.spmm_rowmaj(ctx, a, b, c)
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop(tw0, time.time())
        ms = e0.elapsed_time(e1) / args.steps
        if args.dump_outputs:
            B.dump_rows(args.dump_outputs, "c", c)
        flops = 2.0 * a.nnz * k
        comp_bytes = 12.0 * a.nnz + 8.0 * k * (n + n)
        # e2e: host B (pinned) in, host C out through the reference-facing call
        hb = torch.empty(n, k, dtype=torch.float64).pin_memory()
        hb.copy_(b)
        hc = torch.zeros(n, k, dtype=torch.float64).pin_memory()
        t0 = time.perf_counter()
        reps = 3
        for _ in range(reps):
            ctx.check(ctx.lib.sprs_b200_csr_mulacc_dense_rowmaj(
                ctx.h, a.mirror.h, C.c_void_p(hb.data_ptr()), n, k, k, 1,
                C.c_void_p(hc.data_ptr()), n, k, k, 1))
        e2e_ms = (time.perf_counter() - t0) * 1e3 / reps
        line = {"metric": "csr_spmm_f64_gflops", "value": flops / ms / 1e6, "unit": "GFLOP/s",
                "n_gpus": 1, "steps": args.steps, "warmup": warm, "ms_per_step": ms,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
                "data": "synthetic",
                "config": {"workload": args.workload, "n": n, "nnz": a.nnz, "k": k,
                           "layout": "B, C row-major (csr_mulacc_dense_rowmaj)",
                           "l2_policy": "inputs (1.4 GB) exceed L2; no flush needed"},
                "roofline": {"bound": "hbm", "achieved": comp_bytes / ms / 1e6, "peak": hbm,
                             "unit": "GB/s", "frac": comp_bytes / ms / 1e6 / hbm,
                             "traffic": ncu_traffic(args.workload, 1),
                             "kernel": "spmm_rowmaj_kernel", "peak_source": peak_src,
                             "algorithmic_bytes": "compulsory 12*nnz + 8*k*(cols+rows)"},
                "e2e": {"value": flops / e2e_ms / 1e6, "unit": "GFLOP/s", "ms_per_step": e2e_ms,
                        "h2d_bytes_per_step": 16 * n * k, "d2h_bytes_per_step": 8 * n * k,
                        "api": "sprs_b200_csr_mulacc_dense_rowmaj (host views)"},
                "gpu_launches": ctx.launches - l0, "clocks": clocks}
        if not args.no_cpu_baseline:
            line["cpu_baseline"] = _cpu_spmm(a, b, 100_000)
        print(json.dumps(line))
        return
    # ---- spgemm
    A = G.rmat_csr(ctx, n, npr, seed=seed)
    Bm = G.rmat_csr(ctx, n, npr, seed=seed ^ 0x1000)
    lib = ctx.lib

    def once(keep=False, keep_c=False):
        plan, nnz_c, cm = C.c_void_p(), C.c_uint64(), C.c_void_p()
        ctx.check(lib.sprs_b200_spgemm_symbolic(ctx.h, A.mirror.h, Bm.mirror.h, C.byref(plan),
                                                C.byref(nnz_c)))
        ctx.check(lib.sprs_b200_spgemm_numeric_dev(ctx.h, plan, C.byref(cm)))
        nprod = lib.sprs_b200_spgemm_nprod(plan) if keep else 0
        lib.sprs_b200_spgemm_free(plan)
        if keep_c:
            return nnz_c.value, cm
        lib.sprs_b200_csmat_free(cm)
        return nnz_c.value, nprod
    nnz_c, nprod = once(keep=True)
    for _ in range(max(1, warm - 1)):
        once()
    sampler.start()
    l0 = ctx.launches
    tw0 = time.time()
    t0 = time.perf_counter()
    steps = args.steps
    for i in range(steps):
        # the C-ABI calls are synchronous (they return nnz / a finished mirror); the last
        # product is kept for --dump-outputs
        last = once(keep_c=bool(args.dump_outputs) and i == steps - 1)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    clocks = sampler.stop(tw0, time.time())
    if args.dump_outputs:
        dump_csr_rows(args.dump_outputs, ctx, last[1], n, dev, B.DUMP_BUDGET, B.DUMP_SEED)
        lib.sprs_b200_csmat_free(last[1])
    alg = 12.0 * (A.nnz + nprod + nnz_c) + 8.0 * (n + 1)
    line = {"metric": "csr_spgemm_f64_gflops", "value": 2.0 * nprod / ms / 1e6, "unit": "GFLOP/s",
            "n_gpus": 1, "steps": steps, "warmup": warm, "ms_per_step": ms,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "synthetic",
            "config": {"workload": args.workload, "n": n, "nnzA": A.nnz, "nnzB": Bm.nnz,
                       "n_prod": nprod, "nnzC": nnz_c, "compression": nprod / max(nnz_c, 1),
                       "timing": "host clock around symbolic+numeric (both synchronous), C "
                                 "left on the device"},
            "roofline": {"bound": "hbm", "achieved": alg / ms / 1e6, "peak": hbm, "unit": "GB/s",
                         "frac": alg / ms / 1e6 / hbm, "traffic": None,
                         "kernel": "spgemm symbolic+numeric (whole call)",
                         "peak_source": peak_src,
                         "algorithmic_bytes": "12*(nnzA + n_prod + nnzC) + 8*(n+1)"},
            "e2e": {"value": 2.0 * nprod / ms / 1e6, "unit": "GFLOP/s", "ms_per_step": ms,
                    "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                    "note": "operands resident as mirrors; result kept on device"},
            "gpu_launches": ctx.launches - l0, "clocks": clocks}
    if not args.no_cpu_baseline:
        line["cpu_baseline"] = _cpu_spgemm(A, Bm, 20_000)
    print(json.dumps(line))


def extra_spmm(ctx, G, hbm, dev):
    """BASELINE config 3 as a compact entry of the default line's "extra" (the driver only runs
    the default command): device-timed ms, GFLOP/s, fraction of the compulsory roofline, and a
    bit-exactness check of sampled C rows against the oracle (csr_mulacc_dense_rowmaj)."""
    import torch
    from oracle import oracle as O
    n, k = 1_000_000, 64
    a = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
    b = torch.randn(n, k, device=dev, dtype=torch.float64)
    c = torch.empty(n, k, device=dev, dtype=torch.float64)
    for _ in range(3):
        G.spmm_rowmaj(ctx, a, b, c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = 10
    e0.record()
    for _ in range(steps):
        G.spmm_rowmaj(ctx, a, b, c)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    comp = 12.0 * a.nnz + 8.0 * k * (n + n)
    # parity: the first 2000 rows, bit-exact (sequential unfused sums, prod.rs:189-214)
    r1 = 2000
    e = int(a.indptr[r1].item())
    hip = a.indptr[:r1 + 1].cpu().numpy().view(np.uint32)
    hind = a.indices[:e].cpu().numpy().view(np.uint32)
    hdat = a.data[:e].cpu().numpy()
    ref = np.zeros((r1, k))
    O.csr_mulacc_dense_rowmaj(hip, hind, hdat, b.cpu().numpy(), ref)
    return {"nnz": a.nnz, "k": k, "ms": ms, "gflops": 2.0 * a.nnz * k / ms / 1e6,
            "frac_of_compulsory_roofline": comp / ms / 1e6 / hbm,
            "traffic": ncu_traffic("spmm_rand_1m_k64", 1),
            "parity_vs_oracle": {"bit_exact": bool(np.array_equal(c[:r1].cpu().numpy(), ref)),
                                 "rows_checked": r1}}


def extra_spgemm(ctx, G, hbm, dev):
    """BASELINE config 4 as a compact entry of "extra": host-timed symbolic + numeric (both
    synchronous C-ABI calls, C left on the device), and indptr / indices of a row block of the
    product checked BIT-EXACT against the oracle (smmp.rs:81-189)."""
    import torch
    from oracle import oracle as O
    n = 500_000
    A = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    Bm = G.rmat_csr(ctx, n, 16, seed=0x5EED0004 ^ 0x1000)
    lib = ctx.lib

    def once(keep=False):
        plan, nnz_c, cm = C.c_void_p(), C.c_uint64(), C.c_void_p()
        ctx.check(lib.sprs_b200_spgemm_symbolic(ctx.h, A.mirror.h, Bm.mirror.h, C.byref(plan),
                                                C.byref(nnz_c)))
        ctx.check(lib.sprs_b200_spgemm_numeric_dev(ctx.h, plan, C.byref(cm)))
        nprod = lib.sprs_b200_spgemm_nprod(plan) if keep else 0
        lib.sprs_b200_spgemm_free(plan)
        if keep:
            return nnz_c.value, nprod, cm
        lib.sprs_b200_csmat_free(cm)
        return nnz_c.value, nprod, None
    nnz_c, nprod, cm = once(keep=True)
    # parity on rows [r0, r1) of C against the oracle's product of that row block of A with B
    r0, r1 = 1000, 1400
    d_ip, d_ind, d_dat, ipb = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
    ctx.check(lib.sprs_b200_csmat_device_arrays(cm, C.byref(d_ip), C.byref(ipb), C.byref(d_ind),
                                                C.byref(d_dat)))
    cip = torch.as_tensor(G._DevArray(d_ip.value, n + 1, "<i4" if ipb.value == 4 else "<i8"),
                          device=dev).to(torch.int64)
    if ipb.value == 4:
        cip &= 0xFFFFFFFF
    s, e = int(cip[r0].item()), int(cip[r1].item())
    got_ip = (cip[r0:r1 + 1] - s).cpu().numpy()
    got_ind = torch.as_tensor(G._DevArray(d_ind.value + 4 * s, e - s, "<i4"),
                              device=dev).cpu().numpy().view(np.uint32)
    blk = A.slice_rows(r0, r1)
    a_host, b_host = blk.to_host(), Bm.to_host()
    t_cpu = time.perf_counter()
    oip, oind, _ = O.mul_csr_csr((r1 - r0, n), a_host, (n, n), b_host, threads=0)
    t_cpu = time.perf_counter() - t_cpu
    try:  # the same call, timed: the CPU port beside the GPU number (a reported baseline only)
        b_len = np.diff(b_host[0].astype(np.int64))
        nprod_blk = int(b_len[a_host[1].astype(np.int64)].sum())
        cpu = {"value": 2.0 * nprod_blk / t_cpu / 1e9, "unit": "GFLOP/s", "kind": "port",
               "threads": "the reference's Automatic rule (smmp.rs:210-227)",
               "sample": "rows %d..%d of A times B: %d products" % (r0, r1, nprod_blk)}
    except Exception as e:
        cpu = {"error": repr(e)}
    parity = {"rows_checked": r1 - r0, "nnz_checked": int(e - s),
              "indptr_bit_exact": bool(np.array_equal(got_ip, np.asarray(oip, dtype=np.int64))),
              "indices_bit_exact": bool(np.array_equal(got_ind, np.asarray(oind, dtype=np.uint32)))}
    lib.sprs_b200_csmat_free(cm)
    del blk
    once()
    t0 = time.perf_counter()
    steps = 3
    for _ in range(steps):
        once()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    alg = 12.0 * (A.nnz + nprod + nnz_c) + 8.0 * (n + 1)
    return {"n_prod": nprod, "nnzC": nnz_c, "ms": ms, "gflops": 2.0 * nprod / ms / 1e6,
            "frac_of_roofline": alg / ms / 1e6 / hbm, "parity_vs_oracle": parity,
            "cpu_baseline": cpu,
            "timing": "host clock around symbolic + numeric (synchronous calls), C left on the device"}
