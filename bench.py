#!/usr/bin/env python
"""bench.py -- headline benchmark of the sprs product path on H100.

Metric (BASELINE.json): CSR SpMV f64 GFLOP/s and achieved fraction of the HBM roofline
(2*nnz flops over 12*nnz + 8*n bytes), at 1/2/4/8 H100, beside the sprs CPU path.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--workload NAME] [--impl reference]
                  [--dump-outputs DIR]

--dump-outputs DIR writes what the timed path returned in its last timed step as DIR/<name>.npy
(float64; a fixed, seeded sample of rows when the whole result exceeds 64 MB), so that two builds
can be compared output for output: the inputs are seeded and identical from run to run.

A "step" is one `y = A x` over the whole matrix (all ranks together).  The default
workload is BASELINE config 5 -- the configuration the metric is quoted on: 10M x 10M
R-MAT, ~100 nnz/row (~1e9 nnz, 12 GB, fits one GPU) -- at every N (strong scaling:
contiguous cost-balanced row blocks per rank, x replicated, all-gather of y over NVLink
through the library's own communicator, include/sprs_b200.h).
Other workloads: spmv_rand_1m (config 2), spmm_rand_1m_k64 (config 3),
spgemm_rmat_500k (config 4); at N=1 the default run also reports them under "extra".
One JSON line is printed by rank 0.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_other  # noqa: E402  (needs ROOT on sys.path; imports nothing heavy)

WORKLOADS = {
    # name: (kind, n, nnz_per_row, generator)
    "spmv_rmat_10m": ("spmv", 10_000_000, 100, "rmat"),
    "spmv_rand_1m": ("spmv", 1_000_000, 32, "rand"),
    "spmm_rand_1m_k64": ("spmm", 1_000_000, 32, "rand"),
    "spgemm_rmat_500k": ("spgemm", 500_000, 16, "rmat"),
    # small variant for quick checks and the CPU dry run
    "spmv_rmat_1m": ("spmv", 1_000_000, 100, "rmat"),
}
SEEDS = {"spmv_rmat_10m": 0x5EED0005, "spmv_rand_1m": 0x5EED0002, "spmm_rand_1m_k64": 0x5EED0002,
         "spgemm_rmat_500k": 0x5EED0004, "spmv_rmat_1m": 0x5EED0005}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return json.load(f), "measured (MEASURED_PEAKS.json)"
    return {"hbm_gbs": 3350.0}, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3)"


DUMP_BUDGET = 60_000_000  # bytes of array data --dump-outputs writes, all files together
DUMP_SEED = 0x5EED0D0


def dump_rows(out_dir, name, t, budget=DUMP_BUDGET):
    """Write a device or host array `t` (1-D, or 2-D row-major) to out_dir/<name>.npy in float64:
    all of it when it fits `budget` bytes, else a fixed, seeded sample of its rows, with the
    sampled row numbers (as float64) in <name>_rows.npy."""
    import torch
    os.makedirs(out_dir, exist_ok=True)
    rows = t.shape[0]
    row_bytes = 8 * (t[0].numel() if rows and t.dim() > 1 else 1)
    if rows * row_bytes <= budget:
        np.save(os.path.join(out_dir, name + ".npy"), t.detach().cpu().numpy().astype(np.float64))
        return
    k = budget // (row_bytes + 8)
    sel = np.sort(np.random.default_rng(DUMP_SEED).choice(rows, size=k, replace=False))
    idx = torch.from_numpy(sel).to(t.device)
    np.save(os.path.join(out_dir, name + ".npy"), t[idx].cpu().numpy().astype(np.float64))
    np.save(os.path.join(out_dir, name + "_rows.npy"), sel.astype(np.float64))


class ClockSampler:
    """SM clocks / throttle reasons sampled DURING the timed region (NVML, every 2 ms;
    same fields as the profiling recipe's nvidia-smi clocks line)."""

    def __init__(self, device):
        self.device, self.samples, self.stop_flag, self.t = device, [], False, None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            idx = device
            if vis:
                try:
                    idx = int(vis.split(",")[device])
                except ValueError:
                    idx = device
            self.h = pynvml.nvmlDeviceGetHandleByIndex(idx)
            self.max = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception as e:
            self.nv, self.err = None, repr(e)

    def _loop(self):
        nv = self.nv
        while not self.stop_flag:
            try:
                sm = nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)
                try:
                    rs = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    rs = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                pw = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
                self.samples.append((time.time(), sm, rs, pw))
            except Exception:
                pass
            time.sleep(0.002)

    def start(self):
        if self.nv:
            self.t = threading.Thread(target=self._loop, daemon=True)
            self.t.start()

    def stop(self, t0, t1):
        if not self.nv:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvml unavailable: " + self.err]}
        self.stop_flag = True
        self.t.join()
        inside = [s for s in self.samples if t0 <= s[0] <= t1] or self.samples[-3:]
        bits = 0
        for s in inside:
            bits |= s[2]
        names = {"hw_slowdown": 0x8, "sw_power_cap": 0x4, "hw_thermal_slowdown": 0x40,
                 "sw_thermal_slowdown": 0x20, "hw_power_brake": 0x80, "sync_boost": 0x10,
                 "applications_clocks_setting": 0x2}
        return {"sm_mhz": statistics.median([s[1] for s in inside]) if inside else None,
                "sm_max_mhz": self.max, "reasons": sorted(k for k, v in names.items() if bits & v),
                "power_w_max": max([s[3] for s in inside]) if inside else None,
                "samples": len(inside)}


def rows_to_host(a, rows_t):
    """Host CSR (uint32 indptr / indices, f64 data) of the given SORTED rows of a DeviceCsr."""
    import torch
    ip = a.indptr.to(torch.int64) & 0xFFFFFFFF  # int32 storage of u32 values
    starts = ip[rows_t]
    lens = ip[rows_t + 1] - starts
    sub_ip = torch.zeros(rows_t.numel() + 1, dtype=torch.int64, device=ip.device)
    torch.cumsum(lens, 0, out=sub_ip[1:])
    total = int(sub_ip[-1].item())
    pos = (torch.arange(total, device=ip.device, dtype=torch.int64)
           - torch.repeat_interleave(sub_ip[:-1], lens) + torch.repeat_interleave(starts, lens))
    hind = a.indices[pos].cpu().numpy().view(np.uint32)
    hdat = a.data[pos].cpu().numpy()
    return sub_ip.cpu().numpy().astype(np.uint32), hind, hdat


def parity_vs_oracle(full, x, y, n_random=10000, n_heavy=100, seed=1234):
    """UNTIMED check of a device result against the CPU oracle (the reference's loop,
    oracle/sprs_oracle.cpp after prod.rs:274-298) on the heaviest rows plus a random sample of
    the WHOLE y this rank holds (at N > 1: the all-gathered vector, rows of every rank's block).
    Gate: |got - ref| <= 1e-6 * sum|terms| per row (SURVEY 8d).  Returns (ok, rows, max ratio of
    |got - ref| to the gate)."""
    import torch
    from oracle import oracle as O
    n = full.rows
    ip = full.indptr.to(torch.int64) & 0xFFFFFFFF
    lens = ip[1:] - ip[:-1]
    heavy = torch.topk(lens, min(n_heavy, n)).indices
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    rnd = torch.randint(0, n, (min(n_random, n),), generator=g).to(ip.device)
    rows_t = torch.unique(torch.cat([heavy, rnd]))
    hip, hind, hdat = rows_to_host(full, rows_t)
    hx = x.cpu().numpy()
    ref, bound = np.zeros(rows_t.numel()), np.zeros(rows_t.numel())
    O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, ref)
    O.mul_acc_mat_vec_csr(hip, hind, np.abs(hdat), np.abs(hx), bound)
    got = y[rows_t].cpu().numpy()
    ratio = np.abs(got - ref) / (1e-6 * bound + 1e-300)
    worst = float(np.nanmax(ratio)) if ratio.size else 0.0
    ok = bool(np.all(np.isfinite(got)) and worst <= 1.0)
    return ok, int(rows_t.numel()), worst


def sample_rows_to_host(a, target_nnz, nblocks=8):
    """A bounded sample of the SAME matrix for the CPU baseline: `nblocks` contiguous row
    blocks spread over the matrix, ~target_nnz non-zeros in total, as one host CSR."""
    import torch
    ip = a.indptr.to(torch.int64) & 0xFFFFFFFF
    n = a.rows
    per = max(1, target_nnz // nblocks)
    parts_ip, parts_ind, parts_dat, total, rows = [np.zeros(1, np.int64)], [], [], 0, 0
    for b in range(nblocks):
        r0 = (n * b) // nblocks
        s = int(ip[r0])
        r1 = int(torch.searchsorted(ip, torch.tensor([s + per], device=ip.device))[0])
        r1 = max(r0 + 1, min(r1, (n * (b + 1)) // nblocks))
        e = int(ip[r1])
        parts_ip.append((ip[r0 + 1:r1 + 1] - s + total).cpu().numpy())
        parts_ind.append(a.indices[s:e].cpu().numpy().view(np.uint32))
        parts_dat.append(a.data[s:e].cpu().numpy())
        total += e - s
        rows += r1 - r0
    return (np.concatenate(parts_ip).astype(np.uint32), np.concatenate(parts_ind),
            np.concatenate(parts_dat), rows)


def cpu_spmv_baseline(a, x_t, budget_nnz):
    """Faithful CPU restatement (oracle port), 1 thread -- sprs SpMV is single-threaded
    (SURVEY F6) -- on a bounded sample of the same matrix; plus the all-cores row-chunked
    extension, labelled as not in the reference."""
    from oracle import oracle as O
    hip, hind, hdat, rows = sample_rows_to_host(a, budget_nnz)
    hx = x_t.cpu().numpy()
    nnz = int(hip[-1])
    y = np.zeros(rows)
    O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, y)  # warm-up (page-in)
    ts = []
    for _ in range(3):
        y[:] = 0
        t = time.perf_counter()
        O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, y)
        ts.append(time.perf_counter() - t)
    t1 = statistics.median(ts)
    cores = O.num_procs()
    ts = []
    for _ in range(3):
        y[:] = 0
        t = time.perf_counter()
        O.ext_spmv_csr_omp(hip, hind, hdat, hx, y, cores)
        ts.append(time.perf_counter() - t)
    tn = statistics.median(ts)
    return {"value": 2.0 * nnz / t1 / 1e9, "unit": "GFLOP/s", "cores": 1, "kind": "port",
            "sample": "%d rows / %d nnz of the same matrix (8 row blocks), 1 thread as in sprs "
                      "(SpMV is single-threaded there), median of 3" % (rows, nnz),
            "ext_all_cores": {"value": 2.0 * nnz / tn / 1e9, "cores": cores,
                              "note": "OpenMP row-chunked extension -- NOT in the reference"},
            "host_cores": cores}


# ---- reference arm -------------------------------------------------------------------
def generate_to_dir(workload, out_dir):
    """Child-process entry (`bench.py --gen-to DIR`): builds the workload's matrix and x with the
    device generator and leaves them as .npy files, so that the reference arm's own process
    never maps the product library."""
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    kind, n, npr, gen = WORKLOADS[workload]
    ctx = sp.Context.default(0)
    torch.cuda.set_device(0)
    a = G.make_matrix(ctx, gen, n, npr, SEEDS[workload])
    x = G.normal_vector(ctx, n)
    np.save(os.path.join(out_dir, "indptr.npy"), a.indptr.cpu().numpy().view(np.uint32))
    np.save(os.path.join(out_dir, "indices.npy"), a.indices.cpu().numpy().view(np.uint32))
    np.save(os.path.join(out_dir, "data.npy"), a.data.cpu().numpy())
    np.save(os.path.join(out_dir, "x.npy"), x.cpu().numpy())


def run_reference(args):
    """--impl reference: the reference's CPU implementation of the path (oracle port of
    prod.rs:274-298; the Rust reference cannot be built here), on the box's host cores, same
    metric, the WHOLE matrix of the same config every step.  The inputs come from a child
    process (the device generator) through /dev/shm files: this process loads oracle/ only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    kind, n, npr, gen = WORKLOADS[args.workload]
    from oracle import oracle as O
    tmp_root = "/dev/shm" if os.path.isdir("/dev/shm") else None
    tmp = tempfile.mkdtemp(prefix="sprs_b200_ref_", dir=tmp_root)
    src = "device generator in a child process, handed over as .npy files (%s)" % tmp
    try:
        env = dict(os.environ)
        for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
            env.pop(k, None)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--gen-to", tmp,
                            "--workload", args.workload], env=env, capture_output=True, text=True,
                           timeout=900)
        if r.returncode != 0:
            raise RuntimeError(r.stderr[-300:])
        hip = np.load(os.path.join(tmp, "indptr.npy"))
        hind = np.load(os.path.join(tmp, "indices.npy"))
        hdat = np.load(os.path.join(tmp, "data.npy"))
        hx = np.load(os.path.join(tmp, "x.npy"))
        rows, whole = n, True
    except Exception as e:  # no GPU for the generator: uniform random stand-in of the same shape
        rng = np.random.default_rng(SEEDS[args.workload])
        rows = (1 << 24) // npr
        hind = rng.integers(0, n, size=rows * npr, dtype=np.uint32).reshape(rows, npr)
        hind.sort(axis=1)
        hind = hind.reshape(-1)
        hip = (np.arange(rows + 1, dtype=np.uint64) * npr).astype(np.uint32)
        hdat = rng.standard_normal(rows * npr)
        hx = rng.standard_normal(n)
        whole = False
        src = "numpy uniform stand-in (generator child failed: %s)" % (str(e)[:120],)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    nnz = int(hip[-1])
    y = np.zeros(rows)
    for _ in range(args.warmup):
        y[:] = 0
        O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, y)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        y[:] = 0
        O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, y)
    dt = (time.perf_counter() - t0) / args.steps
    val = 2.0 * nnz / dt / 1e9
    line = {"impl": "reference", "metric": "csr_spmv_f64_gflops", "value": val,
            "unit": "GFLOP/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": args.workload, "n": n, "nnz": nnz if whole else None,
                       "nnz_per_row": npr, "generator": gen, "index_bytes": 4,
                       "whole_matrix": whole, "rows_per_step": rows, "nnz_per_step": nnz,
                       "source": src},
            "cpu_baseline": {"value": val, "unit": "GFLOP/s", "cores": 1, "kind": "port",
                             "sample": "the whole matrix (%d nnz) per step; sprs SpMV/SpMM are "
                                       "single-threaded (SURVEY F6), so 1 thread IS all the "
                                       "threads the reference path can use; host has %d cores" %
                                       (nnz, O.num_procs())},
            "e2e": {"value": val, "unit": "GFLOP/s", "h2d_bytes_per_step": 0,
                    "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


# ---- product arm -----------------------------------------------------------------------
EXCHANGE_TEXT = {
    "fused": "all-gather of y fused into the SpMV kernel: every finished row is stored into %s "
             "by the kernel itself + device flag barrier in peer memory",
    "push": "SpMV, then one put kernel copying this rank's y slice into %s (coalesced 16-byte "
            "stores over NVLink) + device flag barrier in peer memory",
    "nccl": "NCCL all_gather(y), unequal slices (torch.distributed)",
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", default="spmv_rmat_10m", choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extra", action="store_true")
    ap.add_argument("--exchange", default="auto", choices=["auto", "fused", "push", "nccl"],
                    help="N>1 all-gather of y: 'push' = put kernel after the SpMV, 'fused' = stores "
                         "from the SpMV kernel itself (both through the library's communicator: "
                         "NVSwitch multicast address of y when available, else peer mappings), "
                         "'nccl' = one NCCL all_gather; 'auto' = the measured default (DESIGN.md 5)")
    ap.add_argument("--no-multicast", action="store_true",
                    help="keep the symmetric buffers on CUDA IPC peer mappings")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write the last step's result to DIR/<name>.npy")
    ap.add_argument("--gen-to", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--extra-only", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.gen_to:
        return generate_to_dir(args.workload, args.gen_to)
    if args.extra_only:
        return extra_child(args.extra_only)
    if args.impl == "reference":
        return run_reference(args)

    import torch
    import torch.distributed as dist
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    from sprs_b200.dist import (Comm, CommHostSpMV, CommSpMV, RowPartitionedSpMV, fit_row_cost,
                                nnz_balanced_bounds, rebalance_bounds)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world > 1:
        args.gpus = world
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)  # plumbing: id broadcast, timing reductions
    ctx = sp.Context.default(local)
    kind, n, npr, gen = WORKLOADS[args.workload]
    if kind != "spmv":
        return bench_other.run(args, ctx, kind, n, npr, gen, SEEDS[args.workload])
    peaks, peak_src = measured_peaks()
    hbm_peak = float(peaks["hbm_gbs"])

    def allmax(vals):
        t = torch.tensor(vals, device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.tolist()

    # ---- inputs, generated in HBM (every rank builds the same matrix, keeps its block)
    t_gen = time.time()
    full = G.make_matrix(ctx, gen, n, npr, SEEDS[args.workload])
    nnz = full.nnz
    x = G.normal_vector(ctx, n)
    comm = None
    if world > 1:
        ids = [Comm.unique_id(ctx) if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        comm = Comm(ctx, ids[0], rank, world)
    bounds = nnz_balanced_bounds(full.indptr, world)
    r0, r1 = bounds[rank], bounds[rank + 1]
    row_cost = 0.0
    if world > 1:
        # calibrate the partition: time this rank's nnz-balanced block, fit
        # t = alpha*nnz + beta*rows over the ranks, re-cut with rows weighted by beta/alpha
        a = full.slice_rows(r0, r1)
        yt = torch.empty(max(r1 - r0, 1), device=dev, dtype=torch.float64)
        for _ in range(2):
            G.spmv(ctx, a, x, yt)
        ce0, ce1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ce0.record()
        for _ in range(3):
            G.spmv(ctx, a, x, yt)
        ce1.record()
        torch.cuda.synchronize()
        allm = comm.allgather_f64([a.nnz, r1 - r0, ce0.elapsed_time(ce1) / 3e3])
        row_cost = fit_row_cost([m.tolist() for m in allm])
        del a, yt
        bounds = nnz_balanced_bounds(full.indptr, world, row_cost=row_cost)
        r0, r1 = bounds[rank], bounds[rank + 1]
        a = full.slice_rows(r0, r1)
    else:
        a = full
    cpu_base = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:  # rank 0 at N=1 only
        try:
            cpu_base = cpu_spmv_baseline(full, x, 1 << 27)
        except Exception as e:  # a reported baseline must never take the GPU number down
            cpu_base = {"error": repr(e)}
    t_gen = time.time() - t_gen
    if args.exchange == "auto":
        # the SpMV kernel storing every finished row itself (DESIGN.md section 5;
        # tools/scale_modes.py times every mode)
        args.exchange = "fused"
    use_comm = world > 1 and args.exchange in ("fused", "push")

    def make_op(a_blk, bnds):
        if use_comm:
            return CommSpMV(comm, a_blk.mirror, bnds, n, dev, exchange=args.exchange,
                            multicast=not args.no_multicast)
        yb = torch.zeros(n, device=dev, dtype=torch.float64)
        return RowPartitionedSpMV(bnds, rank, world, yb,
                                  lambda xv, ys: G.spmv(ctx, a_blk, xv, ys),
                                  dist=dist if world > 1 else None)

    op = make_op(a, bounds)
    rebalanced = 0
    if world > 1:
        # measured re-balancing with the REAL operator: up to four equal-time re-cuts; the cut
        # with the lowest measured maximum is the one that is timed (a re-cut made from noisy
        # timings can be worse than the one before it)
        def rebuild(nb):
            nonlocal op, a, bounds, r0, r1
            if hasattr(op, "close"):
                op.close()
            del op, a
            torch.cuda.empty_cache()
            bounds = nb
            r0, r1 = bounds[rank], bounds[rank + 1]
            a = full.slice_rows(r0, r1)
            op = make_op(a, bounds)

        def measure():
            for _ in range(2):
                op.step(x)
            ce0, ce1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            tsum = 0.0
            for _ in range(6):
                torch.cuda.synchronize()
                dist.barrier()
                ce0.record()
                op.compute(x)
                ce1.record()
                op.exchange()
                torch.cuda.synchronize()
                tsum += ce0.elapsed_time(ce1)
            return [float(v[0]) for v in comm.allgather_f64([tsum / 6])]

        best = None  # (max time, bounds)
        for rnd in range(5):
            times = measure()
            if best is None or max(times) < best[0]:
                best = (max(times), list(bounds))
            if rnd == 4 or max(times) <= 1.01 * (sum(times) / world):
                break
            nb = rebalance_bounds(full.indptr, bounds, times, row_cost=row_cost)
            if nb == bounds:
                break
            rebuild(nb)
            rebalanced += 1
        if best[1] != list(bounds):
            rebuild(best[1])
    multicast = bool(getattr(op, "multicast", False))

    # ---- parity first, untimed: this rank's WHOLE y against the CPU oracle (every rank)
    op.y.fill_(float("nan"))
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    op.step(x)
    torch.cuda.synchronize()
    if comm is not None:
        comm.check()
    try:
        p_ok, p_rows, p_worst = parity_vs_oracle(full, x, op.y)
        p_err = None
    except Exception as e:
        p_ok, p_rows, p_worst, p_err = False, 0, float("inf"), repr(e)
    p_ok_all, p_worst_all = allmax([0.0 if p_ok else 1.0, p_worst if np.isfinite(p_worst) else 1e300])
    parity = {"ok": p_ok_all == 0.0, "rows_checked_per_rank": p_rows,
              "max_error_over_gate": p_worst_all,
              "gate": "|got - oracle| <= 1e-6 * sum|terms| per row; heaviest 100 rows + 10000 "
                      "random rows of the whole (all-gathered) y, checked on every rank"}
    if p_err:
        parity["error"] = p_err
    # the ceiling of this matrix (N=1): the same streams and gathers without the row logic
    ceiling = None
    if world == 1:
        try:
            import ctypes as C
            ms_c, cov = C.c_double(), C.c_uint64()
            ctx.check(ctx.lib.sprs_b200_diag_gather_ceiling(ctx.h, full.mirror.h,
                                                            C.c_void_p(x.data_ptr()), 5,
                                                            C.byref(ms_c), C.byref(cov)))
            ceiling = {"ms": ms_c.value, "gnnz_s": cov.value / ms_c.value / 1e6,
                       "frac_of_hbm": (12.0 * cov.value + 8.0 * n) / ms_c.value / 1e6 / hbm_peak,
                       "kernel": "sprs_b200_diag_gather_ceiling (csrc/diag.cu): same index/value "
                                 "stream and x gathers as the SpMV, one sum per lane, no rows"}
        except Exception as e:
            ceiling = {"error": repr(e)}
    y = op.y
    local_nnz = a.nnz

    for _ in range(max(args.warmup, 3)):
        op.step(x)
    torch.cuda.synchronize()
    sampler = ClockSampler(local)
    use_sampler = rank == 0 and not os.environ.get("SPRS_BENCH_NO_SAMPLER")
    if use_sampler:  # started BEFORE the barrier so that no rank enters the timed region late
        sampler.start()
        time.sleep(0.05)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()

    # ---- timed region: K steps, CUDA events on the launching stream, max over ranks
    launches0 = ctx.launches
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True),
            torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    tw0 = time.time()
    e_start, e_stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e_start.record()
    for i in range(args.steps):
        evs[i][0].record()
        op.compute(x)
        evs[i][1].record()
        op.exchange()
        evs[i][2].record()
    e_stop.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    tw1 = time.time()
    clocks = sampler.stop(tw0, tw1) if use_sampler else None
    launches = ctx.launches - launches0
    if comm is not None:
        comm.check()
    if args.dump_outputs and rank == 0:
        dump_rows(args.dump_outputs, "y", op.y)  # the whole y = A x of the last timed step
    total_ms = e_start.elapsed_time(e_stop)
    kern_ms = [evs[i][0].elapsed_time(evs[i][1]) for i in range(args.steps)]
    coll_ms = [evs[i][1].elapsed_time(evs[i][2]) for i in range(args.steps)]
    my_kern = statistics.mean(kern_ms)
    total_ms, kern_ms_avg, coll_ms_avg = allmax([total_ms, my_kern, statistics.mean(coll_ms)])
    per_rank_kern = ([float(v[0]) for v in comm.allgather_f64([my_kern])] if comm is not None
                     else [my_kern])
    ms_per_step = total_ms / args.steps

    # ---- e2e: the reference-facing call with HOST buffers, every step: x H2D from pinned
    # memory and y D2H inside the timed region.  N=1: `&A * &x` through sprs_b200_mul_mat_vec.
    # N>1: sprs_b200_mul_mat_vec_rowpart -- every rank moves only ITS slices of x and y.
    import ctypes as C
    rows_local = rows_e2e = r1 - r0
    e2e_steps = max(3, min(args.steps, 10))
    if world == 1:
        hx = torch.empty(n, dtype=torch.float64).pin_memory()
        hx.copy_(x)
        hy = torch.empty(max(rows_local, 1), dtype=torch.float64).pin_memory()

        def e2e_step():
            ctx.check(ctx.lib.sprs_b200_mul_mat_vec(ctx.h, a.mirror.h, C.c_void_p(hx.data_ptr()), n,
                                                    C.c_void_p(hy.data_ptr()), rows_local))
        e2e_api = "sprs_b200_mul_mat_vec (host x, y; A resident as a device mirror)"
        hop = None
    else:
        # The host-vector form has its own cut.  Every y row costs 8 bytes over PCIe on top of
        # its share of the SpMV, so its row blocks are balanced on nnz + (row_cost + c_pcie)*rows,
        # c_pcie = 8 B / (measured D2H rate) in non-zero equivalents of the measured SpMV rate;
        # x (needed by every rank, whatever its rows) is uploaded in EQUAL column slices.
        probe_n = 4 << 20
        hprobe = torch.empty(probe_n, dtype=torch.float64).pin_memory()
        dprobe = torch.empty(probe_n, dtype=torch.float64, device=dev)
        hprobe.copy_(dprobe)
        torch.cuda.synchronize()
        tp = time.perf_counter()
        hprobe.copy_(dprobe)
        torch.cuda.synchronize()
        d2h_bps = 8.0 * probe_n / (time.perf_counter() - tp)
        nnz_per_s = local_nnz / (my_kern * 1e-3)
        vals = comm.allgather_f64([d2h_bps, nnz_per_s])
        d2h_bps = float(np.mean([v[0] for v in vals]))
        nnz_per_s = float(np.mean([v[1] for v in vals]))
        c_pcie = 8.0 / d2h_bps * nnz_per_s
        del hprobe, dprobe
        e2e_bounds = nnz_balanced_bounds(full.indptr, world, row_cost=row_cost + c_pcie)
        x_bounds = [n * g // world for g in range(world + 1)]
        er0, er1 = e2e_bounds[rank], e2e_bounds[rank + 1]
        xc0, xc1 = x_bounds[rank], x_bounds[rank + 1]
        a_e2e = full.slice_rows(er0, er1)
        ref_y_e2e = y[er0:er1].clone()
        rows_e2e = er1 - er0
        hx = torch.empty(max(xc1 - xc0, 1), dtype=torch.float64).pin_memory()
        hx[:xc1 - xc0].copy_(x[xc0:xc1])
        hy = torch.empty(max(rows_e2e, 1), dtype=torch.float64).pin_memory()
        hop = CommHostSpMV(comm, a_e2e.mirror, e2e_bounds, n, multicast=not args.no_multicast,
                           x_bounds=x_bounds)

        def e2e_step():
            hop.step(hx.data_ptr(), hy.data_ptr())
        e2e_api = ("sprs_b200_mul_mat_vec_rowpart (each rank uploads an equal slice of x, x is "
                   "all-gathered over NVLink, each rank downloads the y rows of its block; blocks "
                   "balanced on nnz + %.1f*rows: SpMV row cost + 8 B of PCIe per row)"
                   % (row_cost + c_pcie))
    for _ in range(2):
        e2e_step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        e2e_step()
    torch.cuda.synchronize()
    e2e_ms = (time.perf_counter() - t0) * 1e3 / e2e_steps
    (e2e_ms,) = allmax([e2e_ms])
    ref_y = y[r0:r1] if world == 1 else ref_y_e2e
    got_y = hy[:rows_e2e].to(dev)
    ok = bool(((got_y - ref_y).abs() <= 1e-9 * (ref_y.abs().max() + 1e-300)).all())
    (e2e_bad,) = allmax([0.0 if ok else 1.0])
    if hop is not None:
        hop.close()

    extra = {}
    if rank == 0 and world == 1 and not args.no_extra and args.workload == "spmv_rmat_10m":
        del a, full, op, y
        torch.cuda.empty_cache()
        for name, fn in (("spmv_rand_1m", bench_small_spmv), ("spmm_rand_1m_k64", bench_other.extra_spmm),
                         ("spgemm_rmat_500k", bench_other.extra_spgemm)):
            try:
                res = None
                if name == "spmv_rand_1m":
                    # a sub-millisecond kernel is the one entry that is sensitive to what the
                    # process did before it: measured in a child process, like
                    # tools/sweep_spmv.py does; in this process only if the child fails
                    res = run_extra_in_child(name)
                extra[name] = res if res is not None else fn(ctx, G, hbm_peak, dev)
            except Exception as e:
                extra[name] = {"error": repr(e)}
            torch.cuda.empty_cache()

    if rank == 0:
        flops = 2.0 * nnz
        alg_bytes = 12.0 * nnz + 8.0 * n
        gflops = flops / (ms_per_step * 1e-3) / 1e9
        # roofline of the dominant kernel (spmv_rows_kernel; the carry fix-up kernel -- and at
        # N > 1 the put kernel of the 'push' exchange -- ride in the same event pair):
        # algorithmic bytes this rank's launch moves / its mean duration.
        local_bytes = 12.0 * local_nnz + 8.0 * rows_local
        achieved = local_bytes / (per_rank_kern[0] * 1e-3) / 1e9
        target = ("the NVSwitch multicast address of y (one store per row, replicated by the switch)"
                  if multicast else "every peer's y (CUDA IPC / VMM peer mappings)")
        roof = {"bound": "hbm", "achieved": achieved, "peak": hbm_peak, "unit": "GB/s",
                "frac": achieved / hbm_peak,
                "traffic": bench_other.ncu_traffic(args.workload, world),
                "traffic_source": bench_other.ncu_traffic(args.workload, world, source=True),
                "kernel": "spmv_rows_kernel (+ spmv_fixup_kernel)",
                "kernel_ms": per_rank_kern[0], "kernel_ms_per_rank": per_rank_kern,
                "peak_source": peak_src,
                "algorithmic_bytes": "12*nnz + 8*rows of this rank's block per launch",
                "variant": os.environ.get("SPRS_B200_SPMV_VARIANT", "default 1024,16 (cost units per tile, row cost); 8-warp CTAs, 5 per SM, 4 loads in flight")}
        if ceiling is not None:
            roof["gather_ceiling"] = ceiling
            if "frac_of_hbm" in ceiling:
                roof["frac_of_gather_ceiling"] = (achieved / hbm_peak) / ceiling["frac_of_hbm"]
        line = {
            "metric": "csr_spmv_f64_gflops", "value": gflops, "unit": "GFLOP/s",
            "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": args.workload, "n": n, "nnz": nnz, "nnz_per_row": npr,
                       "generator": gen, "index_bytes": 4,
                       "partition": "contiguous row blocks balanced on nnz + %.2f*rows "
                                    "(row cost fitted from per-rank timings), then %d measured "
                                    "equal-time re-cut(s), the cut with the lowest measured maximum kept" % (row_cost, rebalanced),
                       "collective": ("none" if world == 1 else
                                      (EXCHANGE_TEXT[args.exchange] % target
                                       if args.exchange != "nccl" else EXCHANGE_TEXT["nccl"])),
                       "communicator": (None if comm is None else
                                        "sprs_b200_comm (C ABI: shm rendezvous, %s symmetric buffers, "
                                        "device flag barrier); torch.distributed only broadcasts the id"
                                        % ("VMM + NVSwitch multicast" if multicast else "CUDA IPC")),
                       "l2_policy": "inputs (%.1f GB) exceed the H100's L2 (50 MB); no flush needed" %
                                    (alg_bytes / 1e9),
                       "gen_seconds": round(t_gen, 1)},
            "achieved_hbm_frac": (alg_bytes / (ms_per_step * 1e-3) / 1e9) / (hbm_peak * world),
            "roofline": roof,
            "parity_vs_oracle": parity,
            "collective_ms": coll_ms_avg,
            "e2e": {"value": flops / (e2e_ms * 1e-3) / 1e9, "unit": "GFLOP/s",
                    "ms_per_step": e2e_ms, "h2d_bytes_per_step": 8 * n,
                    "d2h_bytes_per_step": 8 * n, "api": e2e_api,
                    "matches_device_result": e2e_bad == 0.0},
            "gpu_launches": int(launches), "clocks": clocks,
        }
        if cpu_base:
            line["cpu_baseline"] = cpu_base
        if extra:
            line["extra"] = extra
        print(json.dumps(line))
    if world > 1:
        if hasattr(op, "close"):
            op.close()
        comm.close()
        dist.destroy_process_group()


def extra_child(name):
    """Child-process entry (`bench.py --extra-only NAME`): one entry of `extra` measured in a
    process of its own; prints its JSON on the last line."""
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    if name != "spmv_rand_1m":
        raise SystemExit("unknown extra %r" % name)
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    ctx = sp.Context.default(local)
    peaks, _ = measured_peaks()
    out = bench_small_spmv(ctx, G, float(peaks["hbm_gbs"]), torch.device("cuda", local))
    out["process"] = "child process of bench.py (nothing else ran in it)"
    print(json.dumps(out))
    return 0


def run_extra_in_child(name, timeout=600):
    """None when the child did not deliver (the caller then measures in-process)."""
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--extra-only", name],
                           capture_output=True, text=True, timeout=timeout)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        if r.returncode != 0 or not lines:
            return None
        res = json.loads(lines[-1])
        return res if isinstance(res, dict) and "ms" in res else None
    except Exception:
        return None


def bench_small_spmv(ctx, G, hbm_peak, dev):
    """BASELINE config 2 (1M x 1M sprs-rand, 32 nnz/row), reported as an extra line item with
    its own gather ceiling.  392 MB of inputs > L2, so no flush is needed between iterations."""
    import ctypes as C
    import torch
    n = 1_000_000
    a = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
    x = G.normal_vector(ctx, n)
    y = torch.empty(n, device=dev, dtype=torch.float64)
    for _ in range(5):
        G.spmv(ctx, a, x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    k = 50
    e0.record()
    for _ in range(k):
        G.spmv(ctx, a, x, y)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / k
    by = 12.0 * a.nnz + 8.0 * n
    ok, rows, worst = parity_vs_oracle(a, x, y, n_random=20000, n_heavy=10)
    out = {"nnz": a.nnz, "ms": ms, "gflops": 2.0 * a.nnz / ms / 1e6, "achieved_gbs": by / ms / 1e6,
           "frac": by / ms / 1e6 / hbm_peak,
           "parity_vs_oracle": {"ok": ok, "rows_checked": rows, "max_error_over_gate": worst}}
    ms_c, cov = C.c_double(), C.c_uint64()
    ctx.check(ctx.lib.sprs_b200_diag_gather_ceiling(ctx.h, a.mirror.h, C.c_void_p(x.data_ptr()), 20,
                                                    C.byref(ms_c), C.byref(cov)))
    cf = (12.0 * cov.value + 8.0 * n) / ms_c.value / 1e6 / hbm_peak
    out["gather_ceiling"] = {"ms": ms_c.value, "frac_of_hbm": cf}
    out["frac_of_gather_ceiling"] = out["frac"] / cf
    return out


if __name__ == "__main__":
    main()
