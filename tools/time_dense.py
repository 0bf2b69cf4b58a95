"""Times the dense boundary (the dense section of csrc/transpose.cu) at 32768 x 32768: one JSON
line per workload.

    python tools/time_dense.py [--calls 10] [--warmup 2] [--only to_dense,...] [--out DIR]

Workloads (inputs built on the device; A = generate.rand_csr 32768^2, 32 non-zeros per row,
seed 0x5EED0D01; D = N(0,1), torch seed 11):
  to_dense        to_dense(A) into a C-order tensor (the _dev form)
  add_c           add_dense_mat_same_ordering(A, D, 1, 1), D C order
  mul_c           mul_dense_mat_same_ordering(A, D, -0.5), D C order
  add_f           `&A + &D` with D F order: A's to_other_storage conversion is part of the call
  from_dense_0.1  csr_from_dense(M, 1e-3), M with ~0.1 % of its elements non-zero
  from_dense_50   the same with ~50 % non-zero

Each line: the call time (host clock around the call and a device synchronise), median and min
over --calls after --warmup; the kernel-only time (sum of the call's CUDA kernels in a separate
torch.profiler run); the algorithmic bytes -- to_dense 8 R C + 12 nnz + indptr, binops
16 R C + 12 nnz + indptr, from_dense the two-pass 16 R C + 12 nnz + indptr and its one-read floor
8 R C + 12 nnz + indptr -- and the kernel time's fraction of 3.35 TB/s; the single-thread oracle
(tests/dense_oracle.cpp) timed on the first 2048 rows and scaled to the whole matrix; a parity
flag from comparing the whole output on the device with a torch model (to_dense(A) by index_put;
(alpha*X) + (beta*D) and (alpha*X)*D elementwise, each operation rounded on its own; the mask /
nonzero model for from_dense); GPU name, power limit and SM clock read in the same process.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12
N = 32768
SLICE = 2048


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (reported, not fatal)
        return {"gpu": "unknown (%s)" % e}


def bits_equal(x, y):
    import torch
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


def model_dense(a):
    import torch
    ip = a.indptr.long()
    rows = torch.repeat_interleave(torch.arange(a.rows, device=ip.device), ip[1:] - ip[:-1])
    x = torch.zeros((a.rows, a.cols), dtype=torch.float64, device=ip.device)
    x[rows, a.indices.long()] = a.data
    return x


def host_csr(a, r1):
    """CsMat-like host arrays of rows [0, r1) of a DeviceCsr"""
    from types import SimpleNamespace
    import numpy as np
    ip = a.indptr[:r1 + 1].cpu().numpy().astype(np.uint64)
    e = int(ip[-1])
    return SimpleNamespace(storage="CSR", shape=(r1, a.cols), indptr=ip,
                           indices=a.indices[:e].cpu().numpy().view(np.uint32).astype(np.uint64),
                           data=a.data[:e].cpu().numpy())


def oracle_ms(name, a, d):
    """single-thread oracle on the first SLICE rows, scaled to N rows"""
    import numpy as np
    import dense_oracle as DO
    DO.lib()
    if name.startswith("from_dense"):
        m = d[:SLICE].cpu().numpy()
        t0 = time.perf_counter()
        DO.csr_from_dense(m, 1e-3)
    else:
        h = host_csr(a, SLICE)
        if name == "to_dense":
            t0 = time.perf_counter()
            DO.to_dense(h)
        else:
            rhs = d[:SLICE].cpu().numpy()
            if name == "add_f":
                rhs = np.asfortranarray(rhs)
            out = np.zeros(rhs.shape)
            t0 = time.perf_counter()
            DO.binop_dense(h, DO.MUL if name == "mul_c" else DO.ADD, -0.5 if name == "mul_c" else 1.0,
                           1.0, rhs, out)
    return (time.perf_counter() - t0) * 1e3 * N / SLICE


def run(ctx, name, args, a, x):
    import torch
    from sprs_b200 import generate as G
    g = torch.Generator(device="cuda").manual_seed(11)
    d = torch.randn((N, N), dtype=torch.float64, device="cuda", generator=g)
    nnz = a.nnz
    keep = []
    if name == "to_dense":
        out = torch.empty((N, N), dtype=torch.float64, device="cuda")
        call = lambda: G.to_dense(ctx, a, out=out)  # noqa
        nbytes = 8 * N * N + 12 * nnz + 4 * (N + 1)
    elif name in ("add_c", "mul_c"):
        op, alpha = ("add", 1.0) if name == "add_c" else ("mul", -0.5)
        out = torch.empty((N, N), dtype=torch.float64, device="cuda")
        call = lambda: G.binop_dense(ctx, a, d, op, alpha, 1.0, out=out)  # noqa
        nbytes = 16 * N * N + 12 * nnz + 4 * (N + 1)
    elif name == "add_f":
        d = d.t()
        out = torch.empty((N, N), dtype=torch.float64, device="cuda").t()

        def call():
            t = a.mirror.to_other_storage()
            G.binop_dense(ctx, t, d, "add", 1.0, 1.0, out=out)
            keep.append(t)
            return out
        nbytes = 16 * N * N + 12 * nnz + 4 * (N + 1)
    else:
        dens = 0.001 if name == "from_dense_0.1" else 0.5
        d[torch.rand((N, N), device="cuda", generator=g) >= dens] = 0.0
        res = []

        def call():
            res[:] = [G.from_dense(ctx, d, 1e-3)]
            return res[0]
        out = None
    for _ in range(args.warmup):
        call()
        torch.cuda.synchronize()
        keep.clear()
    times = []
    for _ in range(args.calls):
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        keep.clear()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            kernels[e.name] = kernels.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
    kernel_ms = sum(kernels.values())
    line = {"workload": name, "rows": N, "cols": N, "nnzA": nnz}
    if name.startswith("from_dense"):
        m, ip, ind, dat = res[0]
        nnz_c = m.nnz
        w = ip.element_size()
        nbytes = 16 * N * N + 12 * nnz_c + w * (N + 1)
        line.update(nnzC=nnz_c, floor_bytes=8 * N * N + 12 * nnz_c + w * (N + 1))
        keepm = d.abs() > 1e-3
        nz = keepm.nonzero()
        ok = (torch.equal(ip[1:].long(), keepm.sum(dim=1).cumsum(0)) and
              torch.equal(ind.long(), nz[:, 1]) and bits_equal(dat, d[keepm]))
        del nz, keepm
    elif name == "to_dense":
        ok = bits_equal(out, x)
    else:
        ok = True
        for r0 in range(0, N, 4096):
            xs, ds = x[r0:r0 + 4096], d[r0:r0 + 4096]
            want = (xs * -0.5) * ds if name == "mul_c" else (xs * 1.0) + (ds * 1.0)
            ok = ok and bits_equal(out[r0:r0 + 4096], want)
    line.update({
        "call_ms_median": round(statistics.median(times), 3), "call_ms_min": round(min(times), 3),
        "calls": args.calls, "kernel_ms": round(kernel_ms, 3),
        "kernels_ms": {k[:80]: round(v, 3) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])},
        "algorithmic_bytes": nbytes, "roofline_ms": round(nbytes / HBM_BPS * 1e3, 3),
        "kernel_fraction_of_3.35TBps": round(nbytes / HBM_BPS * 1e3 / kernel_ms, 3) if kernel_ms else None,
        "oracle_single_thread_ms": round(oracle_ms(name, a, d), 1),
        "parity": "ok" if ok else "FAIL"})
    if "floor_bytes" in line:
        line["floor_fraction_of_3.35TBps"] = round(line["floor_bytes"] / HBM_BPS * 1e3 / kernel_ms, 3)
    line.update(gpu_info())
    return line


WORKLOADS = ["to_dense", "add_c", "mul_c", "add_f", "from_dense_0.1", "from_dense_50"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    a = G.rand_csr(ctx, N, N, 32, seed=0x5EED0D01)
    x = model_dense(a)
    lines = []
    for name in args.only.split(","):
        line = run(ctx, name, args, a, x)
        print(json.dumps(line), flush=True)
        lines.append(line)
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_dense.jsonl"), "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)
    return 0 if all(x["parity"] == "ok" for x in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
