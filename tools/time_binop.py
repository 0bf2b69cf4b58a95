"""Times the device binops (csrc/binop.cu) on the project's workloads: one JSON line each.

    python tools/time_binop.py [--calls 20] [--warmup 3] [--only rand1m_add,...] [--out DIR]

Workloads (every input built on the device with sprs_b200.generate):
  rand1m_add     config-2 A (seed 0x5EED0002) + B (seed 0x5EED1002), 32 M non-zeros each
  rand1m_mul     the same A .* B (almost empty output: the count pass)
  rmat500k_sym   config-4 R-MAT A + A^T (A^T = the CSR of to_other_storage(A))
  rmat10m_shift  config-5 R-MAT A - 1.0 * I
  rmat10m_scale  config-5 A * 2.0

Each line: nnzA, nnzB, nnzC; the call time (host clock around the blocking call, which ends in
a stream synchronise), median and min over --calls calls after --warmup; the kernel-only time
(sum of the call's CUDA kernels in a separate torch.profiler run); the algorithmic bytes of the
two-pass form, 2 (12 (nnzA + nnzB) + wA (outer+1) + wB (outer+1)) + 12 nnzC + wC (outer+1)
(scale: one pass, read + write), and the kernel time's fraction of 3.35 TB/s; the single-thread
oracle time of the same operation (tests/cpp/oracle_binop.cpp, run chunk by chunk) and a parity
flag from the bit-exact comparison of the timed output with it (the whole output); GPU name,
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12
_CACHE = {}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": clock}
    except Exception as e:  # noqa: BLE001  (reported, not fatal)
        return {"gpu": "unknown (%s)" % e}


def build_inputs(ctx, name):
    import torch
    from sprs_b200 import generate as G
    if name.startswith("rand1m"):
        n = 1_000_000
        return n, G.rand_csr(ctx, n, n, 32, seed=0x5EED0002), G.rand_csr(ctx, n, n, 32, seed=0x5EED1002), []
    if name == "rmat500k_sym":
        n = 500_000
        a = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
        t = G._with_views(ctx, a.mirror.to_other_storage())  # CSC of A = CSR of A^T
        return n, a, G.DeviceCsr(ctx, n, n, t[1], t[2], t[3]), [t]
    n = 10_000_000
    if "rmat10m" not in _CACHE:  # built once for both config-5 workloads
        _CACHE["rmat10m"] = G.rmat_csr(ctx, n, 100, seed=0x5EED0005)
    a = _CACHE["rmat10m"]
    if name == "rmat10m_scale":
        return n, a, None, []
    dev = G._device(ctx)
    eye = G.DeviceCsr(ctx, n, n, torch.arange(n + 1, dtype=torch.int32, device=dev),
                      torch.arange(n, dtype=torch.int32, device=dev),
                      torch.ones(n, dtype=torch.float64, device=dev))
    return n, a, eye, []


OPS = {"rand1m_add": "add", "rand1m_mul": "mul", "rmat500k_sym": "add", "rmat10m_shift": "sub",
       "rmat10m_scale": "scale"}


def run(ctx, name, args):
    import torch
    import binop_oracle as BO
    from sprs_b200 import generate as G
    n, a, b, keep = build_inputs(ctx, name)
    op = OPS[name]
    lib = ctx.lib

    def call():
        out = C.c_void_p()
        if op == "scale":
            ctx.check(lib.sprs_b200_csmat_scale(ctx.h, a.mirror.h, 2.0, C.byref(out)))
        else:
            ctx.check(lib.sprs_b200_csmat_binop(ctx.h, a.mirror.h, b.mirror.h,
                                                {"add": 0, "sub": 1, "mul": 2}[op], C.byref(out)))
        return G.DeviceCsMat(ctx, out)

    for _ in range(args.warmup):
        call().free()
    times = []
    for _ in range(args.calls):
        t0 = time.perf_counter()
        m = call()
        times.append((time.perf_counter() - t0) * 1e3)
        m.free()
    # kernel-only time: one call under torch.profiler (a run of its own)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m = call()
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            kernels[e.name] = kernels.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
    kernel_ms = sum(kernels.values())
    res = G._with_views(ctx, m)
    nnz_a = a.nnz
    nnz_b = b.nnz if b is not None else 0
    nnz_c = res[0].nnz
    wa = a.indptr.element_size()
    wc = res[1].element_size()
    if op == "scale":
        nbytes = 2 * (12 * nnz_a + wa * (n + 1))
        err, oracle_s = BO.compare_chunked(("scale", 2.0), (a.indptr, a.indices, a.data), None,
                                           res[1:], n)
    else:
        wb = b.indptr.element_size()
        nbytes = 2 * (12 * (nnz_a + nnz_b) + wa * (n + 1) + wb * (n + 1)) + 12 * nnz_c + wc * (n + 1)
        err, oracle_s = BO.compare_chunked({"add": BO.ADD, "sub": BO.SUB, "mul": BO.MUL}[op],
                                           (a.indptr, a.indices, a.data),
                                           (b.indptr, b.indices, b.data), res[1:], n)
    line = {"workload": name, "nnzA": nnz_a, "nnzB": nnz_b, "nnzC": nnz_c,
            "call_ms_median": round(statistics.median(times), 3), "call_ms_min": round(min(times), 3),
            "calls": args.calls, "kernel_ms": round(kernel_ms, 3),
            "kernels_ms": {k: round(v, 3) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])},
            "algorithmic_bytes": nbytes, "roofline_ms": round(nbytes / HBM_BPS * 1e3, 3),
            "kernel_fraction_of_3.35TBps": round(nbytes / HBM_BPS * 1e3 / kernel_ms, 3) if kernel_ms else None,
            "oracle_single_thread_ms": round(oracle_s * 1e3, 1),
            "parity": "ok" if err is None else "FAIL: " + err}
    line.update(gpu_info())
    del res, m, keep
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=",".join(OPS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import sprs_b200 as sp
    ctx = sp.Context.default()
    lines = []
    for name in args.only.split(","):
        line = run(ctx, name, args)
        print(json.dumps(line), flush=True)
        lines.append(line)
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_binop.jsonl"), "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)
    return 0 if all(x["parity"] == "ok" for x in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
