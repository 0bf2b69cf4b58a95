"""Times the SpMV hot set (SPRS_B200_SPMV_HOT=auto|0|K, csrc/spmv.cu) on the bench workloads;
one subprocess per setting because the switch is read once per process.

    python tools/sweep_spmv_hot.py 0 12288 16384 24576 0 [K@/path/to/libsprs_b200.so ...]

A setting `K@lib` loads another build of the library (e.g. one compiled with a different
hot-set CTA shape).  Per setting and workload it prints the SpMV time (3 windows of 20 launches:
min / median), the time to adopt the same device arrays again (tile cuts + hot-set build), the
share of the non-zeros the K most-referenced columns hold, and a checksum of y's bits, which
must agree between settings (the hot set does not change a single bit of y).
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, json, time, torch
sys.path.insert(0, %r)
import sprs_b200 as sp
if %r:
    sp._lib.LIB_PATH = %r
from sprs_b200 import generate as G
K = %d
ctx = sp.Context.default(0)
out = {}
for name, gen, n, npr in %s:
    a = G.make_matrix(ctx, gen, n, npr, 0x5EED0005 if gen == "rmat" else 0x5EED0002)
    x = G.normal_vector(ctx, n); y = torch.empty(n, device="cuda", dtype=torch.float64)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    b = G.DeviceCsr(ctx, n, n, a.indptr, a.indices, a.data)
    torch.cuda.synchronize()
    prep_ms = (time.perf_counter() - t0) * 1e3
    del b
    share = None
    if K > 0:
        cnt = torch.zeros(n, device="cuda", dtype=torch.int64)
        for s in range(0, a.nnz, 1 << 27):
            cnt += torch.bincount(a.indices[s:s + (1 << 27)].long(), minlength=n)
        share = float(torch.topk(cnt, min(K, n)).values.sum().item()) / a.nnz
        del cnt
    for _ in range(5): G.spmv(ctx, a, x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(3):
        e0.record()
        for _ in range(20): G.spmv(ctx, a, x, y)
        e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / 20)
    ms.sort()
    bits = int(y.view(torch.int64).sum().item()) ^ int(y.view(torch.int64)[::7].sum().item())
    out[name] = {"ms_min": ms[0], "ms_med": ms[1], "prep_ms": prep_ms, "hot_share": share,
                 "ybits": bits}
    del a, x, y; torch.cuda.empty_cache()
print("RESULT " + json.dumps(out))
'''


def main():
    workloads = [("rand_1m_32", "rand", 1_000_000, 32), ("rmat_10m_100", "rmat", 10_000_000, 100)]
    settings = sys.argv[1:] or ["0", "auto", "12288", "16384", "24576", "0"]
    ref_bits = {}
    for v in settings:
        hot, _, lib = v.partition("@")
        env = dict(os.environ, SPRS_B200_SPMV_HOT=hot)
        k = 0 if hot in ("0", "auto") else int(hot)
        r = subprocess.run([sys.executable, "-c", CHILD % (ROOT, lib, lib, k, repr(workloads))],
                           env=env, capture_output=True, text=True)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        if not line:
            print(v, "FAILED", r.stderr[-1500:], flush=True)
            continue
        res = json.loads(line[0][7:])
        parts = []
        for name, d in res.items():
            same = ref_bits.setdefault(name, d["ybits"]) == d["ybits"]
            parts.append("%s: %.3f / %.3f ms, prep %.0f ms, share %s, y %s" % (
                name, d["ms_min"], d["ms_med"], d["prep_ms"],
                "-" if d["hot_share"] is None else "%.3f" % d["hot_share"],
                "same bits" if same else "BITS DIFFER"))
        print(v.ljust(14), " | ".join(parts), flush=True)


if __name__ == "__main__":
    main()
