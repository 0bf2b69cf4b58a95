"""CPU check of the failure paths of every entry point that allocates device memory, on the
emulator (tests/emu) with the binops, the construction, the triangular solves and the LDL^T
factorization built in as in tests/emu_*.py.

The libraries are linked here with tests/emu/cuemu_fail.cpp in place of the emulator's cuemu.o:
`cuemu_fail_alloc_after(n)` makes the n-th next allocation fail, `cuemu_live_allocs()` counts
allocations minus frees.  For each entry point: one successful warm-up call (so that the ctx
scratch slots and the CSR cache of a CSC operand exist), then for k = 0, 1, 2, ... the k-th
allocation of the call fails until a call no longer reaches allocation k.  Every such call
returns OK -- legitimate where a failed allocation only means "no SpMV hot set", and then the
result must equal the warm-up result -- or ERR_CUDA with a fresh last_error that names the call
and *out NULL; afterwards no allocation is left behind.

The checks run in a child process per library (SPRS_B200_SPMV_HOT forces the hot set, so its
build is on the failure path too).  With SPRS_B200_EMU_ASAN=1 and
LD_PRELOAD=$(gcc -print-file-name=libasan.so) the main library is built from the emulator's
AddressSanitizer objects."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (HERE, ROOT):
    if d not in sys.path:
        sys.path.insert(0, d)

OK, ERR_CUDA = 0, 3
CSR, CSC = 0, 1
SENTINEL = b"bad storage or index width"
_vp, _u64 = C.c_void_p, C.c_uint64


def _ptr(a):
    return a.ctypes.data_as(_vp)


def _f64(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class Lib:
    def __init__(self, path):
        from sprs_b200._lib import PROTOTYPES
        self.lib = C.CDLL(path)
        for name, (res, args) in PROTOTYPES.items():
            if hasattr(self.lib, name):
                fn = getattr(self.lib, name)
                fn.restype, fn.argtypes = res, args
        self.lib.cuemu_fail_alloc_after.restype = C.c_long
        self.lib.cuemu_fail_alloc_after.argtypes = [C.c_long]
        self.lib.cuemu_live_allocs.restype = C.c_long
        ctx = _vp()
        assert self.lib.sprs_b200_ctx_create(0, C.byref(ctx)) == OK
        self.ctx = ctx
        self.keep = []  # host arrays that must outlive the mirrors adopting them

    def __getattr__(self, name):
        return getattr(self.lib, "sprs_b200_" + name)

    def error(self):
        return self.lib.sprs_b200_last_error(self.ctx) or b""

    def upload(self, storage, shape, indptr, indices, data):
        out = _vp()
        st = self.csmat_upload(self.ctx, storage, shape[0], shape[1], _ptr(indptr), 4,
                               _ptr(indices), 4, _f64(data), C.byref(out))
        assert st == OK, self.error()
        return out

    def download(self, m):
        storage, rows = self.csmat_storage(m), self.csmat_rows(m)
        cols, nnz = self.csmat_cols(m), self.csmat_nnz(m)
        ip = np.zeros((rows if storage == CSR else cols) + 1, np.uint64)
        idx, val = np.zeros(max(nnz, 1), np.uint32), np.zeros(max(nnz, 1))
        assert self.csmat_download(self.ctx, m, _ptr(ip), 8, _ptr(idx), 4, _f64(val)) == OK
        return (storage, rows, cols, ip.tobytes(), idx[:nnz].tobytes(), val[:nnz].tobytes())

    def set_sentinel_error(self):
        ip, out = np.zeros(2, np.uint32), _vp()
        assert self.csmat_upload(self.ctx, 7, 1, 1, _ptr(ip), 4, None, 4, None, C.byref(out)) != OK
        assert self.error() == SENTINEL


def rand_csr(rng, rows, cols, per_row, lower=False):
    indptr, indices = [0], []
    for r in range(rows):
        hi = min(r + 1, cols) if lower else cols
        c = set(rng.choice(hi, size=min(per_row, hi), replace=False).tolist())
        if lower and r < cols:
            c.add(r)
        indices += sorted(c)
        indptr.append(len(indices))
    data = rng.standard_normal(len(indices)) + (3.0 if lower else 0.0)
    return (np.array(indptr, np.uint32), np.array(indices, np.uint32), data)


def check(L, name, call, fetch, free, names):
    """call() -> (status, handle or None).  Returns the failures found."""
    st, h = call()
    assert st == OK, (name, st, L.error())
    want = fetch(h)
    free(h)
    base = L.lib.cuemu_live_allocs()
    failures = []
    for k in range(10000):
        L.set_sentinel_error()
        L.lib.cuemu_fail_alloc_after(k)
        st, h = call()
        reached = L.lib.cuemu_fail_alloc_after(-1) < 0
        what = "%s, allocation %d" % (name, k)
        if st == OK:
            try:
                if fetch(h) != want:
                    failures.append("%s: OK but the result differs from the warm-up" % what)
            except AssertionError:
                failures.append("%s: OK but the result cannot be read: %r" % (what, L.error()))
            free(h)
        elif st == ERR_CUDA:
            msg = L.error()
            if msg == SENTINEL or not any(n.encode() in msg for n in names):
                failures.append("%s: last_error %r does not name the call" % (what, msg))
            if h is not None:
                failures.append("%s: *out is not NULL" % what)
        else:
            failures.append("%s: returned %d" % (what, st))
        live = L.lib.cuemu_live_allocs()
        if live != base:
            failures.append("%s: %d allocation(s) left behind" % (what, live - base))
        if not reached:
            if k == 0:
                failures.append("%s: no allocation at all" % name)
            break
    return failures


def out_call(fn):
    """Wraps fn(out_ref) -> status: *out starts non-NULL so that a failed call must clear it."""
    def call():
        out = _vp(0x10)
        st = fn(C.byref(out))
        return st, out if out.value else None
    return call


def mirror_cases(L, rng):
    """(name, call, fetch, free, names) of the entry points that return a mirror."""
    ip, idx, val = rand_csr(rng, 9, 7, 3)
    a = L.upload(CSR, (9, 7), ip, idx, val)
    a_csc = L.upload(CSC, (7, 9), ip, idx, val)  # a CSC mirror (its own shape)
    b_ip, b_idx, b_val = rand_csr(rng, 9, 7, 2)
    b = L.upload(CSR, (9, 7), b_ip, b_idx, b_val)
    fetch, free = L.download, L.csmat_free
    part = ["spmv partition"]
    cases = []
    for storage, shape in ((CSR, (9, 7)), (CSC, (7, 9))):
        cases.append(("upload %d" % storage, out_call(lambda o, s=storage, sh=shape: L.csmat_upload(
            L.ctx, s, sh[0], sh[1], _ptr(ip), 4, _ptr(idx), 4, _f64(val), o)), fetch, free,
            ["upload"] + part))
    L.keep += [ip, idx, val]
    cases.append(("from_device", out_call(lambda o: L.csmat_from_device(
        L.ctx, CSR, 9, 7, len(idx), _ptr(ip), _ptr(idx), _ptr(val), o)), fetch, free,
        ["from_device"] + part))
    tr, tc = rng.integers(0, 9, 30).astype(np.uint32), rng.integers(0, 7, 30).astype(np.uint32)
    tv = rng.standard_normal(30)
    L.keep += [tr, tc, tv]
    cases.append(("from_triplets", out_call(lambda o: L.csmat_from_triplets(
        L.ctx, 9, 7, 30, _ptr(tr), _ptr(tc), 4, _f64(tv), o)), fetch, free,
        ["from_triplets"] + part))
    cases.append(("from_triplets_dev", out_call(lambda o: L.csmat_from_triplets_dev(
        L.ctx, 9, 7, 30, _ptr(tr), _ptr(tc), _ptr(tv), o)), fetch, free,
        ["from_triplets"] + part))
    for nm, m in (("to_other_storage csr", a), ("to_other_storage csc", a_csc)):
        cases.append((nm, out_call(lambda o, m=m: L.csmat_to_other_storage(L.ctx, m, o)), fetch,
                      free, ["to_other_storage"] + part))
    dense = rng.standard_normal((6, 5))
    dense[dense < 0.3] = 0.0
    L.keep.append(dense)
    for storage in (CSR, CSC):
        cases.append(("from_dense %d" % storage, out_call(lambda o, s=storage: L.csmat_from_dense(
            L.ctx, s, 6, 5, _f64(dense), 5, 1, 0.0, o)), fetch, free, ["from_dense"] + part))
    return cases, a, a_csc, b


def main_cases(L, rng):
    cases, a, a_csc, b = mirror_cases(L, rng)
    # SpGEMM: A (9 x 7) * B (7 x 8)
    ip2, idx2, val2 = rand_csr(rng, 7, 8, 3)
    b2 = L.upload(CSR, (7, 8), ip2, idx2, val2)

    def symbolic():
        plan, nnz = _vp(0x10), _u64()
        st = L.spgemm_symbolic(L.ctx, a, b2, C.byref(plan), C.byref(nnz))
        return st, plan if plan.value else None

    def product(plan):
        c = _vp()
        assert L.spgemm_numeric_dev(L.ctx, plan, C.byref(c)) == OK, L.error()
        got = L.download(c)
        L.csmat_free(c)
        return got

    cases.append(("spgemm symbolic", symbolic, product, L.spgemm_free, ["spgemm"]))
    st, plan = symbolic()
    assert st == OK
    cases.append(("spgemm numeric", out_call(lambda o: L.spgemm_numeric_dev(L.ctx, plan, o)),
                  L.download, L.csmat_free, ["spgemm", "spmv partition"]))
    # BiCGSTAB on a square, diagonally dominant matrix (its CSC form takes the cached CSR view)
    sip, sidx, sval = rand_csr(rng, 8, 8, 3, lower=True)
    sq = L.upload(CSC, (8, 8), sip, sidx, sval)
    x0, rhs = np.zeros(8), rng.standard_normal(8)

    def solver_x(h):
        x = np.zeros(8)
        assert L.bicgstab_get(h, 0, _f64(x), 8) == OK
        return x.tobytes()

    cases.append(("bicgstab_new", out_call(lambda o: L.bicgstab_new(
        L.ctx, sq, _f64(x0), _f64(rhs), 8, o)), solver_x, L.bicgstab_free, ["bicgstab"]))
    return cases


def construct_cases(L, rng):
    cases, a, a_csc, b = mirror_cases(L, rng)
    fetch, free, part = L.download, L.csmat_free, ["spmv partition"]
    cases.append(("binop", out_call(lambda o: L.csmat_binop(L.ctx, a, b, 0, o)), fetch, free,
                  ["binop"] + part))
    cases.append(("scale", out_call(lambda o: L.csmat_scale(L.ctx, a_csc, 2.5, o)), fetch, free,
                  ["scale"] + part))
    blocks = (_vp * 4)(a, None, None, b)
    cases.append(("bmat", out_call(lambda o: L.csmat_bmat(L.ctx, 2, 2, blocks, o)), fetch, free,
                  ["bmat"] + part))
    blocks_csc = (_vp * 2)(a, L.upload(CSC, (9, 4), *rand_csr(rng, 4, 9, 2)))
    cases.append(("bmat csc", out_call(lambda o: L.csmat_bmat(L.ctx, 1, 2, blocks_csc, o)), fetch,
                  free, ["bmat"] + part))
    for nm, x, y in (("kron", a, b), ("kron csr csc", a, a_csc), ("kron csc csr", a_csc, a)):
        cases.append((nm, out_call(lambda o, x=x, y=y: L.csmat_kron(L.ctx, x, y, o)), fetch, free,
                      ["kron", "to_other_storage"] + part))
    cases.append(("transpose_view", out_call(lambda o: L.csmat_transpose_view(L.ctx, a_csc, o)),
                  fetch, free, ["transpose_view"] + part))
    return cases


def ldl_cases(L, rng):
    cases = []
    ip, idx, val = rand_csr(rng, 12, 12, 3, lower=True)
    rhs = rng.standard_normal(12)

    def solved(plan):
        x = rhs.copy()
        assert L.trisolve_solve(plan, _f64(x), 12) == OK, L.error()
        return x.tobytes()

    for storage in (CSR, CSC):
        m = L.upload(storage, (12, 12), ip, idx, val)
        cases.append(("trisolve plan %d" % storage, out_call(
            lambda o, m=m: L.trisolve_plan(L.ctx, m, 0, o)), solved, L.trisolve_free,
            ["trisolve", "to_other_storage"]))
    # a symmetric matrix: L + L^T with a heavy diagonal
    d = np.zeros((12, 12))
    for r in range(12):
        for p in range(ip[r], ip[r + 1]):
            d[r, idx[p]] = val[p]
    d = d + d.T + 20 * np.eye(12)
    sip = np.zeros(13, np.uint32)
    sidx, sval = [], []
    for r in range(12):
        nz = np.nonzero(d[r])[0]
        sidx += nz.tolist()
        sval += d[r, nz].tolist()
        sip[r + 1] = len(sidx)
    sidx, sval = np.array(sidx, np.uint32), np.array(sval)
    sym_m = L.upload(CSR, (12, 12), sip, sidx, sval)
    cases.append(("ldl symbolic", out_call(lambda o: L.ldl_symbolic(L.ctx, sym_m, None, 1, o)),
                  L.ldl_nnz, L.ldl_free, ["ldl symbolic"]))
    sym = _vp()
    assert L.ldl_symbolic(L.ctx, sym_m, None, 1, C.byref(sym)) == OK, L.error()

    def diag(num):
        dd = np.zeros(12)
        assert L.ldl_get_d(num, _f64(dd), 12) == OK, L.error()
        return dd.tobytes()

    cases.append(("ldl factor", out_call(lambda o: L.ldl_factor(sym, sym_m, o)), diag, L.ldl_free,
                  ["ldl factor", "trisolve"]))
    return cases


CASES = {"main": main_cases, "construct": construct_cases, "ldl": ldl_cases}


def hooked_library(which, out_dir):
    """The emulated library `which` with cuemu_fail.cpp in place of cuemu.o, built in out_dir."""
    from conftest import emu_library
    from emu_binop import CXXFLAGS, EMU, GEN
    from emu_trisolve import STAND_INS
    emu_library()  # the emulator's objects and the rewritten headers under GEN
    sys.path.insert(0, EMU)
    import transform
    asan = os.environ.get("SPRS_B200_EMU_ASAN") == "1"
    flags = CXXFLAGS + ["-I" + EMU, "-I" + GEN] + (
        ["-fsanitize=address", "-fno-omit-frame-pointer"] if asan else [])
    names = re.search(r"^SRCS = (.*)$", open(os.path.join(EMU, "Makefile")).read(), re.M).group(1)
    objs = [os.path.join(EMU, "build", "asan" if asan else "", n + ".o") for n in names.split()]
    sources = {"main": [], "construct": ["binop.cu", "construct.cu"],
               "ldl": ["trisolve.cu", "ldl.cu"]}[which]
    for name in sources:
        src = transform.transform(name, open(os.path.join(ROOT, "sprs_b200", "csrc", name)).read())
        cpp = os.path.join(out_dir, name[:-3] + ".cpp")
        with open(cpp, "w") as f:
            f.write((STAND_INS if which == "ldl" else "") + src)
        objs.append(cpp)
    objs.append(os.path.join(EMU, "cuemu_fail.cpp"))
    so = os.path.join(out_dir, "libsprs_b200_emu_%s.so" % which)
    subprocess.check_call(["/usr/bin/g++", "-shared"] + flags + ["-o", so] + objs)
    return so


def run(which, path):
    L = Lib(path)
    cases = CASES[which](L, np.random.default_rng(11))
    failures = []
    for name, call, fetch, free, names in cases:
        failures += check(L, name, call, fetch, free, names)
    print("%d entry points checked" % len(cases))
    for f in failures:
        print("FAIL " + f)
    return 1 if failures else 0


@pytest.mark.parametrize("which", ["main", "construct", "ldl"])
def test_emu_alloc_failure(which, tmp_path):
    so = hooked_library(which, str(tmp_path))
    env = dict(os.environ, SPRS_B200_SPMV_HOT="4")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), which, so], env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert "entry points checked" in r.stdout


if __name__ == "__main__":
    sys.exit(run(sys.argv[1], sys.argv[2]))
