"""ctypes front-end of the CPU trisolve oracle (tests/trisolve_oracle.cpp).

TEST INFRASTRUCTURE ONLY: the restatement of lsolve_csr_dense_rhs, usolve_csr_dense_rhs,
lsolve_csc_dense_rhs and usolve_csc_dense_rhs (sprs/src/sparse/linalg/trisolve.rs) that the
device solves are compared with bit for bit, and `levels`, the depth of a solve's dependency
graph.  Compiled on first use (g++, -ffp-contract=off: no FMA, like sprs) into a per-user cache
directory outside the tree.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "trisolve_oracle.cpp")
_LIB = None
FORMS = ("lsolve_csr", "usolve_csr", "lsolve_csc", "usolve_csc")
REASONS = ("diagonal element is 0", "diagonal element is a numeric 0",
           "diagonal element is a structural 0")


def build():
    """Path of the compiled oracle, built when its source changed."""
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), "sprs_b200_test_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "liboracle_trisolve_%s.so" % hashlib.sha1(src).hexdigest()[:12])
    if not os.path.exists(so):
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off",
                               "-Wall", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.oracle_levels.restype = C.c_uint64
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _arrays(indptr, indices, data):
    ip = np.ascontiguousarray(np.asarray(indptr).astype(np.int64) - int(indptr[0])).astype(np.uint64)
    return (ip, np.ascontiguousarray(indices, dtype=np.uint32),
            np.ascontiguousarray(data, dtype=np.float64))


def solve(form, indptr, indices, data, rhs):
    """The reference's `form` (one of FORMS) on a square matrix of len(indptr) - 1 outer
    dimensions, rhs (float64, contiguous) solved in place.  Returns None for Ok, else
    (index, reason) of the SingularMatrix, with rhs left as the reference leaves it."""
    assert form in FORMS and rhs.dtype == np.float64 and rhs.flags.c_contiguous
    ip, ind, dat = _arrays(indptr, indices, data)
    n = len(ip) - 1
    assert rhs.size == n
    index = C.c_uint64(0)
    st = getattr(lib(), "oracle_" + form)(C.c_uint64(n), _p(ip), _p(ind), _p(dat), _p(rhs),
                                          C.byref(index))
    return None if st == 0 else (int(index.value), REASONS[st - 1])


def levels(indptr, indices, upper, csr=True):
    """Depth of the dependency graph of the lower (upper=False) or upper solve: the number of
    rows on its longest chain of dependent rows (n for a bidiagonal chain, 1 for a diagonal)."""
    ip = np.ascontiguousarray(np.asarray(indptr).astype(np.int64) - int(indptr[0])).astype(np.uint64)
    ind = np.ascontiguousarray(indices, dtype=np.uint32)
    n = len(ip) - 1
    lv = np.empty(max(n, 1), dtype=np.uint32)
    return int(lib().oracle_levels(C.c_uint64(n), _p(ip), _p(ind), C.c_int(int(upper)),
                                   C.c_int(int(csr)), _p(lv)))


def first_difference(got, want):
    """None when two vectors agree bit for bit on view(np.uint64), whole vectors, else a
    description of the first difference.  NaN is compared by class: the GPU and the host CPU
    generate different NaN payloads, and no payload is part of the reference's contract."""
    gf, wf = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if gf.shape != wf.shape:
        return "shapes differ: %s vs %s" % (gf.shape, wf.shape)
    g, w = gf.view(np.uint64), wf.view(np.uint64)
    bad = np.flatnonzero((g != w) & ~(np.isnan(gf) & np.isnan(wf)))
    if bad.size:
        k = int(bad[0])
        return "%d entries differ, first at %d: got %r want %r" % (
            bad.size, k, float(np.asarray(got)[k]), float(np.asarray(want)[k]))
    return None
