"""ctypes front-end of the CPU LDL^T oracle (tests/ldl_oracle.cpp).

TEST INFRASTRUCTURE ONLY: the restatement of the sprs-ldl crate (ldl_symbolic, ldl_numeric,
ldl_lsolve, ldl_ltsolve), linalg::diag_solve and `&perm * v` that the device factorization is
compared with bit for bit, and `etree_height`.  Compiled on first use (g++, -ffp-contract=off:
no FMA, like sprs) into a per-user cache directory outside the tree.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ldl_oracle.cpp")
_LIB = None
NONE = np.iinfo(np.uint64).max


def build():
    """Path of the compiled oracle, built when its source changed."""
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), "sprs_b200_test_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "liboracle_ldl_%s.so" % hashlib.sha1(src).hexdigest()[:12])
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
        _LIB.oracle_ldl_numeric.restype = C.c_uint64
        _LIB.oracle_etree_height.restype = C.c_uint64
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u64(a):
    return np.ascontiguousarray(np.asarray(a).astype(np.uint64))


def _perm(n, perm):
    p = np.arange(n, dtype=np.uint64) if perm is None else _u64(perm)
    pinv = np.empty(n, dtype=np.uint64)
    pinv[p.astype(np.int64)] = np.arange(n, dtype=np.uint64)
    return p, pinv


class Factor:
    """The reference's LdlSymbolic + LdlNumeric on one pattern and permutation: `update`
    reruns ldl_numeric with the workspaces carried over, as LdlNumeric::update does."""

    def __init__(self, indptr, indices, perm=None):
        self.ip = _u64(np.asarray(indptr).astype(np.int64) - int(indptr[0]))
        self.idx = np.ascontiguousarray(indices, dtype=np.uint32)
        n = self.n = len(self.ip) - 1
        self.perm, self.pinv = _perm(n, perm)
        self.colptr = np.zeros(n + 1, dtype=np.uint64)
        self.parent = np.zeros(max(n, 1), dtype=np.uint64)
        self.l_nz = np.zeros(max(n, 1), dtype=np.uint64)
        self.flag = np.zeros(max(n, 1), dtype=np.uint64)
        lib().oracle_ldl_symbolic(C.c_uint64(n), _p(self.ip), _p(self.idx), _p(self.perm),
                                  _p(self.pinv), _p(self.colptr), _p(self.parent), _p(self.l_nz),
                                  _p(self.flag))
        nnz = int(self.colptr[-1])
        self.l_idx = np.zeros(max(nnz, 1), dtype=np.uint64)
        self.l_val = np.zeros(max(nnz, 1), dtype=np.float64)
        self.d = np.zeros(max(n, 1), dtype=np.float64)
        self.y = np.zeros(max(n, 1), dtype=np.float64)

    def nnz(self):
        return int(self.colptr[-1])

    def update(self, data):
        """ldl_numeric with these values: None for Ok, else the SingularMatrix index."""
        val = np.ascontiguousarray(data, dtype=np.float64)
        r = int(lib().oracle_ldl_numeric(
            C.c_uint64(self.n), _p(self.ip), _p(self.idx), _p(val), _p(self.perm), _p(self.pinv),
            _p(self.colptr), _p(self.parent), _p(self.l_nz), _p(self.l_idx), _p(self.l_val),
            _p(self.d), _p(self.y), _p(self.flag)))
        return None if r == 0 else r - 1

    def l(self):  # noqa: E743
        """(colptr, row indices, values) of L."""
        nnz = self.nnz()
        return self.colptr.copy(), self.l_idx[:nnz].copy(), self.l_val[:nnz].copy()

    def diag(self):
        return self.d[:self.n].copy()

    def solve(self, b):
        """LdlNumeric::solve: perm * b, ldl_lsolve, diag_solve, ldl_ltsolve, pinv * x."""
        x = perm_mul(self.perm, b)
        cp, li, lv = self.l()
        lsolve(cp, li, lv, x)
        diag_solve(self.diag(), x)
        ltsolve(cp, li, lv, x)
        return perm_mul(self.pinv, x)

    def etree_height(self):
        depth = np.zeros(max(self.n, 1), dtype=np.uint64)
        return int(lib().oracle_etree_height(C.c_uint64(self.n), _p(self.parent), _p(depth)))


def lsolve(colptr, l_idx, l_val, x):
    """ldl_lsolve, x (float64, contiguous) in place."""
    cp, li = _u64(colptr), _u64(l_idx)
    lv = np.ascontiguousarray(l_val, dtype=np.float64)
    lib().oracle_ldl_lsolve(C.c_uint64(len(cp) - 1), _p(cp), _p(li), _p(lv), _p(x))


def ltsolve(colptr, l_idx, l_val, x):
    """ldl_ltsolve, x in place."""
    cp, li = _u64(colptr), _u64(l_idx)
    lv = np.ascontiguousarray(l_val, dtype=np.float64)
    lib().oracle_ldl_ltsolve(C.c_uint64(len(cp) - 1), _p(cp), _p(li), _p(lv), _p(x))


def diag_solve(d, x):
    d = np.ascontiguousarray(d, dtype=np.float64)
    lib().oracle_diag_solve(C.c_uint64(x.size), _p(d), _p(x))


def perm_mul(perm, v):
    p = _u64(perm)
    v = np.ascontiguousarray(v, dtype=np.float64)
    out = np.empty(p.size, dtype=np.float64)
    lib().oracle_perm_mul(C.c_uint64(p.size), _p(p), _p(v), _p(out))
    return out


def first_difference(got, want):
    """None when two arrays agree bit for bit (NaN by class), else the first difference."""
    from trisolve_oracle import first_difference as fd
    return fd(got, want)
