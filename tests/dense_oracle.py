"""ctypes front-end of the CPU oracle of the dense boundary (tests/dense_oracle.cpp).

TEST INFRASTRUCTURE ONLY: the restatement of assign_to_dense (to_dense.rs:12-30), csr_from_dense /
csc_from_dense (csmat.rs:502-549) and csmat_binop_dense_raw with the add / mul closures
(binop.rs:273-433) that the device results are compared with bit for bit.  Compiled on first use
(g++, -ffp-contract=off: no FMA, like sprs) into a per-user cache directory outside the tree.
Dense operands are numpy views of any strides; they are passed by pointer and element strides.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dense_oracle.cpp")
_LIB = None
ADD, MUL = 0, 2


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), "sprs_b200_test_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "liboracle_dense_%s.so" % hashlib.sha1(src).hexdigest()[:12])
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
        _LIB.oracle_csr_from_dense.restype = C.c_uint64
        _LIB.oracle_csr_from_dense.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_int64,
                                               C.c_int64, C.c_double, C.c_void_p, C.c_void_p,
                                               C.c_void_p]
        _LIB.oracle_assign_to_dense.argtypes = [C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_int64, C.c_int64]
        _LIB.oracle_binop_dense.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p,
                                            C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64]
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a.size else C.c_void_p(0)


def _st(a):
    return a.strides[0] // 8, a.strides[1] // 8


def _sparse(m):
    """(storage code, outer, u64 indptr rebased to 0, u64 indices, f64 data) of a CsMat-like"""
    ip = np.asarray(m.indptr).astype(np.uint64)
    ip = ip - ip[0]
    nnz = int(ip[-1])
    return (0 if m.storage == "CSR" else 1, len(ip) - 1, np.ascontiguousarray(ip),
            np.ascontiguousarray(np.asarray(m.indices)[:nnz], dtype=np.uint64),
            np.ascontiguousarray(np.asarray(m.data)[:nnz], dtype=np.float64))


def assign_to_dense(array, m):
    """in place into the writeable view `array` (shape already checked by the caller)"""
    st, outer, ip, idx, d = _sparse(m)
    rs, cs = _st(array)
    lib().oracle_assign_to_dense(st, outer, _p(ip), _p(idx), _p(d), C.c_void_p(array.ctypes.data),
                                 rs, cs)


def to_dense(m):
    out = np.zeros(m.shape)
    if out.size:
        assign_to_dense(out, m)
    return out


def csr_from_dense(m, epsilon):
    """(indptr u64, indices u64, data) of csr_from_dense(m, epsilon)"""
    rows, cols = m.shape
    ip = np.zeros(rows + 1, np.uint64)
    idx = np.zeros(max(rows * cols, 1), np.uint64)
    d = np.zeros(max(rows * cols, 1))
    rs, cs = _st(m) if m.size else (0, 0)
    nnz = lib().oracle_csr_from_dense(rows, cols, C.c_void_p(m.ctypes.data) if m.size else None,
                                      rs, cs, float(epsilon), _p(ip), _p(idx), _p(d))
    return ip, idx[:nnz], d[:nnz]


def csc_from_dense(m, epsilon):
    """csr_from_dense(m.reversed_axes(), epsilon).transpose_into(): the same arrays, read as CSC"""
    return csr_from_dense(m.T, epsilon)


def binop_dense(m, op, alpha, beta, rhs, out):
    """csmat_binop_dense_raw(m, rhs, closure, out) after its checks; out written in place"""
    st, _, ip, idx, d = _sparse(m)
    rows, cols = rhs.shape
    if rows == 0 or cols == 0:
        return
    rrs, rcs = _st(rhs)
    ors, ocs = _st(out)
    lib().oracle_binop_dense(st, rows, cols, _p(ip), _p(idx), _p(d), op, float(alpha), float(beta),
                             C.c_void_p(rhs.ctypes.data), rrs, rcs, C.c_void_p(out.ctypes.data),
                             ors, ocs)


def same_bits(a, b):
    """exact bits, NaN payloads included (copies)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64),
                                                 np.ascontiguousarray(b).view(np.uint64))


def same_values(a, b):
    """exact bits with NaN compared by class (arithmetic results: a NaN's payload is the
    hardware's choice)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    if not np.array_equal(na, nb):
        return False
    return np.array_equal(np.ascontiguousarray(np.where(na, 0.0, a)).view(np.uint64),
                          np.ascontiguousarray(np.where(nb, 0.0, b)).view(np.uint64))
