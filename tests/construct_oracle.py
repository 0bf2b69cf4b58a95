"""ctypes front-end of the CPU construction oracle (tests/construct_oracle.cpp).

TEST INFRASTRUCTURE ONLY.  The C++ side holds the primitives (to_other_storage as a counting
transpose, same_storage_fast_stack, the Kronecker double loop); this module restates, line by
line, how construct.rs composes them:

  vstack(mats)   every CSR? stack them; else to_csr every matrix, then stack
  hstack(mats)   every CSC? stack them; else to_csc every matrix, then stack
  bmat(blocks)   asserts; rows_per_row / cols_per_col; None -> zero(shape); hstack each block
                 row; vstack the rows

It does NOT restate the device's direct design (one output indptr, per-block column offsets), so
the block-row offset rule is checked against the reference's composition, not against itself.
Matrices are Mat(storage, shape, indptr, indices, data) with u64 zero-based arrays.  Compiled on
first use (g++, -ffp-contract=off) into a per-user cache directory outside the tree.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from collections import namedtuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "construct_oracle.cpp")
_LIB = None

Mat = namedtuple("Mat", "storage shape indptr indices data")


class Panic(AssertionError):
    """A panic of the reference's composition (the message is the reference's)."""


def build():
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), "sprs_b200_test_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "liboracle_construct_%s.so" % hashlib.sha1(src).hexdigest()[:12])
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
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def mat(storage, shape, indptr, indices, data):
    ip = np.asarray(indptr).astype(np.int64)
    ip = (ip - ip[0]).astype(np.uint64)
    n = int(ip[-1])
    return Mat(storage, (int(shape[0]), int(shape[1])), ip,
               np.ascontiguousarray(np.asarray(indices)[:n], dtype=np.uint64),
               np.ascontiguousarray(np.asarray(data, dtype=np.float64)[:n]))


def of(m):
    """Mat of a sprs_b200.CsMat (host arrays)."""
    return mat(m.storage, m.shape, m.indptr, m.indices, m.data)


def outer_dims(m):
    return m.shape[0] if m.storage == "CSR" else m.shape[1]


def inner_dims(m):
    return m.shape[1] if m.storage == "CSR" else m.shape[0]


def zero(shape):
    return Mat("CSR", shape, np.zeros(shape[0] + 1, np.uint64), np.zeros(0, np.uint64),
               np.zeros(0))


def transpose_view(m):
    return Mat("CSC" if m.storage == "CSR" else "CSR", (m.shape[1], m.shape[0]), m.indptr,
               m.indices, m.data)


def to_other_storage(m):
    outer, inner = outer_dims(m), inner_dims(m)
    nnz = int(m.indptr[-1])
    ip = np.empty(inner + 1, np.uint64)
    ind = np.empty(max(nnz, 1), np.uint64)
    dat = np.empty(max(nnz, 1))
    lib().oracle_convert(C.c_uint64(outer), C.c_uint64(inner), _p(m.indptr), _p(m.indices),
                         _p(m.data), _p(ip), _p(ind), _p(dat))
    return Mat("CSC" if m.storage == "CSR" else "CSR", m.shape, ip, ind[:nnz], dat[:nnz])


def to_csr(m):
    return m if m.storage == "CSR" else to_other_storage(m)


def to_csc(m):
    return m if m.storage == "CSC" else to_other_storage(m)


def same_storage_fast_stack(mats):
    if not mats:
        raise Panic("Empty stacking list")
    inner = inner_dims(mats[0])
    if any(inner_dims(m) != inner for m in mats):
        raise Panic("Dimension mismatch")
    storage = mats[0].storage
    if any(m.storage != storage for m in mats):
        raise Panic("Storage mismatch")
    outers = np.array([outer_dims(m) for m in mats], np.uint64)
    ips = np.ascontiguousarray(np.concatenate([m.indptr for m in mats]))
    inds = np.ascontiguousarray(np.concatenate([m.indices for m in mats] + [np.zeros(1, np.uint64)]))
    dats = np.ascontiguousarray(np.concatenate([m.data for m in mats] + [np.zeros(1)]))
    nnz = sum(int(m.indptr[-1]) for m in mats)
    ip = np.empty(int(outers.sum()) + 1, np.uint64)
    ind = np.empty(max(nnz, 1), np.uint64)
    dat = np.empty(max(nnz, 1))
    lib().oracle_stack(C.c_uint64(len(mats)), _p(outers), _p(ips), _p(inds), _p(dats), _p(ip),
                       _p(ind), _p(dat))
    outer = int(outers.sum())
    shape = (outer, inner) if storage == "CSR" else (inner, outer)
    return Mat(storage, shape, ip, ind[:nnz], dat[:nnz])


def vstack(mats):
    if all(m.storage == "CSR" for m in mats):
        return same_storage_fast_stack(mats)
    return same_storage_fast_stack([to_csr(m) for m in mats])


def hstack(mats):
    if all(m.storage == "CSC" for m in mats):
        return same_storage_fast_stack(mats)
    return same_storage_fast_stack([to_csc(m) for m in mats])


def bmat(blocks):
    super_rows = len(blocks)
    if super_rows == 0:
        raise Panic("Empty stacking list")
    super_cols = len(blocks[0])
    if super_cols == 0:
        raise Panic("Empty stacking list")
    if not all(len(x) == super_cols for x in blocks):
        raise Panic("Dimension mismatch")
    if any(all(m is None for m in x) for x in blocks):
        raise Panic("Empty bmat row")
    if any(all(x[j] is None for x in blocks) for j in range(super_cols)):
        raise Panic("Empty bmat col")
    rows_per_row = [max([m.shape[0] for m in row if m is not None] + [0]) for row in blocks]
    cols_per_col = [max([row[j].shape[1] for row in blocks if row[j] is not None] + [0])
                    for j in range(super_cols)]
    to_vstack = []
    for i, row in enumerate(blocks):
        with_zeros = [m if m is not None else zero((rows_per_row[i], cols_per_col[j]))
                      for j, m in enumerate(row)]
        to_vstack.append(hstack(with_zeros))
    return vstack(to_vstack)


def kronecker_product(a, b):
    if a.storage != b.storage:
        return kronecker_product(a, to_other_storage(b))
    was_csc = a.storage == "CSC"
    if was_csc:
        a, b = transpose_view(a), transpose_view(b)
    nnz = int(a.indptr[-1]) * int(b.indptr[-1])
    shape = (a.shape[0] * b.shape[0], a.shape[1] * b.shape[1])
    ip = np.empty(shape[0] + 1, np.uint64)
    ind = np.empty(max(nnz, 1), np.uint64)
    dat = np.empty(max(nnz, 1))
    lib().oracle_kron(C.c_uint64(a.shape[0]), _p(a.indptr), _p(a.indices), _p(a.data),
                      C.c_uint64(b.shape[0]), C.c_uint64(b.shape[1]), _p(b.indptr),
                      _p(b.indices), _p(b.data), _p(ip), _p(ind), _p(dat))
    m = Mat("CSR", shape, ip, ind[:nnz], dat[:nnz])
    return transpose_view(m) if was_csc else m


def to_dense(m):
    out = np.zeros(m.shape)
    for o in range(outer_dims(m)):
        for k in range(int(m.indptr[o]), int(m.indptr[o + 1])):
            i = int(m.indices[k])
            if m.storage == "CSR":
                out[o, i] = m.data[k]
            else:
                out[i, o] = m.data[k]
    return out


def first_difference(got, want, kron=False):
    """None when got and want (Mat or anything with storage/shape/indptr/indices/data) agree:
    storage, shape and structure exact, values bit for bit -- NaN payloads included, or, with
    kron=True, NaN compared by position (a product's NaN payload is the hardware's)."""
    if got.storage != want.storage or tuple(got.shape) != tuple(want.shape):
        return "storage/shape %s %s vs %s %s" % (got.storage, got.shape, want.storage, want.shape)
    gi = np.asarray(got.indptr).astype(np.int64)
    wi = np.asarray(want.indptr).astype(np.int64)
    gi, wi = gi - gi[0], wi - wi[0]
    if not np.array_equal(gi, wi):
        return "indptr differs"
    n = int(wi[-1])
    gj, wj = np.asarray(got.indices)[:n].astype(np.int64), np.asarray(want.indices)[:n].astype(np.int64)
    if not np.array_equal(gj, wj):
        return "indices differ at %d" % int(np.flatnonzero(gj != wj)[0])
    gd = np.ascontiguousarray(np.asarray(got.data, np.float64)[:n])
    wd = np.ascontiguousarray(np.asarray(want.data, np.float64)[:n])
    if kron:
        gn, wn = np.isnan(gd), np.isnan(wd)
        bad = (gn != wn) | (~wn & (gd.view(np.uint64) != wd.view(np.uint64)))
    else:
        bad = gd.view(np.uint64) != wd.view(np.uint64)
    if bad.any():
        k = int(np.flatnonzero(bad)[0])
        return "data differs at %d: got %r want %r" % (k, gd[k], wd[k])
    return None
