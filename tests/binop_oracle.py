"""ctypes front-end of the CPU binop oracle (tests/binop_oracle.cpp).

TEST INFRASTRUCTURE ONLY: the restatement of csmat_binop_same_storage_raw (binop.rs:229-271) and
CsMatBase::map that the device results of `&A + &B`, `&A - &B`, mul_mat_same_storage and
`&A * s` are compared with, structure and values bit for bit.  Compiled on first use (g++,
-ffp-contract=off: no FMA, like sprs) into a per-user cache directory outside the tree.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "binop_oracle.cpp")
_LIB = None
ADD, SUB, MUL = 0, 1, 2


def build():
    """Path of the compiled oracle, built when its source changed."""
    src = open(_SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), "sprs_b200_test_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "liboracle_binop_%s.so" % hashlib.sha1(src).hexdigest()[:12])
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
        for suf in ("44", "88", "48"):
            getattr(_LIB, "oracle_binop_" + suf).restype = C.c_size_t
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _suffix(indptr, indices):
    suf = {(4, 4): "44", (8, 8): "88", (4, 8): "48"}.get((indices.dtype.itemsize,
                                                          indptr.dtype.itemsize))
    if suf is None:
        raise TypeError("the binop oracle supports (I, Iptr) byte widths (4,4), (8,8), (4,8)")
    return suf


def binop(op, a, b):
    """csmat_binop_same_storage_raw with f = + (ADD), - (SUB) or * (MUL).  a, b = (indptr,
    indices, data) of the same storage and shape, the same index dtypes; returns the result's
    (indptr, indices, data) in those dtypes."""
    aip, aind, ad = (np.ascontiguousarray(x) for x in a)
    bip, bind, bd = (np.ascontiguousarray(x) for x in b)
    ad = np.ascontiguousarray(ad, dtype=np.float64)
    bd = np.ascontiguousarray(bd, dtype=np.float64)
    bip, bind = bip.astype(aip.dtype, copy=False), bind.astype(aind.dtype, copy=False)
    assert len(aip) == len(bip)
    outer = len(aip) - 1
    cap = int(aip[-1] - aip[0]) + int(bip[-1] - bip[0])
    oip = np.empty(outer + 1, dtype=aip.dtype)
    oind = np.empty(max(cap, 1), dtype=aind.dtype)
    od = np.empty(max(cap, 1), dtype=np.float64)
    f = getattr(lib(), "oracle_binop_" + _suffix(aip, aind))
    n = f(C.c_int(op), C.c_size_t(outer), _p(aip), _p(aind), _p(ad), _p(bip), _p(bind), _p(bd),
          _p(oip), _p(oind), _p(od))
    return oip, oind[:n].copy(), od[:n].copy()


def scale(a, s):
    """CsMatBase::map(|x| x * s): same structure, every stored value times s (zeros kept)."""
    ip, ind, d = a
    d = np.ascontiguousarray(d, dtype=np.float64)
    out = np.empty_like(d)
    lib().oracle_scale(C.c_size_t(d.size), _p(d), C.c_double(s), _p(out))
    return np.array(ip, copy=True), np.array(ind, copy=True), out


def _host(indptr, indices, data, r0, r1):
    """rows [r0, r1) of a device (or CPU) CSR as zero-based host arrays (u64 indptr, u32
    indices); torch int32 storage of u32 values is read back as u32."""
    ip = indptr[r0:r1 + 1].cpu().numpy()
    ip = ip.view(np.uint32).astype(np.uint64) if ip.dtype == np.int32 else ip.astype(np.uint64)
    s, e = int(ip[0]), int(ip[-1])
    return (ip - ip[0], indices[s:e].cpu().numpy().view(np.uint32), data[s:e].cpu().numpy())


def first_difference(got, want):
    """None when (indptr, indices, data) agree -- structure exact, values bit for bit, NaN by
    class -- else a description of the first difference."""
    gi, gj, gd = got
    wi, wj, wd = want
    if not np.array_equal(np.asarray(gi, np.int64), np.asarray(wi, np.int64)):
        r = int(np.flatnonzero(np.asarray(gi, np.int64) != np.asarray(wi, np.int64))[0]) \
            if len(gi) == len(wi) else -1
        return "indptr differs (first at %d)" % r
    if not np.array_equal(np.asarray(gj, np.int64), np.asarray(wj, np.int64)):
        return "indices differ at %d" % int(np.flatnonzero(np.asarray(gj, np.int64) !=
                                                           np.asarray(wj, np.int64))[0])
    gd, wd = np.asarray(gd, np.float64), np.asarray(wd, np.float64)
    gn, wn = np.isnan(gd), np.isnan(wd)
    bad = (gn != wn) | (~wn & (gd.view(np.uint64) != wd.view(np.uint64)))
    if bad.any():
        k = int(np.flatnonzero(bad)[0])
        return "data differs at %d: got %r want %r" % (k, gd[k], wd[k])
    return None


def compare_chunked(op, a, b, c, outer, chunk=1 << 18):
    """The device result c of `a op b` (op = ADD / SUB / MUL, or ("scale", s) with b = None)
    against this oracle, outer dimension by outer dimension in chunks: a, b, c are
    (indptr, indices, data) torch tensors of one storage.  Every chunk is compared whole.
    Returns (first difference or None, seconds spent in the oracle calls)."""
    import time
    spent = 0.0
    for r0 in range(0, max(outer, 1), chunk):
        r1 = min(r0 + chunk, outer)
        ha = _host(*a, r0, r1)
        t0 = time.perf_counter()
        if isinstance(op, tuple):
            want = scale(ha, op[1])
        else:
            want = binop(op, ha, _host(*b, r0, r1))
        spent += time.perf_counter() - t0
        err = first_difference(_host(*c, r0, r1), want)
        if err:
            return "rows %d..%d: %s" % (r0, r1, err), spent
    return None, spent
