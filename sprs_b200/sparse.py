"""Host-side mirror of the sprs operator API for the product path.

The reference's host language is Rust and this image has no Rust toolchain
(DESIGN.md); this module is the Python stand-in for the `sprs-b200` safe wrapper
crate (rust/sprs-b200, source only) so that the parity tests read like the
reference's own tests.  Same names, argument meaning and error behaviour:

  CsMat / CsMat.new_csc / CsMat.eye   sprs/src/sparse/csmat.rs (constructors)
  a @ b, a * b, a.dot(b)              `impl Mul`/`Dot` sprs/src/sparse/csmat.rs:1866-2178,
                                      sprs/src/sparse/vec.rs:1084-1131
  prod.mul_acc_mat_vec_csr, ...       sprs/src/sparse/prod.rs
  smmp.mul_csr_csr, symbolic+numeric  sprs/src/sparse/smmp.rs
  a + b, a - b, a * s                 `impl Add/Sub/Mul<N>` sprs/src/sparse/binop.rs:20-163
  binop.mul_mat_same_storage          sprs/src/sparse/binop.rs:115-130
  to_dense, assign_to_dense           sprs/src/sparse/csmat.rs:1127-1134, to_dense.rs:12-30
  csr_from_dense / csc_from_dense     sprs/src/sparse/csmat.rs:502-549
  a + D, binop.{add,mul}_dense_...    csmat.rs:1951-1987, binop.rs:273-433

Contract violations raise SprsPanic with the reference's panic message
("Dimension mismatch", "Storage mismatch"; sprs Guidelines.rst:9-27); device
failures raise ThirdPartyError(code, msg) like LinalgError::ThirdPartyError
(sprs/src/errors.rs:70).  All arithmetic happens in libsprs_b200.so on the GPU.
"""
import ctypes as C
import threading

import numpy as np

from . import _lib

CSR, CSC = "CSR", "CSC"
_STOR = {CSR: _lib.CSR, CSC: _lib.CSC}


class SprsPanic(AssertionError):
    """A contract violation the reference answers with panic!/assert!."""


class ThirdPartyError(RuntimeError):
    """LinalgError::ThirdPartyError(code, msg) (sprs/src/errors.rs:70)."""

    def __init__(self, code, msg):
        super().__init__("sprs_b200 error %d: %s" % (code, msg))
        self.code = code
        self.msg = msg


class SingularMatrix(ArithmeticError):
    """LinalgError::SingularMatrix(SingularMatrixInfo{index, reason}) (sprs/src/errors.rs:59-69),
    displayed as the reference displays it: "Singular matrix at index {index} ({reason})"."""

    def __init__(self, index, reason):
        super().__init__("Singular matrix at index %d (%s)" % (index, reason))
        self.index = index
        self.reason = reason


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else C.c_void_p(0)


class Context:
    """One device + stream (sprs_b200_ctx).  `Context.default()` is per-thread,
    like the reference's thread-local ThreadingStrategy (smmp.rs:35-38)."""
    _tls = threading.local()

    def __init__(self, device=0):
        self.lib = _lib.load()
        h = C.c_void_p()
        st = self.lib.sprs_b200_ctx_create(int(device), C.byref(h))
        if st != _lib.OK:
            raise ThirdPartyError(st, self.lib.sprs_b200_last_error(None).decode())
        self.h = h
        self.device = device

    @classmethod
    def default(cls, device=None):
        cur = getattr(cls._tls, "ctx", None)
        if cur is None or (device is not None and cur.device != device):
            cur = cls(device or 0)
            cls._tls.ctx = cur
        return cur

    def check(self, st):
        if st == _lib.OK:
            return
        msg = self.lib.sprs_b200_last_error(self.h).decode()
        if st == _lib.ERR_DIMENSION:
            raise SprsPanic("Dimension mismatch")
        if st == _lib.ERR_STORAGE:
            raise SprsPanic("Storage mismatch")
        if st == _lib.ERR_INDEX_RANGE:
            raise SprsPanic(msg or "Index type is not large enough to hold the value")
        if st == _lib.ERR_SINGULAR:  # message: "Singular matrix at index {i} ({reason})"
            head, _, reason = msg.partition(" (")
            raise SingularMatrix(int(head.rsplit(" ", 1)[-1]), reason[:-1])
        if st == _lib.ERR_NOT_SYMMETRIC:
            raise SprsPanic(msg)
        raise ThirdPartyError(st, msg)

    def synchronize(self):
        self.check(self.lib.sprs_b200_ctx_synchronize(self.h))

    @property
    def sm_count(self):
        return self.lib.sprs_b200_ctx_sm_count(self.h)

    @property
    def launches(self):
        return int(self.lib.sprs_b200_launch_count(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.lib.sprs_b200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceCsMat:
    """Owning handle of a device mirror (sprs_b200_csmat); freed like Rust `Drop`."""

    def __init__(self, ctx, handle, keepalive=None):
        self.ctx, self.h, self._keep = ctx, handle, keepalive

    @property
    def rows(self):
        return int(self.ctx.lib.sprs_b200_csmat_rows(self.h))

    @property
    def cols(self):
        return int(self.ctx.lib.sprs_b200_csmat_cols(self.h))

    @property
    def nnz(self):
        return int(self.ctx.lib.sprs_b200_csmat_nnz(self.h))

    @property
    def storage(self):
        return CSR if self.ctx.lib.sprs_b200_csmat_storage(self.h) == _lib.CSR else CSC

    def to_other_storage(self):
        out = C.c_void_p()
        self.ctx.check(self.ctx.lib.sprs_b200_csmat_to_other_storage(self.ctx.h, self.h,
                                                                      C.byref(out)))
        return DeviceCsMat(self.ctx, out)

    def download(self, index_dtype=np.uint32, indptr_dtype=None):
        indptr_dtype = indptr_dtype or index_dtype
        outer = self.rows if self.storage == CSR else self.cols
        ip = np.empty(outer + 1, dtype=indptr_dtype)
        ind = np.empty(self.nnz, dtype=index_dtype)
        dat = np.empty(self.nnz, dtype=np.float64)
        self.ctx.check(self.ctx.lib.sprs_b200_csmat_download(
            self.ctx.h, self.h, _ptr(ip), ip.dtype.itemsize, _ptr(ind), ind.dtype.itemsize,
            _ptr(dat)))
        return ip, ind, dat

    def free(self):
        if self.h:
            self.ctx.lib.sprs_b200_csmat_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class CsVec:
    """CsVecBase{dim, indices, data} (sprs/src/sparse.rs:166-182)."""

    def __init__(self, dim, indices, data):
        self.dim = int(dim)
        self.indices = np.asarray(indices, dtype=np.int64)
        self.data = np.asarray(data, dtype=np.float64)
        if self.indices.shape != self.data.shape:
            raise SprsPanic("indices and data lengths differ")
        if self.indices.size and (np.any(np.diff(self.indices) <= 0) or
                                  self.indices[-1] >= self.dim):
            raise SprsPanic("Unsorted or out-of-bounds indices")

    @classmethod
    def empty(cls, dim):
        return cls(dim, [], [])

    def nnz(self):
        return int(self.indices.size)

    def to_dense(self):
        x = np.zeros(self.dim)
        x[self.indices] = self.data
        return x

    def __eq__(self, o):
        return (isinstance(o, CsVec) and self.dim == o.dim and
                np.array_equal(self.indices, o.indices) and np.array_equal(self.data, o.data))

    def __repr__(self):
        return "CsVec(dim=%d, indices=%s, data=%s)" % (self.dim, self.indices.tolist(),
                                                        self.data.tolist())

    def _merge_dot(self, dim, idx, dat, start=0.0):
        """Sum of self[i] * rhs[i] over the common pattern in ascending index order (dot_acc,
        vec.rs:846-881) on the device: row_view(self) through the merge-dot kernel
        (csrc/csvec.cu) -- the reference's terms in the reference's order, added one by one to
        `start`."""
        if self.nnz() == 0 or len(idx) == 0:
            return start
        row = CsMat((1, dim), np.array([0, self.nnz()]), self.indices, self.data)
        ctx = row.context()
        vi = np.ascontiguousarray(idx, dtype=np.uint64)
        vd = np.ascontiguousarray(dat, dtype=np.float64)
        y = np.array([start], dtype=np.float64)
        ctx.check(ctx.lib.sprs_b200_csr_mul_csvec_acc(ctx.h, row.device().h, dim, vi.size, _ptr(vi),
                                                      8, _ptr(vd), _ptr(y), 1))
        return float(y[0])

    def dot(self, rhs):
        """CsVecBase::dot / dot_acc (vec.rs:825-881): rhs is a CsVec (sorted-merge dot) or any
        dense vector (every entry of self meets one of rhs).  Panics if the dimensions differ
        (`assert_eq!(self.dim(), rhs.dim())`, vec.rs:856)."""
        if isinstance(rhs, CsVec):
            if self.dim != rhs.dim:
                raise SprsPanic("Dimension mismatch: %d != %d" % (self.dim, rhs.dim))
            return self._merge_dot(self.dim, rhs.indices, rhs.data)
        d = np.ascontiguousarray(rhs, dtype=np.float64)  # dot_acc: the sum starts from +0.0
        if d.ndim != 1 or d.size != self.dim:
            raise SprsPanic("Dimension mismatch: %d != %d" % (self.dim, d.size))
        return self._merge_dot(self.dim, np.arange(self.dim, dtype=np.uint64), d)

    def dot_dense(self, rhs):
        """CsVecBase::dot_dense (vec.rs:894-904): `Iterator::sum` of the products, and std's
        f64 sum folds from -0.0 (rust-lang/rust#129321), not from the +0.0 of dot_acc.  So an
        empty vector, or one whose every product is -0.0, gives -0.0; any other result is the
        same as dot_acc's.  (Pinned from the std source: no Rust toolchain runs these tests.)"""
        d = np.ascontiguousarray(rhs, dtype=np.float64)
        if d.ndim != 1 or d.size != self.dim:
            raise SprsPanic("Dimension mismatch: %d != %d" % (self.dim, d.size))
        return self._merge_dot(self.dim, np.arange(self.dim, dtype=np.uint64), d, start=-0.0)

    # `&v * &A` = row_view(v) * A (vec.rs:1084-1102)
    def __mul__(self, rhs):
        if isinstance(rhs, CsMat):
            row = CsMat((1, self.dim), np.array([0, self.nnz()]), self.indices, self.data)
            c = row * rhs
            c = c if c.is_csr() else c.to_other_storage()
            return CsVec(rhs.cols(), c.indices[:c.indptr[1]], c.data[:c.indptr[1]])
        return NotImplemented

    __matmul__ = __mul__


class CsMat:
    """CsMatBase{storage, nrows, ncols, indptr, indices, data} (sparse.rs:94-109) with
    host arrays owned here (as Rust owns its Vecs) and a lazily-built device mirror."""
    __array_ufunc__ = None  # let `ndarray @ CsMat` reach __rmatmul__ (dense.dot(&sparse))

    def __init__(self, shape, indptr, indices, data, storage=CSR, index_dtype=None, ctx=None):
        self.storage = storage
        self.shape = (int(shape[0]), int(shape[1]))
        indptr = np.ascontiguousarray(indptr)
        indices = np.ascontiguousarray(indices)
        if index_dtype is None:  # sprs default is usize (SURVEY F7)
            index_dtype = indices.dtype if indices.dtype.kind in "ui" and indices.dtype.itemsize in (4, 8) \
                else np.uint64
        self.indptr = indptr.astype(index_dtype if indptr.dtype.kind not in "ui" or
                                    indptr.dtype.itemsize not in (4, 8) else indptr.dtype,
                                    copy=False)
        self.indices = indices.astype(index_dtype, copy=False)
        self.data = np.ascontiguousarray(data, dtype=np.float64)
        self._ctx = ctx
        self._dev = None
        self._check_structure()

    # -- constructors (csmat.rs `new`, `new_csc`, `eye`, `zero`)
    @classmethod
    def new(cls, shape, indptr, indices, data, **kw):
        return cls(shape, indptr, indices, data, CSR, **kw)

    @classmethod
    def new_csc(cls, shape, indptr, indices, data, **kw):
        return cls(shape, indptr, indices, data, CSC, **kw)

    @classmethod
    def from_triplets(cls, shape, row_inds, col_inds, data, index_dtype=np.uint64, ctx=None):
        """TriMat::new + to_csr (sprs/src/sparse/triplet.rs, triplet_iter.rs:127-224): COO in
        any order, duplicate entries summed, built by the device radix sort."""
        ctx = ctx or Context.default()
        r = np.ascontiguousarray(row_inds, dtype=np.uint64)
        c = np.ascontiguousarray(col_inds, dtype=np.uint64)
        d = np.ascontiguousarray(data, dtype=np.float64)
        if not (r.shape == c.shape == d.shape):
            raise SprsPanic("row_inds, col_inds and data must have the same length")
        if r.size and (int(r.max()) >= shape[0] or int(c.max()) >= shape[1]):
            raise SprsPanic("Out of bounds index")
        h = C.c_void_p()
        ctx.check(ctx.lib.sprs_b200_csmat_from_triplets(ctx.h, shape[0], shape[1], r.size, _ptr(r),
                                                        _ptr(c), 8, _ptr(d), C.byref(h)))
        dev = DeviceCsMat(ctx, h)
        ip, ind, dat = dev.download(index_dtype)
        m = cls(shape, ip, ind, dat, CSR, ctx=ctx)
        m._dev = dev
        return m

    @classmethod
    def eye(cls, n, **kw):
        return cls((n, n), np.arange(n + 1), np.arange(n), np.ones(n), CSR, **kw)

    @classmethod
    def zero(cls, shape, **kw):
        return cls(shape, np.zeros(shape[0] + 1, dtype=np.int64), [], [], CSR, **kw)

    def _check_structure(self):
        """check_compressed_structure (sparse.rs:300-369), vectorised."""
        outer = self.outer_dims()
        if self.indptr.size != outer + 1:
            raise SprsPanic("Indptr length does not match dimension")
        ip = self.indptr.astype(np.int64)
        if np.any(np.diff(ip) < 0):
            raise SprsPanic("Unsorted indptr")
        nnz = int(ip[-1] - ip[0])
        if self.indices.size < nnz or self.data.size < nnz:
            raise SprsPanic("Indices or data shorter than nnz")
        if nnz:
            ind = self.indices[:nnz].astype(np.int64)
            if ind.max() >= self.inner_dims():
                raise SprsPanic("Out of bounds index")
            d = np.diff(ind)
            starts = (ip[1:-1] - ip[0])
            starts = starts[(starts > 0) & (starts < nnz)]
            ok = d > 0
            ok[starts - 1] = True
            if not ok.all():
                raise SprsPanic("Unsorted indices")

    # -- shape helpers
    def rows(self):
        return self.shape[0]

    def cols(self):
        return self.shape[1]

    def nnz(self):
        return int(self.indptr[-1] - self.indptr[0])

    def is_csr(self):
        return self.storage == CSR

    def is_csc(self):
        return self.storage == CSC

    def outer_dims(self):
        return self.shape[0] if self.storage == CSR else self.shape[1]

    def inner_dims(self):
        return self.shape[1] if self.storage == CSR else self.shape[0]

    def __eq__(self, o):
        return (isinstance(o, CsMat) and self.storage == o.storage and self.shape == o.shape and
                np.array_equal(self.indptr.astype(np.int64) - int(self.indptr[0]),
                               o.indptr.astype(np.int64) - int(o.indptr[0])) and
                np.array_equal(self.indices[:self.nnz()], o.indices[:o.nnz()]) and
                np.array_equal(self.data[:self.nnz()], o.data[:o.nnz()]))

    def __repr__(self):
        return "CsMat(%s, %s, nnz=%d)" % (self.storage, self.shape, self.nnz())

    # -- views (zero-copy, like sprs)
    def transpose_view(self):
        """transpose_view / transpose_into: same arrays, other storage, swapped shape."""
        t = object.__new__(CsMat)
        t.storage = CSC if self.storage == CSR else CSR
        t.shape = (self.shape[1], self.shape[0])
        t.indptr, t.indices, t.data = self.indptr, self.indices, self.data
        t._ctx, t._dev = self._ctx, None
        return t

    transpose_into = transpose_view

    def __iter__(self):
        """`into_iter` of a matrix view (csmat.rs): (value, (row, col)) in storage order."""
        ip = self.indptr.astype(np.int64) - int(self.indptr[0])
        for o in range(self.outer_dims()):
            for k in range(int(ip[o]), int(ip[o + 1])):
                i = int(self.indices[k])
                yield float(self.data[k]), ((o, i) if self.is_csr() else (i, o))

    def slice_outer(self, start=None, stop=None):
        """slice_outer (slicing.rs:65-89): contiguous outer block, NON-zero-based indptr
        kept as is (indptr.rs:122-124); the upload rebases it (proper_indptr).  None = the
        open end of a range (`..5`, `9..`, `..`); a `slice` object is accepted as well."""
        if isinstance(start, slice):
            start, stop = start.start, start.stop
        start = 0 if start is None else int(start)
        stop = self.outer_dims() if stop is None else int(stop)
        if not 0 <= start <= stop <= self.outer_dims():
            raise SprsPanic("Index out of bounds")  # range.rs / indptr.rs slice asserts
        t = object.__new__(CsMat)
        t.storage = self.storage
        n = stop - start
        t.shape = (n, self.shape[1]) if self.storage == CSR else (self.shape[0], n)
        t.indptr = self.indptr[start:stop + 1]
        s = int(self.indptr[start] - self.indptr[0])
        e = int(self.indptr[stop] - self.indptr[0])
        t.indices, t.data = self.indices[s:e], self.data[s:e]
        t._ctx, t._dev = self._ctx, None
        return t

    def to_dense(self):
        """CsMat::to_dense (csmat.rs:1127-1134) on the device: a C-order array holding every
        stored value as its exact bits and +0.0 everywhere else, for CSR and CSC alike."""
        out = np.empty(self.shape)  # the device writes every element
        if out.size:
            ctx = self.context()
            ctx.check(ctx.lib.sprs_b200_csmat_to_dense(ctx.h, self.device().h, _ptr(out),
                                                       self.shape[1]))
        return out

    @classmethod
    def csr_from_dense(cls, m, epsilon, index_dtype=np.uint64, ctx=None):
        """CsMat::csr_from_dense (csmat.rs:502-539) on the device: every x of the 2-D float64
        view m with |x| > epsilon, epsilon clamped to +0.0 when it is not > 0 (so +-0.0 and NaN
        are never kept), stored as the same bits, columns ascending within each row."""
        return _from_dense(cls, m, epsilon, CSR, index_dtype, ctx)

    @classmethod
    def csc_from_dense(cls, m, epsilon, index_dtype=np.uint64, ctx=None):
        """CsMat::csc_from_dense (csmat.rs:544-549): csr_from_dense of the transposed view,
        transposed -- a CSC matrix with rows ascending within each column."""
        return _from_dense(cls, m, epsilon, CSC, index_dtype, ctx)

    # -- device mirror
    def context(self):
        if self._ctx is None:
            self._ctx = Context.default()
        return self._ctx

    def device(self):
        if self._dev is None:
            ctx = self.context()
            h = C.c_void_p()
            nnz = self.nnz()
            ctx.check(ctx.lib.sprs_b200_csmat_upload(
                ctx.h, _STOR[self.storage], self.shape[0], self.shape[1], _ptr(self.indptr),
                self.indptr.dtype.itemsize, _ptr(self.indices[:nnz]),
                self.indices.dtype.itemsize, _ptr(self.data[:nnz]), C.byref(h)))
            self._dev = DeviceCsMat(ctx, h)
        return self._dev

    def to_other_storage(self):
        """to_other_storage (csmat.rs:1405-1426) via the device counting sort."""
        # raw::convert_mat_storage asserts that rows() fits the index type before any work
        # (csmat.rs:1794-1797; sprs/tests/gh374.rs)
        if self.rows() > np.iinfo(self.indices.dtype).max:
            raise SprsPanic("Index type is not large enough to hold the number of rows requested "
                            "(I::max_value=%d vs. required %d)"
                            % (np.iinfo(self.indices.dtype).max, self.rows()))
        d = self.device().to_other_storage()
        ip, ind, dat = d.download(self.indices.dtype, self.indptr.dtype)
        return CsMat(self.shape, ip, ind, dat, CSC if self.storage == CSR else CSR,
                     ctx=self._ctx)

    def to_csr(self):
        return self if self.is_csr() else self.to_other_storage()

    def to_csc(self):
        return self if self.is_csc() else self.to_other_storage()

    # -- operators: `impl Mul` blocks of csmat.rs / vec.rs
    def __mul__(self, rhs):
        if isinstance(rhs, CsMat):
            return csmat_mul_csmat(self, rhs)
        if isinstance(rhs, CsVec):
            return _csmat_mul_csvec(self, rhs)
        if isinstance(rhs, np.ndarray):
            if rhs.ndim == 1:
                return _csmat_mul_dense_vec(self, rhs)
            if rhs.ndim == 2:
                return _csmat_mul_dense_mat(self, rhs)
        if isinstance(rhs, (float, int, np.floating, np.integer)):
            return _csmat_scale(self, float(rhs))
        return NotImplemented

    __matmul__ = __mul__

    def dot(self, rhs):
        return self.__mul__(rhs)

    # -- `impl Add` / `impl Sub` / `impl Mul<N>` of binop.rs:20-163
    def __add__(self, rhs):
        """`&A + &B` (binop.rs:20-65): a new matrix in lhs storage; rhs converted with
        to_other_storage when the storages differ; entries whose sum is 0.0 are dropped."""
        if isinstance(rhs, CsMat):
            return _csmat_binop_other_storage(self, rhs, _lib.BINOP_ADD)
        if isinstance(rhs, np.ndarray) and rhs.ndim == 2:
            return _csmat_add_dense(self, rhs)
        return NotImplemented

    def __sub__(self, rhs):
        """`&A - &B` (binop.rs:67-112), same rules as `+`."""
        if isinstance(rhs, CsMat):
            return _csmat_binop_other_storage(self, rhs, _lib.BINOP_SUB)
        return NotImplemented

    def __rmatmul__(self, lhs):
        """dense.dot(&sparse) = (sparse^T . dense^T)^T  (csmat.rs:2050-2099)."""
        if isinstance(lhs, np.ndarray) and lhs.ndim == 2:
            return (self.transpose_view() * lhs.T).T
        return NotImplemented


# ------------------------------------------------------------------------------------
def _new_trusted_like(lhs, dev):
    """The CsMat of a device result in lhs's storage, shape and index dtypes (new_trusted,
    binop.rs:210-217); the result's mirror stays attached for the next device operation."""
    ip, ind, dat = dev.download(lhs.indices.dtype, lhs.indptr.dtype)
    out = object.__new__(CsMat)
    out.storage, out.shape = lhs.storage, lhs.shape
    out.indptr, out.indices, out.data = ip, ind, dat
    out._ctx, out._dev = lhs._ctx, dev
    return out


def _csmat_binop(lhs, rhs_dev, op):
    """csmat_binop (binop.rs:178-271) on the device: lhs a CsMat, rhs a mirror of the same
    storage.  The reference asserts the shapes first, then the storage."""
    ctx = lhs.context()
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_binop(ctx.h, lhs.device().h, rhs_dev.h, op, C.byref(out)))
    return _new_trusted_like(lhs, DeviceCsMat(ctx, out))


def _csmat_binop_other_storage(lhs, rhs, op):
    """Add / Sub (binop.rs:20-112): shapes checked, then rhs converted to lhs's storage."""
    if lhs.shape != rhs.shape:
        raise SprsPanic("Dimension mismatch")
    rhs_dev = rhs.device() if rhs.storage == lhs.storage else rhs.device().to_other_storage()
    return _csmat_binop(lhs, rhs_dev, op)


# `impl Mul<N> for &CsMatBase` binop.rs:132-163 -> CsMatBase::map (csmat.rs:1289-1305)
def _csmat_scale(a, s):
    ctx = a.context()
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_scale(ctx.h, a.device().h, s, C.byref(out)))
    return _new_trusted_like(a, DeviceCsMat(ctx, out))


class binop:
    """Free functions of sprs/src/sparse/binop.rs."""

    @staticmethod
    def mul_mat_same_storage(lhs, rhs):
        """binop.rs:115-130: element-wise (Hadamard) product of two matrices of the same shape
        AND storage -- no conversion: mixed storage panics "Storage mismatch"."""
        if lhs.shape != rhs.shape:
            raise SprsPanic("Dimension mismatch")
        if lhs.storage != rhs.storage:
            raise SprsPanic("Storage mismatch")
        return _csmat_binop(lhs, rhs.device(), _lib.BINOP_MUL)

    @staticmethod
    def add_dense_mat_same_ordering(lhs, rhs, alpha, beta):
        """binop.rs:279-323: alpha * lhs + beta * rhs, lhs sparse, rhs a 2-D float64 view, as
        (alpha*x) + (beta*y) with x = +0.0 where lhs has no entry.  The result is C order when
        rhs's fastest axis is Axis(1), F order otherwise; a CSR lhs needs a C-like rhs and a CSC
        one an F-like rhs ("Storage mismatch"), after the shapes ("Dimension mismatch")."""
        out = np.zeros(rhs.shape, order="C" if fastest_axis(rhs) == 1 else "F")
        _binop_dense(lhs.device(), _lib.BINOP_ADD, alpha, beta, rhs, out)
        return out

    @staticmethod
    def mul_dense_mat_same_ordering(lhs, rhs, alpha):
        """binop.rs:331-371: (alpha*x)*y element-wise, x = +0.0 where lhs has no entry, so a
        missing position gives -0.0 for a negative y and NaN for an infinite or NaN y.  Layout
        and panics as add_dense_mat_same_ordering."""
        out = np.zeros(rhs.shape, order="C" if fastest_axis(rhs) == 1 else "F")
        _binop_dense(lhs.device(), _lib.BINOP_MUL, alpha, 0.0, rhs, out)
        return out

    @staticmethod
    def csmat_binop_dense_raw_add(lhs, rhs, alpha, beta, out):
        """csmat_binop_dense_raw (binop.rs:384-433) with the add closure, into the given writeable
        out view (which may be rhs itself)."""
        _binop_dense(lhs.device(), _lib.BINOP_ADD, alpha, beta, rhs, out)

    @staticmethod
    def csmat_binop_dense_raw_mul(lhs, rhs, alpha, out):
        """csmat_binop_dense_raw with the mul closure, into out."""
        _binop_dense(lhs.device(), _lib.BINOP_MUL, alpha, 0.0, rhs, out)


# ---- the dense boundary: to_dense.rs, csmat.rs:502-549, binop.rs:273-433
def dense_strides(a, writeable=False):
    """The element strides (rs, cs) a float64 2-D view is passed to the library with.  ndarray
    gives an array with a zero-length axis all-zero strides (its default C and F strides and
    its slicing both do), where numpy keeps non-zero ones: such a view is passed as (0, 0), so
    that fastest_axis sees what the reference sees (DESIGN.md 4.11)."""
    if not isinstance(a, np.ndarray) or a.ndim != 2:
        raise TypeError("a 2-D numpy array is required (ArrayView2)")
    if a.dtype != np.float64:
        raise TypeError("f64 only on the H100 path (other N stay on the CPU code)")
    if writeable and not a.flags.writeable:
        raise ValueError("the dense array must be writeable (ArrayViewMut)")
    if 0 in a.shape:
        return 0, 0
    if a.strides[0] % 8 or a.strides[1] % 8:
        raise TypeError("strides must be whole float64 elements")
    return a.strides[0] // 8, a.strides[1] // 8


def fastest_axis(a):
    """utils::fastest_axis (sparse.rs:400-406): Axis(0) iff strides[1] > strides[0] (signed);
    equal strides -- length-1 axes, broadcasts, empty arrays -- give Axis(1)."""
    rs, cs = dense_strides(a)
    return 0 if cs > rs else 1


def assign_to_dense(array, spmat):
    """to_dense.rs:12-30: array[r, c] = v for every stored (v, (r, c)) of spmat, copied as bits;
    every other element of the writeable view is left as it is.  Asserts cols, then rows."""
    rs, cs = dense_strides(array, writeable=True)
    if spmat.cols() != array.shape[1] or spmat.rows() != array.shape[0]:
        raise SprsPanic("Dimension mismatch")
    ctx = spmat.context()
    ctx.check(ctx.lib.sprs_b200_assign_to_dense(ctx.h, spmat.device().h, _ptr(array),
                                                array.shape[0], array.shape[1], rs, cs))


def _binop_dense(lhs_dev, op, alpha, beta, rhs, out):
    """csmat_binop_dense_raw on the device: shapes, then storage, checked by the library in the
    reference's order."""
    rrs, rcs = dense_strides(rhs)
    ors, ocs = dense_strides(out, writeable=True)
    ctx = lhs_dev.ctx
    ctx.check(ctx.lib.sprs_b200_csmat_binop_dense(
        ctx.h, lhs_dev.h, op, float(alpha), float(beta), _ptr(rhs), rhs.shape[0], rhs.shape[1],
        rrs, rcs, _ptr(out), out.shape[0], out.shape[1], ors, ocs))


def _csmat_add_dense(a, d):
    """`&A + &D` (csmat.rs:1951-1987): alpha = beta = 1; A converted with to_other_storage first
    when its storage does not match D's fastest axis; the result has D's layout."""
    c_like = fastest_axis(d) == 1
    lhs = a.device() if a.is_csr() == c_like else a.device().to_other_storage()
    out = np.zeros(d.shape, order="C" if c_like else "F")
    _binop_dense(lhs, _lib.BINOP_ADD, 1.0, 1.0, d, out)
    return out


def _from_dense(cls, m, epsilon, storage, index_dtype, ctx):
    rs, cs = dense_strides(m)
    ctx = ctx or Context.default()
    h = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_from_dense(ctx.h, _STOR[storage], m.shape[0], m.shape[1],
                                                 _ptr(m), rs, cs, float(epsilon), C.byref(h)))
    dev = DeviceCsMat(ctx, h)
    ip, ind, dat = dev.download(np.uint64)
    # Iptr::from_usize / I::from_usize (indexing.rs:104-107): the indptr is built first
    mx = np.iinfo(index_dtype).max
    for a in (ip, ind):
        big = np.nonzero(a > mx)[0]
        if big.size:
            raise SprsPanic("Failed to convert %d to index type" % int(a[big[0]]))
    out = object.__new__(cls)
    out.storage, out.shape = storage, (int(m.shape[0]), int(m.shape[1]))
    out.indptr, out.indices, out.data = ip.astype(index_dtype), ind.astype(index_dtype), dat
    out._ctx, out._dev = ctx, dev
    return out


# `impl Mul<&ArrayBase<_, Ix1>> for &CsMatBase`  csmat.rs:2119-2160
def _csmat_mul_dense_vec(a, x):
    if a.cols() != x.shape[0]:
        raise SprsPanic("Dimension mismatch")
    ctx = a.context()
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty(a.rows(), dtype=np.float64)  # Array::zeros(rows) in the reference
    ctx.check(ctx.lib.sprs_b200_mul_mat_vec(ctx.h, a.device().h, _ptr(x), x.size, _ptr(y),
                                            y.size))
    return y


# `impl Mul<&ArrayBase<_, Ix2>> for &CsMatBase`  csmat.rs:1989-2048
def _csmat_mul_dense_mat(a, b):
    rows, cols = a.rows(), b.shape[1]
    if cols >= 8:  # csmat.rs:2009: wide rhs -> rowmaj kernel, C-order result
        res = np.zeros((rows, cols))
        f = prod.csr_mulacc_dense_rowmaj if a.is_csr() else prod.csc_mulacc_dense_rowmaj
    else:          # narrow rhs -> colmaj kernel, F-order result
        res = np.zeros((rows, cols), order="F")
        f = prod.csr_mulacc_dense_colmaj if a.is_csr() else prod.csc_mulacc_dense_colmaj
    f(a, b, res)
    return res


# `impl Mul<&CsVecBase> for &CsMatBase`  vec.rs:1104-1131 -> prod::csr_mul_csvec
def _csmat_mul_csvec(a, v):
    if a.is_csr():
        return prod.csr_mul_csvec(a, v)
    col = CsMat((v.dim, 1), np.array([0, v.nnz()]), v.indices, v.data, CSC)  # col_view
    c = (a * col)
    c = c if c.is_csc() else c.to_other_storage()
    return CsVec(a.rows(), c.indices[:c.indptr[1]], c.data[:c.indptr[1]])


# csmat_mul_csmat  csmat.rs:1895-1949
def csmat_mul_csmat(lhs, rhs):
    ls, rs = lhs.storage, rhs.storage
    if (ls, rs) == (CSR, CSR):
        return smmp.mul_csr_csr(lhs, rhs)
    if (ls, rs) == (CSR, CSC):
        return smmp.mul_csr_csr(lhs, rhs.to_other_storage())
    if (ls, rs) == (CSC, CSR):
        rhs_csc = rhs.to_other_storage()
        return smmp.mul_csr_csr(rhs_csc.transpose_view(), lhs.transpose_view()).transpose_into()
    return smmp.mul_csr_csr(rhs.transpose_view(), lhs.transpose_view()).transpose_into()


class prod:
    """Free functions of sprs/src/sparse/prod.rs (same argument order)."""

    @staticmethod
    def _vec(name, mat, in_vec, res_vec):
        if not (isinstance(res_vec, np.ndarray) and res_vec.dtype == np.float64 and
                res_vec.flags.c_contiguous):
            raise TypeError("res_vec must be a contiguous float64 array (DenseVectorMut)")
        x = np.ascontiguousarray(in_vec, dtype=np.float64)
        ctx = mat.context()
        # the reference asserts dimensions, then storage (prod.rs:114-118)
        if mat.cols() != x.size or mat.rows() != res_vec.size:
            raise SprsPanic("Dimension mismatch")
        want = CSR if name.endswith("csr") else CSC
        if mat.storage != want:
            raise SprsPanic("Storage mismatch")
        f = getattr(ctx.lib, "sprs_b200_" + name)
        ctx.check(f(ctx.h, mat.device().h, _ptr(x), x.size, _ptr(res_vec), res_vec.size))

    @staticmethod
    def mul_acc_mat_vec_csr(mat, in_vec, res_vec):
        """prod.rs:103-127: res_vec += mat * in_vec."""
        prod._vec("mul_acc_mat_vec_csr", mat, in_vec, res_vec)

    @staticmethod
    def mul_acc_mat_vec_csc(mat, in_vec, res_vec):
        """prod.rs:74-99."""
        prod._vec("mul_acc_mat_vec_csc", mat, in_vec, res_vec)

    @staticmethod
    def _dense(name, lhs, rhs, out):
        if rhs.dtype != np.float64 or out.dtype != np.float64:
            raise TypeError("f64 only on the H100 path (other N stay on the CPU code)")
        # assert order of prod.rs:198-201
        if lhs.cols() != rhs.shape[0] or lhs.rows() != out.shape[0] or \
                rhs.shape[1] != out.shape[1]:
            raise SprsPanic("Dimension mismatch")
        if lhs.storage != (CSR if name.startswith("csr") else CSC):
            raise SprsPanic("Storage mismatch")
        ctx = lhs.context()
        f = getattr(ctx.lib, "sprs_b200_" + name)
        ctx.check(f(ctx.h, lhs.device().h, _ptr(rhs), rhs.shape[0], rhs.shape[1],
                    rhs.strides[0] // 8, rhs.strides[1] // 8, _ptr(out), out.shape[0],
                    out.shape[1], out.strides[0] // 8, out.strides[1] // 8))

    @staticmethod
    def csr_mulacc_dense_rowmaj(lhs, rhs, out):
        """prod.rs:189-214: out += lhs * rhs (any-stride views)."""
        prod._dense("csr_mulacc_dense_rowmaj", lhs, rhs, out)

    @staticmethod
    def csr_mulacc_dense_colmaj(lhs, rhs, out):
        """prod.rs:274-298."""
        prod._dense("csr_mulacc_dense_colmaj", lhs, rhs, out)

    @staticmethod
    def csc_mulacc_dense_rowmaj(lhs, rhs, out):
        """prod.rs:219-241."""
        prod._dense("csc_mulacc_dense_rowmaj", lhs, rhs, out)

    @staticmethod
    def csc_mulacc_dense_colmaj(lhs, rhs, out):
        """prod.rs:246-269."""
        prod._dense("csc_mulacc_dense_colmaj", lhs, rhs, out)

    @staticmethod
    def csvec_dot_by_binary_search(vec1, vec2):
        """prod.rs:13-72: dot product of two sparse vectors -- the matching entries multiplied
        and summed in ascending index order.  On the device this is row_view(vec1) times vec2
        through the merge-dot kernel (csrc/csvec.cu): same terms, same order, same bits."""
        # the reference does not compare the dimensions here
        return vec1._merge_dot(max(vec1.dim, vec2.dim), vec2.indices, vec2.data)

    @staticmethod
    def csr_mul_csvec(lhs, rhs):
        """prod.rs:162-184: row i of the result is the sorted-merge dot of row i with rhs
        (vec.rs:846-881) -- only entries present in both patterns are multiplied, summed in
        ascending column order (csrc/csvec.cu, bit-identical) -- and exact zeros are
        dropped (prod.rs:178-180)."""
        if rhs.dim == 0:
            return CsVec.empty(0)
        if lhs.cols() != rhs.dim:
            raise SprsPanic("Dimension mismatch")
        if not lhs.is_csr():
            raise SprsPanic("Storage mismatch")
        ctx = lhs.context()
        vi = np.ascontiguousarray(rhs.indices, dtype=np.uint64)
        vd = np.ascontiguousarray(rhs.data, dtype=np.float64)
        y = np.empty(lhs.rows())
        ctx.check(ctx.lib.sprs_b200_csr_mul_csvec(ctx.h, lhs.device().h, rhs.dim, vi.size,
                                                  _ptr(vi), 8, _ptr(vd), _ptr(y), y.size))
        nz = np.nonzero(y != 0.0)[0]  # `val != N::zero()`: NaN is kept, -0.0 is dropped
        return CsVec(lhs.rows(), nz, y[nz])


class smmp:
    """sprs/src/sparse/smmp.rs: two-phase SpGEMM (symbolic pattern, numeric values)."""

    @staticmethod
    def mul_csr_csr(lhs, rhs):
        """smmp.rs:196-237.  Output arrays are allocated HERE (the caller), like the
        Vecs the reference allocates between symbolic and numeric."""
        if lhs.cols() != rhs.rows():
            raise SprsPanic("Dimension mismatch")  # assert_eq!(lhs.cols(), rhs.rows())
        if not (lhs.is_csr() and rhs.is_csr()):
            raise SprsPanic("Storage mismatch")
        ctx = lhs.context()
        plan, nnz_c = C.c_void_p(), C.c_uint64()
        ctx.check(ctx.lib.sprs_b200_spgemm_symbolic(ctx.h, lhs.device().h, rhs.device().h,
                                                    C.byref(plan), C.byref(nnz_c)))
        try:
            ip = np.empty(lhs.rows() + 1, dtype=lhs.indptr.dtype)
            ind = np.empty(nnz_c.value, dtype=lhs.indices.dtype)
            dat = np.empty(nnz_c.value, dtype=np.float64)
            ctx.check(ctx.lib.sprs_b200_spgemm_numeric(
                ctx.h, plan, _ptr(ip), ip.dtype.itemsize, _ptr(ind), ind.dtype.itemsize,
                _ptr(dat)))
        finally:
            ctx.lib.sprs_b200_spgemm_free(plan)
        out = object.__new__(CsMat)  # new_trusted (smmp.rs:409-415)
        out.storage, out.shape = CSR, (lhs.rows(), rhs.cols())
        out.indptr, out.indices, out.data = ip, ind, dat
        out._ctx, out._dev = lhs._ctx, None
        return out
