"""Sparse LDL^T factorization on the device: the mirror of the sprs-ldl crate
(sprs-ldl/src/lib.rs).

`LdlSymbolic`, `LdlNumeric` (`new`, `new_perm`, `update`, `solve`, `l`, `d`, `nnz`,
`problem_size`), the `Ldl` builder, `ldl_lsolve` and `ldl_ltsolve` compute what the reference
computes, bit for bit: L D L^T = P A P^T with the permutation the caller gives, or none
(csrc/ldl.cu).  The symbolic analysis runs on the host; the numeric factorization, `update` and
`solve` run on the GPU.  `LdlNumeric.solve_dev` solves a device-resident right-hand side.

Differences a caller can see:
  * the builder computes no fill-reducing ordering: asking for
    FillInReduction.ReverseCuthillMcKee (the builder's default, as in the reference) or
    CAMDSuiteSparse raises NotImplementedError when the factorization is built.  Use
    FillInReduction.NoReduction, or compute a permutation and call `LdlNumeric.new_perm`;
  * after an `update` that raises SingularMatrix, `l()`, `d()`, `solve` and `solve_dev` raise
    it too until an `update` succeeds.  The reference keeps the partial factor readable;
  * an `update` with a matrix whose pattern is not the symbolic one raises SprsPanic before
    any work is done, and the factor stays as it was.  The reference leaves that unspecified.
"""
import ctypes as C
import enum

import numpy as np

from . import _lib
from .sparse import CSC, CsMat, DeviceCsMat, SingularMatrix, SprsPanic

_NUMERIC_ZERO = "diagonal element is a numeric 0"


class SymmetryCheck(enum.Enum):
    """sprs::SymmetryCheck."""
    CheckSymmetry = 0
    DontCheckSymmetry = 1


class PermutationCheck(enum.Enum):
    """sprs::PermutationCheck."""
    CheckPerm = 0
    NoCheckPerm = 1


class FillInReduction(enum.Enum):
    """sprs::FillInReduction."""
    NoReduction = 0
    ReverseCuthillMcKee = 1
    CAMDSuiteSparse = 2


def _device(mat):
    if isinstance(mat, CsMat):
        return mat.device(), mat.shape
    if isinstance(mat, DeviceCsMat):
        return mat, (mat.rows, mat.cols)
    raise TypeError("mat must be a CsMat or a DeviceCsMat")


def is_symmetric(mat):
    """sprs::is_symmetric (sparse/symmetric.rs), on the device: square, and every entry has a
    transposed partner with an equal value (NaN is not equal to itself)."""
    dev, _ = _device(mat)
    out = C.c_int()
    dev.ctx.check(dev.ctx.lib.sprs_b200_is_symmetric(dev.ctx.h, dev.h, C.byref(out)))
    return bool(out.value)


class Ldl:
    """Builder of a factorization (sprs-ldl `Ldl`), with the reference's defaults:
    CheckSymmetry, ReverseCuthillMcKee, CheckPerm."""

    def __init__(self, check_symmetry=SymmetryCheck.CheckSymmetry,
                 fill_red_method=FillInReduction.ReverseCuthillMcKee,
                 check_perm=PermutationCheck.CheckPerm):
        self._check_symmetry = check_symmetry
        self._fill_red_method = fill_red_method
        self._check_perm = check_perm

    @classmethod
    def new(cls):
        return cls()

    def check_symmetry(self, check):
        return Ldl(check, self._fill_red_method, self._check_perm)

    def check_perm(self, check):
        return Ldl(self._check_symmetry, self._fill_red_method, check)

    def fill_in_reduction(self, method):
        return Ldl(self._check_symmetry, method, self._check_perm)

    def perm(self, mat):
        """The permutation the builder factors in: the identity for NoReduction."""
        if self._fill_red_method == FillInReduction.NoReduction:
            return np.arange(_device(mat)[1][0], dtype=np.uint32)
        raise NotImplementedError(
            "%s is not available on the device: use FillInReduction.NoReduction, or compute a "
            "permutation and call LdlNumeric.new_perm" % self._fill_red_method.name)

    def symbolic(self, mat):
        return LdlSymbolic.new_perm(mat, self.perm(mat), self._check_symmetry)

    def numeric(self, mat):
        return self.symbolic(mat).factor(mat)


class LdlSymbolic:
    """The elimination tree and the structure of L for one pattern and permutation
    (sprs-ldl `LdlSymbolic`)."""

    def __init__(self, mat, perm, check_symmetry):
        dev, (rows, cols) = _device(mat)
        if rows != cols:
            raise SprsPanic("matrix should be square")
        ctx = dev.ctx
        p = None
        if perm is not None:
            p = np.ascontiguousarray(perm, dtype=np.int64)
            if p.ndim != 1 or p.size != rows:
                # checked after the symmetry, as the C entry point checks the values
                if check_symmetry == SymmetryCheck.CheckSymmetry and not is_symmetric(dev):
                    raise SprsPanic("Matrix is not symmetric")
                raise SprsPanic("assertion failed: perm_is_valid(&perm) (length %d for %d rows)"
                                % (p.size, rows))
            if p.size and (p.min() < 0 or p.max() >= rows):
                p = np.full(rows, rows, dtype=np.int64)  # refused by the library, in its order
            p = p.astype(np.uint32)
        h = C.c_void_p()
        st = ctx.lib.sprs_b200_ldl_symbolic(
            ctx.h, dev.h, p.ctypes.data_as(C.c_void_p) if p is not None and p.size else None,
            int(check_symmetry == SymmetryCheck.CheckSymmetry), C.byref(h))
        if st == _lib.ERR_ARGUMENT:
            raise SprsPanic("assertion failed: perm_is_valid(&perm)")
        if st == _lib.ERR_DIMENSION:
            raise SprsPanic("matrix should be square")
        ctx.check(st)
        self._ctx, self._h, self._n = ctx, h, rows
        self._index_dtype = mat.indices.dtype if isinstance(mat, CsMat) else np.uint32

    @classmethod
    def new(cls, mat):
        """LdlSymbolic::new: the identity permutation, symmetry checked."""
        _, (rows, cols) = _device(mat)
        if rows != cols:
            raise SprsPanic("assertion `left == right` failed\n  left: %d\n right: %d"
                            % (rows, cols))
        return cls(mat, None, SymmetryCheck.CheckSymmetry)

    @classmethod
    def new_perm(cls, mat, perm, check_symmetry=SymmetryCheck.CheckSymmetry):
        """LdlSymbolic::new_perm: perm[k] is the outer vector of mat that is row k of P A P^T."""
        return cls(mat, perm, check_symmetry)

    def problem_size(self):
        return self._n

    def nnz(self):
        """The number of non-zeros of L."""
        return int(self._ctx.lib.sprs_b200_ldl_nnz(self._h))

    def factor(self, mat):
        """LdlSymbolic::factor: the numeric factorization of mat (same pattern).  Raises
        SingularMatrix as the reference returns Err(SingularMatrix)."""
        return LdlNumeric._factor(self, mat)

    def free(self):
        if getattr(self, "_h", None):
            self._ctx.lib.sprs_b200_ldl_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class LdlNumeric:
    """A numeric factorization L D L^T = P A P^T (sprs-ldl `LdlNumeric`)."""

    @classmethod
    def _factor(cls, sym, mat):
        if sym._n <= 1:  # DStack::with_capacity(n) in LdlSymbolic::factor
            raise SprsPanic("assertion failed: n > 1")
        dev, _ = _device(mat)
        self = cls.__new__(cls)
        self._sym, self._ctx, self._n = sym, sym._ctx, sym._n
        h = C.c_void_p()
        st = self._ctx.lib.sprs_b200_ldl_factor(sym._h, dev.h, C.byref(h))
        self._h = h if h.value else None
        if st == _lib.ERR_STRUCTURE:
            raise SprsPanic(self._ctx.lib.sprs_b200_last_error(self._ctx.h).decode())
        self._ctx.check(st)
        return self

    @classmethod
    def new(cls, mat):
        """LdlNumeric::new: the identity permutation, symmetry checked."""
        return LdlSymbolic.new(mat).factor(mat)

    @classmethod
    def new_perm(cls, mat, perm, check_symmetry=SymmetryCheck.CheckSymmetry):
        """LdlNumeric::new_perm."""
        return LdlSymbolic.new_perm(mat, perm, check_symmetry).factor(mat)

    def update(self, mat):
        """LdlNumeric::update with a matrix of the same pattern and new values.  Raises
        SingularMatrix, or SprsPanic when the pattern is not the symbolic one (nothing is
        computed then, and the factor stays as it was)."""
        dev, _ = _device(mat)
        st = self._ctx.lib.sprs_b200_ldl_update(self._h, dev.h)
        if st == _lib.ERR_STRUCTURE:
            raise SprsPanic(self._ctx.lib.sprs_b200_last_error(self._ctx.h).decode())
        if st == _lib.ERR_DIMENSION:
            raise SprsPanic("Dimension mismatch")
        self._ctx.check(st)

    def singular(self):
        """The SingularMatrix of the last factor / update, or None."""
        idx = C.c_uint64()
        if not self._ctx.lib.sprs_b200_ldl_singular(self._h, C.byref(idx)):
            return None
        return SingularMatrix(int(idx.value), _NUMERIC_ZERO)

    def solve(self, rhs):
        """x with A x = rhs (a new array), as LdlNumeric::solve."""
        b = np.ascontiguousarray(rhs, dtype=np.float64)
        if b.ndim != 1 or b.size != self._n:
            raise SprsPanic("assertion `left == right` failed\n  left: %d\n right: %d"
                            % (self._n, b.size))
        x = np.empty(self._n, dtype=np.float64)
        self._ctx.check(self._ctx.lib.sprs_b200_ldl_solve(
            self._h, b.ctypes.data_as(C.c_void_p), x.ctypes.data_as(C.c_void_p), b.size))
        return x

    def solve_dev(self, d_b, d_x, stream=None):
        """Enqueue the solve of n doubles at device address d_b into d_x (may be the same) on
        `stream` (a cudaStream_t as an int; None = the legacy default stream).  Asynchronous;
        one stream at a time."""
        self._ctx.check(self._ctx.lib.sprs_b200_ldl_solve_dev(
            self._h, C.c_void_p(int(d_b)), C.c_void_p(int(d_x)),
            C.c_void_p(int(stream) if stream else 0)))

    def l(self):  # noqa: E743  (the reference's name)
        """L as a CSC CsMat (unit diagonal not stored), as LdlNumeric::l."""
        n, nnz = self._n, self.nnz()
        ip = np.empty(n + 1, dtype=np.uint32)
        ind = np.empty(nnz, dtype=np.uint32)
        dat = np.empty(nnz, dtype=np.float64)
        self._ctx.check(self._ctx.lib.sprs_b200_ldl_get_l(
            self._h, ip.ctypes.data_as(C.c_void_p), ind.ctypes.data_as(C.c_void_p) if nnz else None,
            dat.ctypes.data_as(C.c_void_p) if nnz else None))
        dt = self._sym._index_dtype
        return CsMat((n, n), ip.astype(dt), ind.astype(dt), dat, CSC, ctx=self._ctx)

    def d(self):
        """The diagonal D, as LdlNumeric::d."""
        d = np.empty(self._n, dtype=np.float64)
        self._ctx.check(self._ctx.lib.sprs_b200_ldl_get_d(self._h, d.ctypes.data_as(C.c_void_p),
                                                          self._n))
        return d

    def problem_size(self):
        return self._n

    def nnz(self):
        return self._sym.nnz()

    def free(self):
        if getattr(self, "_h", None):
            self._ctx.lib.sprs_b200_ldl_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _unit(l, transpose):
    """L + I (transpose=False: CSC, for lsolve_csc) or L^T + I (True: L's CSC arrays read as
    CSR, for usolve_csr), L strictly lower as the factorization makes it.  Dividing by the unit
    diagonal is exact, so these solves compute the reference's unit-diagonal sweeps bit for
    bit."""
    if not isinstance(l, CsMat) or not l.is_csc():
        raise TypeError("l must be a CSC CsMat")
    n = l.cols()
    ip = l.indptr.astype(np.int64) - int(l.indptr[0])
    ind = l.indices[:l.nnz()].astype(np.int64)
    # column i: its diagonal first (its row indices are all > i), then its entries
    new_ip = ip + np.arange(n + 1)
    pos = np.arange(ind.size) + np.repeat(np.arange(n), np.diff(ip)) + 1
    out_ind = np.empty(ind.size + n, dtype=np.int64)
    out_dat = np.empty(ind.size + n, dtype=np.float64)
    out_ind[new_ip[:-1]] = np.arange(n)
    out_dat[new_ip[:-1]] = 1.0
    out_ind[pos] = ind
    out_dat[pos] = l.data[:l.nnz()]
    cls = CsMat.new if transpose else CsMat.new_csc
    return cls((n, n), new_ip, out_ind.astype(np.uint32), out_dat, ctx=l._ctx)


def ldl_lsolve(l, x):
    """sprs-ldl ldl_lsolve: x (a contiguous float64 array) solved in place with the unit lower
    triangular L (CSC, strictly lower), column by column: x_j -= L_ji x_i."""
    from .linalg import trisolve
    trisolve.lsolve_csc_dense_rhs(_unit(l, False), x)


def ldl_ltsolve(l, x):
    """sprs-ldl ldl_ltsolve: x solved in place with L^T, columns in descending order, each
    x_i -= L_ji x_j over column i in stored order."""
    from .linalg import trisolve
    trisolve.usolve_csr_dense_rhs(_unit(l, True), x)


__all__ = ["Ldl", "LdlSymbolic", "LdlNumeric", "SymmetryCheck", "PermutationCheck",
           "FillInReduction", "ldl_lsolve", "ldl_ltsolve", "is_symmetric"]
