"""Iterative solvers on the device SpMV (SURVEY.md 8f rank 3).

`bicgstab.BiCGSTAB` mirrors sprs::linalg::bicgstab::BiCGSTAB<f64>
(sprs/src/sparse/linalg/bicgstab.rs:95-300): same constructor, `solve`, `step`,
`soft_restart`, `hard_restart` and accessors.  All vectors stay in HBM between iterations
(csrc/solver.cu); this module only holds the handle.

`trisolve` mirrors sprs::linalg::trisolve (sprs/src/sparse/linalg/trisolve.rs): the four
dense-rhs solves, bit-identical to the reference (csrc/trisolve.cu), and `TriSolvePlan` for
repeated solves of one matrix and the device-resident form.

`diag_solve` mirrors sprs::linalg::diag_solve.  The LDL^T factorization is in `sprs_b200.ldl`.

Differences a caller can see in BiCGSTAB, both forced by the host language:
  * vectors are dense float64 arrays (a CsVec argument is densified; the reference's CsVec
    arithmetic is dense arithmetic on the union pattern, binop.rs:442-470), accessors return
    numpy arrays;
  * `solve` returns the solver for Ok and raises `NotConverged(solver)` for Err -- the
    reference returns `Result<Box<Self>, Box<Self>>` and its tests `.unwrap()` it.
"""
import ctypes as C

import numpy as np

from . import _lib
from .sparse import CsMat, CsVec, DeviceCsMat, SingularMatrix, SprsPanic

_X, _R, _RHAT, _P, _B = range(5)


class NotConverged(Exception):
    """`Err(solver)` of BiCGSTAB::solve (bicgstab.rs:173-174): the iteration limit was
    reached; `.solver` holds the state reached so far."""

    def __init__(self, solver):
        super().__init__("BiCGSTAB did not reach the tolerance in %d iterations (err = %g)" %
                         (solver.iteration_count(), solver.err()))
        self.solver = solver


def _dense(v, n):
    if isinstance(v, CsVec):
        if v.dim != n:
            raise SprsPanic("Dimension mismatch")
        return v.to_dense()
    a = np.ascontiguousarray(v, dtype=np.float64)
    if a.shape != (n,):
        raise SprsPanic("Dimension mismatch")
    return a


class BiCGSTAB:
    """Stabilized bi-conjugate gradient solver for A x = b (bicgstab.rs:95-116)."""

    def __init__(self, a, x0, b):
        """BiCGSTAB::new (bicgstab.rs:120-146): r = b - A x0, rhat = p = r."""
        if isinstance(a, CsMat):
            rows, cols = a.shape
        elif isinstance(a, DeviceCsMat):
            rows, cols = a.rows, a.cols
        else:
            raise TypeError("a must be a CsMat or a DeviceCsMat")
        # the reference panics in `&a * &x0` / `&b - ..` before anything is computed
        x0 = _dense(x0, cols)
        b = _dense(b, rows)
        if rows != cols:  # `&a * &p` with p = r
            raise SprsPanic("Dimension mismatch")
        dev = a.device() if isinstance(a, CsMat) else a
        self._a, self._dev, self._ctx = a, dev, dev.ctx
        n = rows
        h = C.c_void_p()
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_new(
            self._ctx.h, dev.h, x0.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
            n, C.byref(h)))
        self._h, self._n = h, n

    @classmethod
    def new(cls, a, x0, b):
        return cls(a, x0, b)

    @classmethod
    def with_operator(cls, ctx, n, matvec, x0, b):
        """The same solver with y = A x delegated to `matvec(d_x, d_y, stream)` (raw device
        addresses of n doubles each and the cudaStream_t to enqueue on, as ints): a
        matrix-free operator, or the row-partitioned SpMV + all-gather of sprs_b200.dist
        (every rank keeps full-length vectors and takes identical steps, see
        dist.row_partitioned_bicgstab).  sprs_b200_bicgstab_new_op."""
        from . import _lib
        x0 = _dense(x0, n)
        b = _dense(b, n)
        self = cls.__new__(cls)

        def thunk(_user, d_x, d_y, stream):
            try:
                matvec(int(d_x or 0), int(d_y or 0), int(stream or 0))
                return 0
            except Exception as e:  # an exception must not unwind through the C frames
                self._op_error = e
                return 1

        self._op_error = None
        self._thunk = _lib.MATVEC_FN(thunk)  # kept alive with the solver
        self._a, self._dev, self._ctx, self._n = None, None, ctx, n
        h = C.c_void_p()
        st = ctx.lib.sprs_b200_bicgstab_new_op(ctx.h, n, self._thunk, None,
                                               x0.ctypes.data_as(C.c_void_p),
                                               b.ctypes.data_as(C.c_void_p), 0, C.byref(h))
        if st and self._op_error is not None:
            raise self._op_error
        ctx.check(st)
        self._h = h
        return self

    def _check(self, st):
        if st and getattr(self, "_op_error", None) is not None:
            e, self._op_error = self._op_error, None
            raise e
        self._ctx.check(st)

    @classmethod
    def solve(cls, a, x0, b, tol, max_iter):
        """BiCGSTAB::solve (bicgstab.rs:151-175).  Ok -> the solver; Err -> NotConverged."""
        return cls(a, x0, b).run(tol, max_iter)

    def run(self, tol, max_iter):
        """The loop of `solve` on an existing solver (bicgstab.rs:156-175)."""
        conv = C.c_int(0)
        self._check(self._ctx.lib.sprs_b200_bicgstab_solve(self._h, float(tol), int(max_iter),
                                                           C.byref(conv)))
        if not conv.value:
            raise NotConverged(self)
        return self

    def step(self):
        """One iteration (bicgstab.rs:198-234); returns the running error estimate."""
        err = C.c_double()
        self._check(self._ctx.lib.sprs_b200_bicgstab_step(self._h, C.byref(err)))
        return err.value

    def soft_restart(self):
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_soft_restart(self._h))

    def hard_restart(self):
        self._check(self._ctx.lib.sprs_b200_bicgstab_hard_restart(self._h))

    def with_restart_threshold(self, thresh):
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_set_restart_threshold(self._h,
                                                                               float(thresh)))
        return self

    # -- accessors (bicgstab.rs:236-298)
    def _stats(self):
        counts = (C.c_uint64 * 3)()
        scal = (C.c_double * 3)()
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_stats(self._h, counts, scal))
        return list(counts), list(scal)

    def iteration_count(self):
        return int(self._stats()[0][0])

    def soft_restart_count(self):
        return int(self._stats()[0][1])

    def hard_restart_count(self):
        return int(self._stats()[0][2])

    def err(self):
        return self._stats()[1][0]

    def rho(self):
        return self._stats()[1][1]

    def soft_restart_threshold(self):
        return self._stats()[1][2]

    def a(self):
        return self._a

    def _vec(self, which):
        out = np.empty(self._n, dtype=np.float64)
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_get(
            self._h, which, out.ctypes.data_as(C.c_void_p), self._n))
        return out

    def x(self):
        return self._vec(_X)

    def b(self):
        return self._vec(_B)

    def r(self):
        return self._vec(_R)

    def rhat(self):
        return self._vec(_RHAT)

    def p(self):
        return self._vec(_P)

    def device_vector(self, name):
        """Raw device address of x / r / rhat / p / b (borrowed; valid until the solver is
        dropped) for callers that keep working on the GPU."""
        which = {"x": _X, "r": _R, "rhat": _RHAT, "p": _P, "b": _B}[name]
        ptr = C.c_void_p()
        self._ctx.check(self._ctx.lib.sprs_b200_bicgstab_get_dev(self._h, which, C.byref(ptr)))
        return ptr.value

    def free(self):
        if getattr(self, "_h", None):
            self._ctx.lib.sprs_b200_bicgstab_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class bicgstab:  # noqa: N801  (module path of the reference: sprs::linalg::bicgstab)
    BiCGSTAB = BiCGSTAB
    NotConverged = NotConverged


_REASONS = {_lib.SINGULAR_IS_ZERO: "diagonal element is 0",
            _lib.SINGULAR_NUMERIC: "diagonal element is a numeric 0",
            _lib.SINGULAR_STRUCTURAL: "diagonal element is a structural 0"}


class TriSolvePlan:
    """The analysis of one matrix and triangle for repeated solves (sprs_b200_trisolve_plan):
    the diagonal of every row and the first singular index in processing order.  `mat` is a
    CsMat or DeviceCsMat, square; lower=True solves L x = b, False U x = b, in the matrix's
    storage (CSR: lsolve_csr / usolve_csr, CSC: lsolve_csc / usolve_csc).  The plan reads the
    matrix's values when it is built: it must not change while the plan lives (a CsMat's device
    mirror never does)."""

    def __init__(self, mat, lower=True):
        if isinstance(mat, CsMat):
            rows, cols = mat.shape
        elif isinstance(mat, DeviceCsMat):
            rows, cols = mat.rows, mat.cols
        else:
            raise TypeError("mat must be a CsMat or a DeviceCsMat")
        if rows != cols:
            raise SprsPanic("Non square matrix passed to solver")
        dev = mat.device() if isinstance(mat, CsMat) else mat
        self._mat, self._dev, self._ctx, self.n = mat, dev, dev.ctx, rows
        h = C.c_void_p()
        st = self._ctx.lib.sprs_b200_trisolve_plan(
            self._ctx.h, dev.h, _lib.TRI_LOWER if lower else _lib.TRI_UPPER, C.byref(h))
        if st == _lib.ERR_DIMENSION:
            raise SprsPanic("Non square matrix passed to solver")
        self._ctx.check(st)
        self._h = h

    def singular(self):
        """SingularMatrix every solve of this plan raises, or None."""
        idx, reason = C.c_uint64(), C.c_int()
        if not self._ctx.lib.sprs_b200_trisolve_singular(self._h, C.byref(idx), C.byref(reason)):
            return None
        return SingularMatrix(int(idx.value), _REASONS[reason.value])

    def _status(self, st):
        if st == _lib.ERR_SINGULAR:
            raise self.singular()
        self._ctx.check(st)

    def solve(self, rhs):
        """rhs (a contiguous float64 array of n entries) solved in place.  Raises SingularMatrix
        after leaving rhs as the reference leaves it."""
        _check_rhs(rhs)
        if rhs.size != self.n:
            raise SprsPanic("Dimension mismatch")
        self._status(self._ctx.lib.sprs_b200_trisolve_solve(
            self._h, rhs.ctypes.data_as(C.c_void_p), rhs.size))

    def solve_dev(self, d_rhs, stream=None):
        """Enqueue the solve of n doubles at device address d_rhs on `stream` (a cudaStream_t
        as an int; None = the legacy default stream).  Asynchronous; raises SingularMatrix
        (the work enqueued all the same) when the plan is singular.  One stream at a time."""
        self._status(self._ctx.lib.sprs_b200_trisolve_solve_dev(
            self._h, C.c_void_p(int(d_rhs)), C.c_void_p(int(stream) if stream else 0)))

    def free(self):
        if getattr(self, "_h", None):
            self._ctx.lib.sprs_b200_trisolve_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def diag_solve(diag, x):
    """sprs::linalg::diag_solve (sparse/linalg.rs): x (a contiguous, writeable float64 array)
    divided in place by diag, entry by entry, on the device."""
    from .sparse import Context
    _check_rhs(x)
    d = np.ascontiguousarray(diag, dtype=np.float64)
    if d.ndim != 1 or d.size != x.size:
        raise SprsPanic("assertion `left == right` failed\n  left: %d\n right: %d"
                        % (d.size, x.size))
    ctx = Context.default()
    ctx.check(ctx.lib.sprs_b200_diag_solve(ctx.h, d.ctypes.data_as(C.c_void_p),
                                           x.ctypes.data_as(C.c_void_p), x.size))


def _check_rhs(rhs):
    if not (isinstance(rhs, np.ndarray) and rhs.dtype == np.float64 and rhs.ndim == 1 and
            rhs.flags.c_contiguous and rhs.flags.writeable):
        raise TypeError("rhs must be a contiguous, writeable float64 array (DenseVectorMut)")


def _dense_rhs_solve(mat, rhs, lower, csr):
    """check_solver_dimensions (trisolve.rs:10-21), then the storage assert, then the solve."""
    _check_rhs(rhs)
    if not isinstance(mat, CsMat):
        raise TypeError("mat must be a CsMat")
    if mat.rows() != mat.cols():
        raise SprsPanic("Non square matrix passed to solver")
    if mat.cols() != rhs.size:
        raise SprsPanic("Dimension mismatch")
    if mat.is_csr() != csr:
        raise SprsPanic("Storage mismatch")
    plan = TriSolvePlan(mat, lower)
    try:
        plan.solve(rhs)
    finally:
        plan.free()


class trisolve:  # noqa: N801  (module path of the reference: sprs::linalg::trisolve)
    """Free functions of sprs/src/sparse/linalg/trisolve.rs.  `rhs` is solved in place; a
    singular matrix raises SingularMatrix (the reference's Err(LinalgError::SingularMatrix))
    with rhs left as the reference leaves it."""
    TriSolvePlan = TriSolvePlan

    @staticmethod
    def lsolve_csr_dense_rhs(lower_tri_mat, rhs):
        """trisolve.rs:30-73."""
        _dense_rhs_solve(lower_tri_mat, rhs, True, True)

    @staticmethod
    def usolve_csr_dense_rhs(upper_tri_mat, rhs):
        """trisolve.rs:219-262."""
        _dense_rhs_solve(upper_tri_mat, rhs, False, True)

    @staticmethod
    def lsolve_csc_dense_rhs(lower_tri_mat, rhs):
        """trisolve.rs:85-149."""
        _dense_rhs_solve(lower_tri_mat, rhs, True, False)

    @staticmethod
    def usolve_csc_dense_rhs(upper_tri_mat, rhs):
        """trisolve.rs:161-210."""
        _dense_rhs_solve(upper_tri_mat, rhs, False, False)


__all__ = ["BiCGSTAB", "NotConverged", "bicgstab", "TriSolvePlan", "trisolve", "diag_solve"]
