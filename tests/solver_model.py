"""Host model of BiCGSTAB (bicgstab.rs:95-300) whose every operation has a fixed order, so a run
can be compared BIT FOR BIT with the oracle's restatement or with the device solver.

The algebra is that of the reference, one rounding per operation: every product and every sum
or difference is its own numpy operation (numpy never fuses them), and the scalar algebra is done
on float64 scalars in the reference's order.  Two parts are plug-ins:

  matvec   y = A x for a fresh y: `oracle_matvec` (the oracle's sequential row sums),
           `device_matvec` (the library's sprs_b200_spmv_dev on a device mirror -- the entry the
           solver's own SpMV calls, so it gives the same bits for the same mirror) or
           `model_matvec` (the SpMV's order restated on the host, tests/spmv_model.py).
  reduce   the sum of a vector of products: `sequential` (+0.0 + t0 + t1 + ..., vec.rs:846-881,
           907-913, the oracle's order) or `device(grid)`, the order of csrc/solver.cu:
             * thread t of the grid's grid * 256 threads visits chunks t, t + grid*256, ... of 4
               consecutive elements, adding each chunk's elements in index order to a running sum
               that starts at +0.0;
             * a warp combines its lanes with shfl_down 16/8/4/2/1 (lane i += lane i + o);
             * lane 0 of warps 0..7 are added one after another (block_reduce2);
             * final_reduce_kernel: thread t adds partials t, t + 256, ... from +0.0, then the same
               warp tree and warp sequence.
           Unused lanes, chunks and partials are padded with +0.0.  A running sum that starts at
           +0.0 never becomes -0.0 under round-to-nearest, and x + (+0.0) == x for every other x
           (NaN and infinities included), so the padding changes no bit.

No np.sum / np.dot / `@` anywhere: those sum pairwise or through BLAS, in an order that is not the
model's.  Sequential sums use np.add.accumulate, which is defined as r[i] = r[i-1] + a[i].

Test helper, not part of the package."""
import numpy as np

import exact

RED_THREADS = 256      # csrc/solver.cu: threads per block of every solver kernel
RED_MAX_BLOCKS = 1024  # csrc/solver.cu: most partial sums of one reduction
CHUNK = 4              # elements per chunk of the grid-stride loops
WARP = 32


# ---------------------------------------------------------------- launch shape
def grid_cap(sm_count):
    """Most blocks of a solver kernel: min(4 * sm_count, 1024)."""
    return min(4 * sm_count, RED_MAX_BLOCKS)


def grid_for(n, sm_count):
    """Blocks of every solver kernel for n rows (create_common): min(ceil(n / 1024), cap), >= 1."""
    return max(1, min(-(-n // (CHUNK * RED_THREADS)), grid_cap(sm_count)))


def seams(n, sm_count):
    """The reduction seams a solve of n rows reaches on a device with sm_count SMs."""
    grid = grid_for(n, sm_count)
    out = set()
    if n % CHUNK:
        out.add("tail of %d" % (n % CHUNK))
    if -(-n // CHUNK) > grid * RED_THREADS:
        out.add("thread with 2+ chunks")
    if grid > RED_THREADS:
        out.add("more than 256 partials")
    if grid > 2 * RED_THREADS:
        out.add("final thread with 3 partials")
    return out


ALL_SEAMS = ("tail of 1", "tail of 2", "tail of 3", "thread with 2+ chunks",
             "more than 256 partials", "final thread with 3 partials")


# ---------------------------------------------------------------- reductions
def sequential(terms):
    """+0.0 + t0 + t1 + ... in index order (the oracle's dot / squared norm)."""
    terms = np.asarray(terms, dtype=np.float64)
    if terms.size == 0:
        return np.float64(0.0)
    return np.add.accumulate(np.concatenate(([0.0], terms)))[-1]


def _block_tree(s):
    """block_reduce2 on per-thread sums s of shape (blocks, 256): one result per block."""
    s = s.reshape(s.shape[0], RED_THREADS // WARP, WARP)
    for o in (16, 8, 4, 2, 1):
        s = s[..., :o] + s[..., o:2 * o]  # only lanes < o matter for lane 0
    s = s[..., 0]
    a = s[:, 0]
    for w in range(1, RED_THREADS // WARP):
        a = a + s[:, w]
    return a


def device(grid):
    """The reduction of csrc/solver.cu over `grid` blocks (see the module docstring)."""
    def reduce(terms):
        terms = np.asarray(terms, dtype=np.float64)
        n = terms.size
        if n == 0:
            return np.float64(0.0)  # finish_reduce: no kernel runs, the host sets 0
        threads = grid * RED_THREADS
        sweeps = -(-n // (CHUNK * threads))
        pad = np.zeros(sweeps * threads * CHUNK)
        pad[:n] = terms
        pad = pad.reshape(sweeps, threads, CHUNK)  # [sweep, thread, k] = element 4c + k
        acc = np.zeros(threads)
        for s in range(sweeps):
            for k in range(CHUNK):
                acc = acc + pad[s, :, k]
        partials = _block_tree(acc.reshape(grid, RED_THREADS))
        rounds = -(-grid // RED_THREADS)
        pp = np.zeros(rounds * RED_THREADS)
        pp[:grid] = partials
        pp = pp.reshape(rounds, RED_THREADS)
        acc = np.zeros(RED_THREADS)
        for j in range(rounds):
            acc = acc + pp[j]
        return _block_tree(acc.reshape(1, RED_THREADS))[0]
    return reduce


# ---------------------------------------------------------------- systems and matvecs
def dominant_system(n, seed, max_off=8):
    """Non-symmetric, strictly diagonally dominant n x n CSR (u32) with ragged rows of
    0..max_off off-diagonal N(0,1) entries; x0 and b N(0,1)."""
    import scipy.sparse as sparse
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, max_off + 1, n)
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, max(n, 1), rows.size)
    a = sparse.csr_matrix((rng.standard_normal(rows.size), (rows, cols)), shape=(n, n))
    a.sum_duplicates()
    a = (a + sparse.diags(np.asarray(abs(a).sum(axis=1)).ravel() + 1.0)).tocsr()
    a.sort_indices()
    csr = (a.indptr.astype(np.uint32), a.indices.astype(np.uint32), a.data.copy())
    return csr, rng.standard_normal(n), rng.standard_normal(n)


def oracle_matvec(O, indptr, indices, data):
    """y = A x with the oracle's row sums (prod.rs:103-127 into a zero vector)."""
    rows = len(indptr) - 1
    return lambda x: O.mul_acc_mat_vec_csr(indptr, indices, data, x, np.zeros(rows))


def model_matvec(indptr, indices, data):
    """y = A x in the device SpMV's order, restated on the host (tests/spmv_model.py)."""
    import spmv_model
    return lambda x: spmv_model.spmv(indptr, indices, data, x)


def device_matvec(ctx, mirror):
    """y = A x through sprs_b200_spmv_dev on a CSR DeviceCsMat, with torch buffers."""
    import torch
    from sprs_b200 import generate as G
    dev = G._device(ctx)
    rows = mirror.rows

    def matvec(x):
        if rows == 0:
            return np.zeros(0)
        xt = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(dev)
        yt = torch.empty(rows, dtype=torch.float64, device=dev)
        G.spmv(ctx, mirror, xt, yt)
        G._sync()
        return yt.cpu().numpy()
    return matvec


# ---------------------------------------------------------------- the solver
class Model:
    """BiCGSTAB::new / step / soft_restart / hard_restart / solve with the accessors of
    sprs_b200.linalg.BiCGSTAB and oracle.BiCGSTAB (x(), err(), iteration_count(), ...)."""

    def __init__(self, matvec, reduce, x0, b):
        """bicgstab.rs:120-146: r = b - A x0, rhat = p = r, err = |r|, rho = err^2."""
        self._matvec, self._reduce = matvec, reduce
        self._b = np.array(b, dtype=np.float64)
        self._x = np.array(x0, dtype=np.float64)
        self._iterations = self._soft = self._hard = 0
        self._threshold = np.float64(0.1)
        self._residual()

    @classmethod
    def solve(cls, matvec, reduce, x0, b, tol, max_iter):
        """bicgstab.rs:151-175: (ok, model), as oracle.BiCGSTAB.solve returns."""
        m = cls(matvec, reduce, x0, b)
        return m.run(tol, max_iter), m

    def _residual(self):
        ax = self._matvec(self._x)
        self._r = self._b - ax
        self._rhat = self._r.copy()
        self._p = self._r.copy()
        self._err = np.sqrt(self._reduce(self._r * self._r))
        self._rho = self._err * self._err

    def soft_restart(self):
        """bicgstab.rs:177-184."""
        self._soft += 1
        self._rhat = self._r.copy()
        self._rho = self._err * self._err
        self._p = self._r.copy()

    def hard_restart(self):
        """bicgstab.rs:186-196."""
        self._hard += 1
        self._residual()  # r, err, and the soft restart's rhat = p = r, rho = err^2

    def step(self):
        """bicgstab.rs:198-234; returns err."""
        with np.errstate(all="ignore"):
            self._iterations += 1
            v = self._matvec(self._p)
            alpha = self._rho / self._reduce(self._rhat * v)
            h = self._x + self._p * alpha
            s = self._r - v * alpha
            t = self._matvec(s)
            omega = self._reduce(t * s) / self._reduce(t * t)
            self._x = h + omega * s
            self._r = s - t * omega
            self._err = np.sqrt(self._reduce(self._r * self._r))
            rho_prev = self._rho
            self._rho = self._reduce(self._rhat * self._r)
            if np.abs(self._rho) / (self._err * self._err) < self._threshold:
                self.soft_restart()
            else:
                beta = (self._rho / rho_prev) * (alpha / omega)
                self._p = self._r + (self._p - v * omega) * beta
        return self._err

    def run(self, tol, max_iter):
        """The loop of solve: True for Ok (the true error confirmed below tol), False for Err."""
        for _ in range(max_iter):
            self.step()
            if self._err < tol:
                self.hard_restart()
                if self._err < tol:
                    return True
        return False

    def with_restart_threshold(self, thresh):
        self._threshold = np.float64(thresh)
        return self

    def x(self):
        return self._x

    def r(self):
        return self._r

    def rhat(self):
        return self._rhat

    def p(self):
        return self._p

    def b(self):
        return self._b

    def err(self):
        return float(self._err)

    def rho(self):
        return float(self._rho)

    def iteration_count(self):
        return self._iterations

    def soft_restart_count(self):
        return self._soft

    def hard_restart_count(self):
        return self._hard

    def soft_restart_threshold(self):
        return float(self._threshold)


# ---------------------------------------------------------------- comparison
def assert_same(got, want, what):
    """Bit-equality; where `want` holds a NaN, any NaN (payloads differ between host and GPU)."""
    want = np.asarray(want, dtype=np.float64)
    if np.isnan(want).any():
        exact.assert_same_class(got, want, what)
    else:
        exact.assert_bits(got, want, what)


def assert_same_state(got, want, what):
    """x, r, rhat, p, b, err, rho, the three counters and the threshold of two solvers (any of
    Model, oracle.BiCGSTAB, sprs_b200.linalg.BiCGSTAB) agree bit for bit."""
    for name in ("x", "r", "rhat", "p", "b"):
        assert_same(getattr(got, name)(), getattr(want, name)(), "%s: %s" % (what, name))
    assert_same([got.err(), got.rho(), got.soft_restart_threshold()],
          [want.err(), want.rho(), want.soft_restart_threshold()],
          what + ": (err, rho, threshold)")
    counts = lambda s: (s.iteration_count(), s.soft_restart_count(), s.hard_restart_count())
    assert counts(got) == counts(want), "%s: (iterations, soft, hard restarts) %s, want %s" % (
        what, counts(got), counts(want))
