"""The device BiCGSTAB (csrc/solver.cu) BIT FOR BIT against tests/solver_model.py with the
device's reduction order and the library's own SpMV, at every step.

The order of every operation of a device step is fixed: unfused element-wise kernels
(--fmad=false), the scalar algebra on the host in the reference's order, and dot products summed
in a documented order that depends only on n and the grid (min(ceil(n / 1024), 4 * sm_count,
1024) blocks).  The model restates that order on the host, and its algebra is pinned to the
oracle by test_solver_model.py, so any difference here is a bug.  The sizes are derived from
sm_count so that the kernels' seams occur: tail chunks of 1-3 elements, threads that sweep the
grid twice, more than 256 block partials, final-reduce threads that add three partials.

The file sorts after the validated suites so that a surprise here cannot hide them under -x."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import solver_model as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


SIZES = ["1", "2", "3", "5", "6", "7", "9", "1023", "1024", "1025",
         "F-1", "F", "F+1", "2F+3", "F+4", "257 partials"]


def size_of(name, sm_count):
    """n for a SIZES entry; F = 4 * 256 * C, one chunk for every thread of the largest grid (C
    blocks).  F + 4 gives C partials with a second sweep, so where C > 512 some final-reduce
    threads add three.  None where the size reaches nothing new (257 partials need C > 256)."""
    cap = M.grid_cap(sm_count)
    full = M.CHUNK * M.RED_THREADS * cap
    if name == "257 partials":
        return M.RED_THREADS * M.CHUNK * M.RED_THREADS + 1 if cap > M.RED_THREADS else None
    if name.isdigit():
        return int(name)
    k, _, d = name.partition("F")
    return (int(k) if k else 1) * full + (int(d) if d else 0)


def sizes(sm_count):
    return [n for n in (size_of(s, sm_count) for s in SIZES) if n is not None]


def test_solver_sizes_reach_every_seam(sp):
    """Each reduction seam occurs at some size wherever the device allows it: more than 256
    partials needs sm_count >= 65, a final thread with 3 partials sm_count >= 129 (a 132-SM
    H100 SXM reaches all).  Unreachable seams are named, not failed."""
    sm = sp.Context.default().sm_count
    reached = set().union(*(M.seams(n, sm) for n in sizes(sm)))
    possible = set(M.ALL_SEAMS)
    if M.grid_cap(sm) <= M.RED_THREADS:
        possible.discard("more than 256 partials")
    if M.grid_cap(sm) <= 2 * M.RED_THREADS:
        possible.discard("final thread with 3 partials")
    missing = possible - reached
    assert not missing, "sizes for sm_count %d miss: %s" % (sm, sorted(missing))
    print("sm_count %d, grid cap %d: reached %s; not reachable on this device: %s"
          % (sm, M.grid_cap(sm), sorted(reached), sorted(set(M.ALL_SEAMS) - possible)))


def _csr_operand(sp, n, seed):
    csr, x0, b = M.dominant_system(n, seed)
    return sp.CsMat((n, n), *csr), csr, x0, b


def _model(sp, mirror, x0, b):
    ctx = sp.Context.default()
    return M.Model(M.device_matvec(ctx, mirror), M.device(M.grid_for(len(b), ctx.sm_count)),
                   x0, b)


def _indptr_bytes(ctx, mirror):
    ip, ipb, ind, dat = C.c_void_p(), C.c_int(), C.c_void_p(), C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_device_arrays(mirror.h, C.byref(ip), C.byref(ipb),
                                                    C.byref(ind), C.byref(dat)))
    return ipb.value


def _run(solver, tol, max_iter):
    from sprs_b200.linalg import NotConverged
    if isinstance(solver, M.Model):
        return solver.run(tol, max_iter)
    try:
        solver.run(tol, max_iter)
        return True
    except NotConverged:
        return False


def _sequence(dev, mod, what, finite):
    """new; 6 steps; soft + hard restart; 3 steps at thresholds 0 and 1e300; solve to 1e-9."""
    M.assert_same_state(dev, mod, what + " new")
    for it in range(1, 7):
        M.assert_same([dev.step()], [mod.step()], "%s step %d: err" % (what, it))
        M.assert_same_state(dev, mod, "%s step %d" % (what, it))
    dev.soft_restart()
    mod.soft_restart()
    M.assert_same_state(dev, mod, what + " soft restart")
    dev.hard_restart()
    mod.hard_restart()
    M.assert_same_state(dev, mod, what + " hard restart")
    for thresh in (0.0, 1e300):
        dev.with_restart_threshold(thresh)
        mod.with_restart_threshold(thresh)
        soft = mod.soft_restart_count()
        for it in range(1, 4):
            dev.step()
            mod.step()
            M.assert_same_state(dev, mod, "%s threshold %g step %d" % (what, thresh, it))
        if finite:  # 0 never restarts, 1e300 restarts after every step
            assert mod.soft_restart_count() == soft + (3 if thresh else 0)
    if finite:  # the comparison means something: no NaN hides a difference
        assert np.isfinite(mod.x()).all() and np.isfinite(mod.p()).all() and np.isfinite(mod.err())
    dev.with_restart_threshold(0.1)
    mod.with_restart_threshold(0.1)
    ok_dev, ok_mod = _run(dev, 1e-9, 300), _run(mod, 1e-9, 300)
    assert ok_dev == ok_mod, what + " solve: Ok/Err"
    M.assert_same_state(dev, mod, what + " solve")
    if finite:
        assert ok_mod and mod.hard_restart_count() >= 2


@pytest.mark.parametrize("size", SIZES)
def test_bicgstab_bits_by_size(sp, size):
    """A CSR host operand: the whole state bit-exact against the model after every operation
    of _sequence, and the same Ok/Err and counters from solve."""
    ctx = sp.Context.default()
    n = size_of(size, ctx.sm_count)
    if n is None:
        pytest.skip("%s: needs sm_count >= 65" % size)
    a, _, x0, b = _csr_operand(sp, n, 1000 + n)
    dev = sp.linalg.BiCGSTAB(a, x0, b)
    if os.environ.get("SPRS_B200_FORCE_INDPTR64") == "1":
        assert _indptr_bytes(ctx, a.device()) == 8
    _sequence(dev, _model(sp, a.device(), x0, b), "n=%d:" % n, finite=n >= 1000)


@pytest.mark.parametrize("form", ["csc", "device_mirror", "new_dev"])
def test_bicgstab_bits_every_operand_form(sp, form):
    """A CSC operand (the solver runs on its cached CSR form), a DeviceCsMat and
    sprs_b200_bicgstab_new_dev (x0, b in device memory) give the CSR host form's bits."""
    import torch
    from sprs_b200 import generate as G
    from sprs_b200.linalg import BiCGSTAB
    ctx = sp.Context.default()
    n = M.CHUNK * M.RED_THREADS * M.grid_cap(ctx.sm_count) + 3
    a, csr, x0, b = _csr_operand(sp, n, 77)
    ref = BiCGSTAB(a, x0, b)
    if form == "csc":
        import scipy.sparse as sparse
        c = sparse.csr_matrix((csr[2], csr[1], csr[0]), shape=(n, n)).tocsc()
        c.sort_indices()
        op = sp.CsMat.new_csc((n, n), c.indptr.astype(np.uint32), c.indices.astype(np.uint32),
                              c.data.copy())
        dev = BiCGSTAB(op, x0, b)
        mod = _model(sp, op.to_csr().device(), x0, b)
    elif form == "device_mirror":
        dev = BiCGSTAB(a.device(), x0, b)
        mod = _model(sp, a.device(), x0, b)
    else:
        d = G._device(ctx)
        xt = torch.from_numpy(x0).to(d)
        bt = torch.from_numpy(b).to(d)
        G._sync()  # sprs_b200.h: the arrays must be complete when new_dev is called
        h = C.c_void_p()
        ctx.check(ctx.lib.sprs_b200_bicgstab_new_dev(ctx.h, a.device().h, G._dptr(xt),
                                                     G._dptr(bt), n, C.byref(h)))
        del xt, bt  # copied by the solver
        dev = BiCGSTAB.__new__(BiCGSTAB)
        dev._a, dev._dev, dev._ctx, dev._h, dev._n = a, a.device(), ctx, h, n
        mod = _model(sp, a.device(), x0, b)
    M.assert_same_state(dev, ref, form + " new vs CSR")
    for it in range(1, 5):
        dev.step()
        ref.step()
        mod.step()
        M.assert_same_state(dev, ref, "%s step %d vs CSR" % (form, it))
        M.assert_same_state(dev, mod, "%s step %d vs model" % (form, it))
    dev.hard_restart()
    ref.hard_restart()
    M.assert_same_state(dev, ref, form + " hard restart vs CSR")
    assert _run(dev, 1e-9, 300) and _run(ref, 1e-9, 300)
    M.assert_same_state(dev, ref, form + " solve vs CSR")


def test_bicgstab_bits_empty_system(sp, O):
    """n = 0: the oracle's state (err 0, rho 0); solve is Ok after 1 iteration, 1 hard restart."""
    ip = np.zeros(1, np.uint32)
    a = sp.CsMat((0, 0), ip, np.zeros(0, np.uint32), np.zeros(0))
    dev = sp.linalg.BiCGSTAB(a, np.zeros(0), np.zeros(0))
    ref = O.BiCGSTAB((ip, np.zeros(0, np.uint32), np.zeros(0)), np.zeros(0), np.zeros(0))
    mod = _model(sp, a.device(), np.zeros(0), np.zeros(0))
    M.assert_same_state(dev, ref, "n=0 new vs oracle")
    M.assert_same_state(dev, mod, "n=0 new vs model")
    assert (dev.err(), dev.rho()) == (0.0, 0.0)
    ok_ref = O.lib().oracle_bicgstab_solve(ref._h, C.c_double(1e-9), C.c_size_t(10))
    assert ok_ref and _run(dev, 1e-9, 10) and _run(mod, 1e-9, 10)
    M.assert_same_state(dev, ref, "n=0 solve vs oracle")
    M.assert_same_state(dev, mod, "n=0 solve vs model")
    assert (dev.iteration_count(), dev.hard_restart_count()) == (1, 1)


def test_bicgstab_bits_exact_initial_guess(sp, O):
    """x0 solves the system exactly (at most 2 entries per row, so A x0 has the same bits in
    every summation order): r = 0, the first step's alpha = 0/0, and the device reaches the
    oracle's and the model's NaN state and NotConverged (NaN payloads may differ)."""
    import scipy.sparse as sparse
    n = 5000
    rng = np.random.default_rng(5)
    off = rng.standard_normal(n)
    cols = (np.arange(n) + 1 + rng.integers(0, n - 1, n)) % n  # never the diagonal
    a = sparse.csr_matrix((off, (np.arange(n), cols)), shape=(n, n))
    a = (a + sparse.diags(np.abs(off) + 1.0)).tocsr()
    a.sort_indices()
    assert np.diff(a.indptr).max() == 2
    csr = (a.indptr.astype(np.uint32), a.indices.astype(np.uint32), a.data.copy())
    x0 = rng.standard_normal(n)
    b = O.mul_acc_mat_vec_csr(*csr, x0, np.zeros(n))
    op = sp.CsMat((n, n), *csr)
    dev = sp.linalg.BiCGSTAB(op, x0, b)
    ref = O.BiCGSTAB(csr, x0, b)
    mod = _model(sp, op.device(), x0, b)
    M.assert_same_state(dev, ref, "exact x0: new vs oracle")
    M.assert_same_state(dev, mod, "exact x0: new vs model")
    assert dev.err() == 0.0 and not np.any(dev.r())
    ok_ref = O.lib().oracle_bicgstab_solve(ref._h, C.c_double(1e-9), C.c_size_t(3))
    assert not ok_ref and not _run(dev, 1e-9, 3) and not _run(mod, 1e-9, 3)
    assert np.isnan(ref.err()) and np.isnan(ref.x()).all()
    M.assert_same_state(dev, ref, "exact x0: solve vs oracle")
    M.assert_same_state(dev, mod, "exact x0: solve vs model")


def test_bicgstab_bits_rmat_full_size(sp):
    """An R-MAT of ~4M rows (n % 4 == 3) with the hot set at its `auto` setting, x0 and b on the
    device (sprs_b200_bicgstab_new_dev): five steps bit-exact and finite."""
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 4_000_003
    a = G.rmat_csr(ctx, n, 16, seed=0x5EED0006)
    x0 = G.normal_vector(ctx, n, 11)
    b = G.normal_vector(ctx, n, 12)
    G._sync()  # sprs_b200.h: the arrays must be complete when new_dev is called
    h = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_bicgstab_new_dev(ctx.h, a.mirror.h, G._dptr(x0), G._dptr(b), n,
                                                 C.byref(h)))
    dev = sp.linalg.BiCGSTAB.__new__(sp.linalg.BiCGSTAB)
    dev._a, dev._dev, dev._ctx, dev._h, dev._n = a, a.mirror, ctx, h, n
    mod = _model(sp, a.mirror, x0.cpu().numpy(), b.cpu().numpy())
    assert M.grid_for(n, ctx.sm_count) == M.grid_cap(ctx.sm_count)
    M.assert_same_state(dev, mod, "R-MAT new")
    for it in range(1, 6):
        dev.step()
        mod.step()
        M.assert_same_state(dev, mod, "R-MAT step %d" % it)
        for name in ("x", "r", "rhat", "p"):
            assert np.isfinite(getattr(mod, name)()).all(), (it, name)
        assert np.isfinite([mod.err(), mod.rho()]).all(), it
    dev.free()


def test_bicgstab_bits_indptr64_child_process():
    """The step-by-step sizes again with SPRS_B200_FORCE_INDPTR64=1 (read once per process):
    the uint64-indptr SpMV feeds the solver."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPRS_B200_")}
    env["SPRS_B200_FORCE_INDPTR64"] = "1"
    if os.environ.get("SPRS_B200_EMU") == "1":
        env["SPRS_B200_EMU"] = "1"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider",
                        os.path.abspath(__file__), "-k", "test_bicgstab_bits_by_size"],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
