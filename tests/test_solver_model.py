"""tests/solver_model.py with sequential sums and the oracle's SpMV is the oracle's BiCGSTAB
(oracle/sprs_oracle.cpp, a restatement of bicgstab.rs) BIT FOR BIT: every vector, err, rho and
the three counters, after new, after every step, after explicit restarts and after solve.

This pins the model's algebra to the reference, so that the device test
(test_gpu_zzz_solver_bits.py), which swaps in the device's summation order and SpMV, checks the
solver against an algebra that is itself checked.  No GPU needed."""
import numpy as np
import pytest

import solver_model as M


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


SIZES = list(range(8)) + [3001]


@pytest.mark.parametrize("thresh", [0.0, 0.1, 1e300])
@pytest.mark.parametrize("n", SIZES)
def test_model_matches_oracle_step_by_step(O, n, thresh):
    """new, six steps at the threshold, an explicit soft and hard restart: the whole state
    after each.  n = 0..7 includes the empty system and n = 1, which is solved by its first
    step and then meets 0/0 (NaN where the oracle has NaN)."""
    csr, x0, b = M.dominant_system(n, 100 + n)
    ref = O.BiCGSTAB(csr, x0, b)
    mod = M.Model(M.oracle_matvec(O, *csr), M.sequential, x0, b)
    M.assert_same_state(mod, ref, "new")
    ref.with_restart_threshold(thresh)
    mod.with_restart_threshold(thresh)
    for it in range(1, 7):
        e_ref, e_mod = ref.step(), mod.step()
        M.assert_same_state(mod, ref, "step %d" % it)
        M.assert_same([e_mod], [e_ref], "step %d: returned err" % it)
    mod.soft_restart()
    ref.soft_restart()
    M.assert_same_state(mod, ref, "soft restart")
    mod.hard_restart()
    ref.hard_restart()
    M.assert_same_state(mod, ref, "hard restart")
    if n > 100:
        # the comparison means something: nothing degenerated to NaN on the way
        assert np.isfinite(mod.x()).all() and np.isfinite(mod.err())
        if thresh == 0.0:
            assert mod.soft_restart_count() == 1  # only the explicit one
        if thresh == 1e300:
            assert mod.soft_restart_count() == 7  # every step, and the explicit one


@pytest.mark.parametrize("n", SIZES)
def test_model_solve_matches_oracle(O, n):
    """solve to 1e-9 (Ok on the large system) and solve with tol = 0 (Err after max_iter)."""
    csr, x0, b = M.dominant_system(n, 200 + n)
    ok_ref, ref = O.BiCGSTAB.solve(csr, x0, b, 1e-9, 200)
    ok_mod, mod = M.Model.solve(M.oracle_matvec(O, *csr), M.sequential, x0, b, 1e-9, 200)
    assert ok_mod == ok_ref
    M.assert_same_state(mod, ref, "solve(1e-9)")
    if n > 100:
        assert ok_mod and mod.hard_restart_count() >= 1 and mod.iteration_count() > 5
    if n == 0:  # the empty system: err 0 < tol after one step and one hard restart
        assert ok_mod and (mod.iteration_count(), mod.hard_restart_count()) == (1, 1)
    ok_ref, ref = O.BiCGSTAB.solve(csr, x0, b, 0.0, 4)
    ok_mod, mod = M.Model.solve(M.oracle_matvec(O, *csr), M.sequential, x0, b, 0.0, 4)
    assert not ok_ref and not ok_mod
    M.assert_same_state(mod, ref, "solve(0)")


def _literal_device_sum(terms, grid):
    """csrc/solver.cu's reduction transcribed loop for loop, one Python float at a time."""
    n, threads = len(terms), grid * M.RED_THREADS
    n_chunks = (n + 3) // 4
    sums = []
    for t in range(threads):  # FOR_EACH_CHUNK + the `k < cnt` sums of dot2_kernel
        s, c = 0.0, t
        while c < n_chunks:
            for k in range(4):
                if 4 * c + k < n:
                    s = s + float(terms[4 * c + k])
            c += threads
        sums.append(s)

    def block_reduce2(v):
        warps = []
        for w in range(8):
            lane = v[32 * w:32 * w + 32]
            for o in (16, 8, 4, 2, 1):  # __shfl_down_sync: a lane past 31 reads its own value
                lane = [lane[i] + (lane[i + o] if i + o < 32 else lane[i]) for i in range(32)]
            warps.append(lane[0])
        a = warps[0]
        for w in range(1, 8):
            a = a + warps[w]
        return a

    partials = [block_reduce2(sums[256 * b:256 * b + 256]) for b in range(grid)]
    final = []
    for t in range(256):  # final_reduce_kernel
        s, b = 0.0, t
        while b < grid:
            s = s + partials[b]
            b += 256
        final.append(s)
    return block_reduce2(final)


@pytest.mark.parametrize("grid,n", [(1, 1), (1, 7), (1, 1023), (2, 2 * 1024 * 3 + 2),
                                    (300, 300 * 1024 + 3), (520, 520 * 1024 + 1)])
def test_device_reduction_matches_a_literal_transcription(grid, n):
    """The vectorised device(grid) order equals the kernels' loops transcribed one add at a
    time, on terms of widely different magnitudes (where a change of order shows): tails, two
    sweeps, more than 256 partials and final threads that add three."""
    rng = np.random.default_rng(n)
    terms = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 9, n)
    got = M.device(grid)(terms)
    want = _literal_device_sum(terms, grid)
    assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (got, want)
    if n > 1000:  # and the order is not the sequential one
        assert got != M.sequential(terms)
