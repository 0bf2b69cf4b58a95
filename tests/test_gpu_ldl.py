"""The LDL^T factorization on the device (csrc/ldl.cu, sprs_b200.ldl) against the CPU
restatement of the sprs-ldl crate (tests/ldl_oracle.cpp): L's colptr, indices and values, D,
x of solve and the SingularMatrix, bit for bit on view(np.uint64) (NaN by class), and the
reference's own known answers (tests/golden/ldl_fixtures.json).

Small tests run on the emulator as well (tests/test_emu_ldl.py runs them on the emulated build
that has the factorization, tests/emu_ldl.py); `*_large`, `*_child_process` and `test_cpp*`
ones need the H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import ldl_oracle as LO
from conftest import ROOT

pytestmark = pytest.mark.gpu

if os.environ.get("SPRS_B200_EMU_LDL_LIB"):  # test infrastructure: the emulated build with the
    import sprs_b200 as _sp                  # factorization (tests/emu_ldl.py)
    _sp._lib.LIB_PATH = os.environ["SPRS_B200_EMU_LDL_LIB"]

KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "ldl_fixtures.json")))
NUMERIC = "diagonal element is a numeric 0"


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    lib = sprs_b200._lib.load()  # the product library must export the factorization
    if os.path.basename(sprs_b200._lib.LIB_PATH).startswith("libsprs_b200_emu") and \
            not hasattr(lib, "sprs_b200_ldl_symbolic"):
        pytest.skip("the emulated build of tests/emu has no LDL^T: tests/test_emu_ldl.py runs "
                    "this file on one that has")
    return sprs_b200


def f(v):
    return np.array([float(s) for s in v])


def same(got, want, what):
    d = LO.first_difference(got, want)
    assert d is None, "%s: %s" % (what, d)


def as_storage(m, storage):
    m = sps.csr_matrix(m) if storage == "CSR" else sps.csc_matrix(m)
    m.sort_indices()
    return m


def mirror(sp, m, storage, idx=np.uint32):
    cls = sp.CsMat.new if storage == "CSR" else sp.CsMat.new_csc
    return cls(m.shape, m.indptr.astype(idx), m.indices.astype(idx), m.data)


def run(sp, m, storage="CSC", perm=None, check=True, b=None, idx=np.uint32, seed=0):
    """Factor m (scipy, square) on the device through the Python mirror and on the oracle;
    the same SingularMatrix (or none), and when none the same L, D and x of a solve.  Returns
    the numeric factor (None if singular)."""
    m = as_storage(m, storage)
    n = m.shape[0]
    mat = mirror(sp, m, storage, idx)
    ldl = sp.ldl
    check = ldl.SymmetryCheck.CheckSymmetry if check else ldl.SymmetryCheck.DontCheckSymmetry
    fa = LO.Factor(m.indptr, m.indices, perm)
    want_err = fa.update(m.data)
    try:
        num = ldl.LdlNumeric.new_perm(mat, np.arange(n) if perm is None else perm, check)
        got_err = None
    except sp.SingularMatrix as e:
        got_err, num = e.index, None
        assert e.reason == NUMERIC and str(e) == "Singular matrix at index %d (%s)" % (e.index, NUMERIC)
    assert got_err == want_err
    if num is None:
        return None
    assert num.nnz() == fa.nnz() and num.problem_size() == n
    cp, li, lv = fa.l()
    lm = num.l()
    assert lm.is_csc() and lm.shape == (n, n)
    assert np.array_equal(lm.indptr.astype(np.uint64), cp)
    assert np.array_equal(lm.indices.astype(np.uint64), li)
    same(lm.data, lv, "L")
    same(num.d(), fa.diag(), "D")
    rhs = np.random.default_rng(seed).standard_normal(n) if b is None else np.asarray(b, float)
    same(num.solve(rhs), fa.solve(rhs), "x")
    return num


# ---- inputs
def laplacian(shape):
    """The 2-D 5-point / 3-D 7-point Laplacian of a grid, natural (row-major) order."""
    ops = []
    for k, s in enumerate(shape):
        t = sps.diags([-np.ones(s - 1), 2 * np.ones(s), -np.ones(s - 1)], [-1, 0, 1])
        eyes = [sps.identity(x) for x in shape]
        eyes[k] = t
        op = eyes[0]
        for e in eyes[1:]:
            op = sps.kron(op, e)
        ops.append(op)
    return sps.csr_matrix(sum(ops))


def nested_dissection(shape):
    """A geometric nested-dissection order of a grid: both halves, then the middle plane of
    the longest axis, recursively (perm[k] = the grid point that is row k)."""
    ids = np.arange(int(np.prod(shape))).reshape(shape)
    out = []

    def rec(block):
        if block.size <= 8:
            out.extend(block.ravel().tolist())
            return
        ax = int(np.argmax(block.shape))
        mid = block.shape[ax] // 2
        rec(np.take(block, range(mid), axis=ax))
        rec(np.take(block, range(mid + 1, block.shape[ax]), axis=ax))
        out.extend(np.take(block, [mid], axis=ax).ravel().tolist())

    rec(ids)
    return np.array(out, dtype=np.int64)


def random_spd(rng, n, per_row):
    m = sps.random(n, n, density=min(1.0, per_row / n), random_state=rng,
                   data_rvs=rng.standard_normal)
    a = (m + m.T).tocsr()
    return sps.csr_matrix(a + sps.diags(1.0 + np.asarray(abs(a).sum(axis=1)).ravel()))


def random_indefinite(rng, n, per_row):
    """Symmetric, diagonal of random sign dominating its row: factorable, D of both signs."""
    a = random_spd(rng, n, per_row).tolil()
    sign = rng.choice([-1.0, 1.0], n)
    for i in range(n):
        a[i, i] = a[i, i] * sign[i]
    return sps.csr_matrix(a)


# ---- 1. the reference's known answers
def test_ldl_kat_factor_solve1(sp):
    k = KATS["test_mat1"]
    mat = sp.CsMat.new_csc((10, 10), k["indptr"], k["indices"], f(k["data"]))
    num = sp.ldl.LdlNumeric.new(mat)
    lm = num.l()
    assert lm.indptr.tolist() == k["l_colptr"] and lm.indices.tolist() == k["l_indices"]
    same(lm.data, f(k["l_data"]), "L")
    same(num.d(), f(k["d"]), "D")
    same(num.solve(f(k["b"])), f(k["x"]), "x")
    assert num.nnz() == 13 and num.problem_size() == 10
    # the same through the builder and the symbolic / factor split
    sym = sp.ldl.Ldl.new().fill_in_reduction(sp.ldl.FillInReduction.NoReduction).symbolic(mat)
    assert sym.nnz() == 13
    same(sym.factor(mat).solve(f(k["b"])), f(k["x"]), "x")


def test_ldl_kat_solve1(sp):
    k = KATS["test_mat1"]
    l = sp.CsMat.new_csc((10, 10), k["l_colptr"], k["l_indices"], f(k["l_data"]))
    x = f(k["b"])
    sp.ldl.ldl_lsolve(l, x)
    same(x, f(k["lsolve"]), "lsolve")
    sp.linalg.diag_solve(f(k["d"]), x)
    same(x, f(k["dsolve"]), "dsolve")
    sp.ldl.ldl_ltsolve(l, x)
    same(x, f(k["x"]), "ltsolve")


def test_ldl_kat_permuted(sp):
    k = KATS["permuted_ldl_solve"]
    for storage in ("CSC", "CSR"):  # the matrix is symmetric: both storages hold one array set
        cls = sp.CsMat.new_csc if storage == "CSC" else sp.CsMat.new
        mat = cls((4, 4), k["indptr"], k["indices"], f(k["data"]))
        num = sp.ldl.LdlNumeric.new_perm(mat, k["perm"], sp.ldl.SymmetryCheck.CheckSymmetry)
        assert num.solve(f(k["b"])).tolist() == f(k["x"]).tolist()


def test_ldl_builder_orderings(sp):
    k = KATS["permuted_ldl_solve"]
    mat = sp.CsMat.new_csc((4, 4), k["indptr"], k["indices"], f(k["data"]))
    for method in (sp.ldl.FillInReduction.ReverseCuthillMcKee,
                   sp.ldl.FillInReduction.CAMDSuiteSparse):
        b = sp.ldl.Ldl.new().fill_in_reduction(method)
        with pytest.raises(NotImplementedError, match="NoReduction.*new_perm"):
            b.numeric(mat)
    with pytest.raises(NotImplementedError):
        sp.ldl.Ldl.new().numeric(mat)  # the reference's default is ReverseCuthillMcKee
    num = sp.ldl.Ldl.new().fill_in_reduction(sp.ldl.FillInReduction.NoReduction) \
        .check_symmetry(sp.ldl.SymmetryCheck.DontCheckSymmetry).numeric(mat)
    assert np.allclose(num.solve(f(k["b"])), f(k["x"]))


# ---- 2. storages, permutations, structures
@pytest.mark.parametrize("storage", ["CSR", "CSC"])
@pytest.mark.parametrize("permuted", [False, True])
def test_ldl_random_spd(sp, storage, permuted):
    rng = np.random.default_rng(1 + permuted)
    for n, per_row in ((50, 4), (700, 9)):
        a = random_spd(rng, n, per_row)
        run(sp, a, storage, rng.permutation(n) if permuted else None, seed=n)


def test_ldl_random_indefinite(sp):
    rng = np.random.default_rng(3)
    a = random_indefinite(rng, 600, 7)
    num = run(sp, a, "CSR", rng.permutation(600))
    d = num.d()
    assert (d < 0).any() and (d > 0).any()


@pytest.mark.parametrize("shape", [(30, 30), (9, 9, 9)])
@pytest.mark.parametrize("order", ["natural", "nd"])
def test_ldl_laplacians(sp, shape, order):
    a = laplacian(shape)
    perm = None if order == "natural" else nested_dissection(shape)
    run(sp, a, "CSC", perm)


def test_ldl_forest(sp):
    """Isolated vertices and independent blocks: an elimination forest of many roots."""
    rng = np.random.default_rng(4)
    blocks = [random_spd(rng, s, 3) for s in (1, 5, 1, 40, 2, 1, 17)]
    a = sps.block_diag(blocks, format="csr")
    run(sp, a, "CSR")
    run(sp, a, "CSC", rng.permutation(a.shape[0]))


def test_ldl_arrow(sp):
    """Every row reaches the last: its pattern is all n - 1 columns."""
    n = 3000
    a = sps.lil_matrix((n, n))
    a.setdiag(float(n))
    a[n - 1, :n - 1] = 1.0
    a[:n - 1, n - 1] = 1.0
    num = run(sp, sps.csr_matrix(a), "CSR")
    assert num.nnz() == n - 1


def test_ldl_chain_large(sp):
    """A tridiagonal 10^5 chain: every row waits for the one before."""
    n = 100_000
    rng = np.random.default_rng(5)
    off = rng.standard_normal(n - 1)
    a = sps.diags([off, 4.0 + rng.random(n), off], [-1, 0, 1], format="csr")
    run(sp, a, "CSR")


def test_ldl_signed_zeros_and_non_finite(sp):
    rng = np.random.default_rng(6)
    a = random_spd(rng, 200, 5).tocsr()
    a.sort_indices()
    # off-diagonal -0.0 (a symmetric pair): the workspace starts at +0.0, so y becomes +0.0
    r = sps.triu(a, 1).tocoo()
    i, j = r.row[0], r.col[0]
    b = a.tolil()
    b[i, j] = b[j, i] = -0.0
    run(sp, sps.csr_matrix(b), "CSR")
    for bad in (np.nan, np.inf, -np.inf):
        c = a.tolil()
        c[i, j] = c[j, i] = bad
        if np.isnan(bad):  # NaN != NaN: not symmetric for the reference's check
            with pytest.raises(sp.SprsPanic, match="^Matrix is not symmetric$"):
                run(sp, sps.csr_matrix(c), "CSC")
        run(sp, sps.csr_matrix(c), "CSC", check=not np.isnan(bad))


def zero_pivot(n, k, how):
    """The 1-D Laplacian with D_k == 0: how "0.0" / "-0.0" stores that diagonal and zeros row
    and column k's other entries; "cancel" makes a_kk equal to the term D_k subtracts."""
    a = laplacian((n,)).tocsr()
    a.sort_indices()
    rows = np.repeat(np.arange(n), np.diff(a.indptr))
    at = np.flatnonzero((rows == a.indices) & (rows == k))[0]
    if how == "cancel":
        fa = LO.Factor(a.indptr, a.indices)
        fa.update(a.data)
        y = -1.0
        a.data[at] = (y / fa.diag()[k - 1]) * y
    else:
        a.data[((rows == k) | (a.indices == k)) & (rows != a.indices)] = 0.0
        a.data[at] = float(how)
    return a


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("how", ["0.0", "-0.0", "cancel"])
def test_ldl_zero_pivot(sp, where, how):
    n = 9
    k = {"first": 0, "middle": 4, "last": n - 1}[where]
    if how == "cancel" and k == 0:
        pytest.skip("row 0 has no term to cancel")
    m = zero_pivot(n, k, how)
    fa = LO.Factor(m.indptr, m.indices)
    assert fa.update(m.data) == k
    assert run(sp, m, "CSR") is None
    # a second zero pivot later: only the first counts
    if k < n - 1:
        m2 = zero_pivot(n, k, how)
        m2.data[m2.indptr[n - 1]:m2.indptr[n]][m2.indices[m2.indptr[n - 1]:m2.indptr[n]] == n - 1] = 0.0
        assert run(sp, m2, "CSC") is None


def test_ldl_dont_check_symmetry(sp):
    """A non-symmetric input is factored from the entries the reference reads."""
    rng = np.random.default_rng(8)
    a = random_spd(rng, 300, 6).tolil()
    a[5, 200] = 3.0   # no partner
    a[250, 7] = -1.5
    a = sps.csr_matrix(a)
    with pytest.raises(sp.SprsPanic, match="^Matrix is not symmetric$"):
        run(sp, a, "CSR")
    assert not sp.is_symmetric(mirror(sp, as_storage(a, "CSR"), "CSR"))
    run(sp, a, "CSR", check=False)
    run(sp, a, "CSC", rng.permutation(300), check=False)


def test_is_symmetric(sp):
    rng = np.random.default_rng(9)
    a = as_storage(random_spd(rng, 100, 5), "CSR")
    assert sp.is_symmetric(mirror(sp, a, "CSR"))
    b = a.copy()
    b.data[np.flatnonzero(b.indices != np.repeat(np.arange(100), np.diff(b.indptr)))[0]] += 1.0
    assert not sp.is_symmetric(mirror(sp, b, "CSR"))
    c = a.copy()
    c.data[0] = np.nan  # a diagonal NaN is not equal to itself
    assert not sp.is_symmetric(mirror(sp, c, "CSR"))
    assert not sp.is_symmetric(sp.CsMat.new((2, 3), [0, 1, 2], [0, 1], [1., 1.]))


# ---- 3. update
def test_ldl_update(sp):
    rng = np.random.default_rng(10)
    a = as_storage(random_spd(rng, 400, 6), "CSC")
    perm = rng.permutation(400)
    mat = mirror(sp, a, "CSC")
    num = sp.ldl.LdlNumeric.new_perm(mat, perm)
    fa = LO.Factor(a.indptr, a.indices, perm)
    assert fa.update(a.data) is None
    r = a.copy()
    r.data = rng.random(r.nnz)
    b = as_storage(a + a.multiply(r + r.T), "CSC")  # new values, the same pattern
    assert np.array_equal(b.indices, a.indices) and np.array_equal(b.indptr, a.indptr)
    num.update(mirror(sp, b, "CSC"))
    assert fa.update(b.data) is None
    same(num.l().data, fa.l()[2], "L after update")
    same(num.d(), fa.diag(), "D after update")
    x = rng.standard_normal(400)
    same(num.solve(x), fa.solve(x), "x after update")
    # a changed pattern: refused, nothing computed, the factor stays
    c = a.tolil()
    c[0, 399] = c[399, 0] = 0.5
    c = as_storage(c, "CSC")
    launches = mat.context().launches
    with pytest.raises(sp.SprsPanic, match="pattern differs"):
        num.update(mirror(sp, c, "CSC"))
    assert mat.context().launches - launches <= 1  # the pattern comparison only
    same(num.solve(x), fa.solve(x), "x after a refused update")


def test_ldl_singular_update(sp):
    """A handle factored successfully, then updated with values whose D_k is zero: the update
    raises the reference's SingularMatrix, l, d and solve raise until an update succeeds, and
    the next good update restores a factor identical to the oracle's."""
    n = 9
    good = zero_pivot(n, 4, "cancel")
    good.data[good.indices == np.repeat(np.arange(n), np.diff(good.indptr))] = 2.0  # the Laplacian
    fa = LO.Factor(good.indptr, good.indices)
    assert fa.update(good.data) is None
    num = sp.ldl.LdlNumeric.new(mirror(sp, good, "CSR"))
    assert num.singular() is None
    x = np.arange(1.0, n + 1)
    for k, how in ((4, "cancel"), (0, "-0.0"), (n - 1, "0.0")):
        bad = zero_pivot(n, k, how)
        assert np.array_equal(bad.indices, good.indices) and np.array_equal(bad.indptr, good.indptr)
        with pytest.raises(sp.SingularMatrix) as e:
            num.update(mirror(sp, bad, "CSR"))
        assert (e.value.index, e.value.reason) == (k, NUMERIC)
        assert (num.singular().index, num.singular().reason) == (k, NUMERIC)
        for call in (num.l, num.d, lambda: num.solve(x), lambda: num.solve_dev(0, 0)):
            with pytest.raises(sp.SingularMatrix) as e:
                call()
            assert e.value.index == k
        num.update(mirror(sp, good, "CSR"))
        assert num.singular() is None
        same(num.l().data, fa.l()[2], "L after recovery")
        same(num.d(), fa.diag(), "D after recovery")
        same(num.solve(x), fa.solve(x), "x after recovery")


def test_ldl_solve_dev_back_to_back(sp):
    import torch
    from sprs_b200 import generate as G
    rng = np.random.default_rng(11)
    n = 5000
    a = as_storage(laplacian((50, 100)), "CSR")
    perm = nested_dissection((50, 100))
    mat = mirror(sp, a, "CSR")
    num = sp.ldl.LdlNumeric.new_perm(mat, perm)
    fa = LO.Factor(a.indptr, a.indices, perm)
    assert fa.update(a.data) is None
    ctx = mat.context()
    bs = [rng.standard_normal(n) for _ in range(3)]
    db = [torch.from_numpy(b.copy()).to(G._device(ctx)) for b in bs]
    dx = [torch.empty_like(b) for b in db]
    for b, x in zip(db, dx):
        num.solve_dev(b.data_ptr(), x.data_ptr())
    num.solve_dev(db[2].data_ptr(), db[2].data_ptr())  # in place
    G._sync()
    for b, x in zip(bs, dx):
        same(x.cpu().numpy(), fa.solve(b), "solve_dev")
    same(db[2].cpu().numpy(), fa.solve(bs[2]), "solve_dev in place")


def test_ldl_tiny(sp):
    """n = 0 and 1: the C entry points work; the mirror panics in `factor` as the reference's
    DStack::with_capacity(n) does."""
    import ctypes as C
    for n in (0, 1):
        mat = sp.CsMat.new_csc((n, n), np.arange(n + 1), np.arange(n), np.full(n, 4.0))
        with pytest.raises(sp.SprsPanic, match="n > 1"):
            sp.ldl.LdlNumeric.new(mat)
        dev = mat.device()
        ctx, lib = dev.ctx, dev.ctx.lib
        sym, num = C.c_void_p(), C.c_void_p()
        ctx.check(lib.sprs_b200_ldl_symbolic(ctx.h, dev.h, None, 1, C.byref(sym)))
        assert lib.sprs_b200_ldl_nnz(sym) == 0
        ctx.check(lib.sprs_b200_ldl_factor(sym, dev.h, C.byref(num)))
        b = np.full(max(n, 1), 2.0)
        x = np.zeros(max(n, 1))
        ctx.check(lib.sprs_b200_ldl_solve(num, b.ctypes.data_as(C.c_void_p),
                                          x.ctypes.data_as(C.c_void_p), n))
        if n:
            assert x[0] == 0.5
        lib.sprs_b200_ldl_free(num)
        lib.sprs_b200_ldl_free(sym)


# ---- 4. the panics, in the reference's order
def test_ldl_panics(sp):
    ldl = sp.ldl
    rect = sp.CsMat.new((2, 3), [0, 1, 2], [0, 1], [1., 1.])
    with pytest.raises(sp.SprsPanic, match="^matrix should be square$"):
        ldl.LdlNumeric.new_perm(rect, [0, 1], ldl.SymmetryCheck.CheckSymmetry)
    with pytest.raises(sp.SprsPanic, match="left == right"):
        ldl.LdlNumeric.new(rect)
    nonsym = sp.CsMat.new((3, 3), [0, 2, 3, 4], [0, 1, 1, 2], [1., 5., 1., 1.])
    for bad in ([0, 1, 1], [0, 1, 3], [0, 1]):  # not symmetric comes before a bad permutation
        with pytest.raises(sp.SprsPanic, match="^Matrix is not symmetric$"):
            ldl.LdlNumeric.new_perm(nonsym, bad, ldl.SymmetryCheck.CheckSymmetry)
        with pytest.raises(sp.SprsPanic, match="perm_is_valid"):
            ldl.LdlNumeric.new_perm(nonsym, bad, ldl.SymmetryCheck.DontCheckSymmetry)
    sq = sp.CsMat.new((3, 3), [0, 1, 2, 3], [0, 1, 2], [1., 2., 4.])
    num = ldl.LdlNumeric.new(sq)
    with pytest.raises(sp.SprsPanic):
        num.solve(np.zeros(2))
    assert num.solve(np.ones(3)).tolist() == [1.0, 0.5, 0.25]


# ---- 5. 64-bit indptr (child process: SPRS_B200_FORCE_INDPTR64 is read once per process)
_WIDTH_CHILD = r"""
import json, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np
import test_gpu_ldl as T
import sprs_b200 as sp
rng = np.random.default_rng(12)
errs = []
for storage in ("CSR", "CSC"):
    for perm in (None, rng.permutation(500)):
        try:
            T.run(sp, T.random_spd(rng, 500, 8), storage, perm, idx=np.uint64)
        except AssertionError as e:
            errs.append(str(e))
print(json.dumps(errs))
"""


def test_ldl_indptr64_child_process(tmp_path):
    script = tmp_path / "child.py"
    script.write_text(_WIDTH_CHILD % {"root": ROOT, "tests": os.path.join(ROOT, "tests")})
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []


# ---- 6. the C++ host mirror
def test_cpp_ldl_kats(tmp_path):
    exe = str(tmp_path / "test_ldl_kats")
    lib_dir = os.path.join(ROOT, "sprs_b200")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_ldl_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK ")
