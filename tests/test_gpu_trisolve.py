"""Sparse triangular solves on the device (csrc/trisolve.cu) against the CPU restatement of
sprs::linalg::trisolve (tests/trisolve_oracle.cpp): every form, whole vectors, bit for bit on
view(np.uint64) (NaN by class), the SingularMatrix index and reason, and the partial rhs the
reference leaves behind.

Small tests run on the emulator as well (tests/test_emu_trisolve.py runs them on the emulated
build that has the solves, tests/emu_trisolve.py); `*_full_size`, `*_child_process`, `*_large`
and `test_cpp*` ones need the H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import trisolve_oracle as TO
from conftest import ROOT

pytestmark = pytest.mark.gpu

if os.environ.get("SPRS_B200_EMU_TRISOLVE_LIB"):  # test infrastructure: the emulated build with
    import sprs_b200 as _sp                       # the solves (tests/emu_trisolve.py)
    _sp._lib.LIB_PATH = os.environ["SPRS_B200_EMU_TRISOLVE_LIB"]

ZERO, NUMERIC, STRUCTURAL = TO.REASONS


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    lib = sprs_b200._lib.load()  # the product library must export the solves (AttributeError)
    if os.path.basename(sprs_b200._lib.LIB_PATH).startswith("libsprs_b200_emu") and \
            not hasattr(lib, "sprs_b200_trisolve_plan"):
        pytest.skip("the emulated build of tests/emu has no trisolve: tests/test_emu_trisolve.py "
                    "runs this file on one that has")
    return sprs_b200


def storage_of(form):
    return "CSR" if form.endswith("csr") else "CSC"


def as_storage(m, form):
    """scipy matrix m in the form's storage, indices sorted"""
    m = sps.csr_matrix(m) if form.endswith("csr") else sps.csc_matrix(m)
    m.sort_indices()
    return m


def run(sp, form, m, b, idx=np.uint32):
    """The device solve through the Python mirror and the oracle on the same input: the same
    SingularMatrix (or none) and the same x, bit for bit.  Returns x."""
    m = as_storage(m, form)
    n = m.shape[0]
    cls = sp.CsMat.new if form.endswith("csr") else sp.CsMat.new_csc
    mat = cls((n, n), m.indptr.astype(idx), m.indices.astype(idx), m.data)
    x = np.array(b, dtype=np.float64)
    got_err = None
    try:
        getattr(sp.linalg.trisolve, form + "_dense_rhs")(mat, x)
    except sp.SingularMatrix as e:
        got_err = (e.index, e.reason)
        assert str(e) == "Singular matrix at index %d (%s)" % got_err
    want = np.array(b, dtype=np.float64)
    want_err = TO.solve(form, m.indptr, m.indices, m.data, want)
    assert got_err == want_err, (form, got_err, want_err)
    d = TO.first_difference(x, want)
    assert d is None, "%s: %s" % (form, d)
    return x


def dominant(rng, n, nnz_per_row, scale=False, lower=None):
    """Random n x n with N(0,1) entries in both triangles (lower=None) or one, and a diagonal
    1 + sum |row|.  scale: each value times 2^k, k uniform in [-20, 20]."""
    m = sps.random(n, n, density=min(1.0, nnz_per_row / n), format="csr", random_state=rng,
                   data_rvs=rng.standard_normal)
    if scale:
        m.data *= np.exp2(rng.integers(-20, 21, m.nnz))
    if lower is not None:
        m = sps.tril(m, -1) if lower else sps.triu(m, 1)
    m = sps.csr_matrix(m)
    m.setdiag(0.0)
    m.eliminate_zeros()
    d = 1.0 + np.asarray(abs(m).sum(axis=1)).ravel()
    return sps.csr_matrix(m + sps.diags(d))


# ---- 1. the reference's KATs through the Python mirror
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_trisolve_kats(sp, idx):
    with open(os.path.join(ROOT, "tests", "golden", "trisolve_fixtures.json")) as f:
        kats = json.load(f)
    for form, k in kats.items():
        cls = sp.CsMat.new if k["storage"] == "CSR" else sp.CsMat.new_csc
        mat = cls(tuple(k["shape"]), np.array(k["indptr"], idx), np.array(k["indices"], idx),
                  np.array(k["data"], np.float64))
        x = np.array(k["b"], np.float64)
        getattr(sp.linalg.trisolve, form + "_dense_rhs")(mat, x)
        assert x.tolist() == k["x"], form


# ---- 2. values: N(0,1), 2^+-20 scaling, non-triangular inputs, NaN / Inf
@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_random_values(sp, form):
    rng = np.random.default_rng(1)
    for n, per_row, scale in ((700, 9, False), (1500, 20, True)):
        m = dominant(rng, n, per_row, scale)        # both triangles populated
        run(sp, form, m, rng.standard_normal(n))
        tri = dominant(rng, n, per_row, scale, lower=form.startswith("l"))
        run(sp, form, tri, rng.standard_normal(n) * np.exp2(rng.integers(-20, 21, n)))


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_nan_inf(sp, form):
    rng = np.random.default_rng(2)
    n = 400
    m = sps.csr_matrix(dominant(rng, n, 8))
    k = rng.choice(m.nnz, 12, replace=False)
    m.data[k[:4]] = np.nan
    m.data[k[4:8]] = np.inf
    m.data[k[8:]] = -np.inf
    b = rng.standard_normal(n)
    b[rng.choice(n, 6, replace=False)] = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e308]
    x = run(sp, form, m, b)
    assert np.isnan(x).any()
    # a NaN diagonal is not singular
    m = sps.csr_matrix(dominant(rng, n, 8))
    m[n // 2, n // 2] = np.nan
    run(sp, form, m, rng.standard_normal(n))


# ---- 3. singular matrices: the index, the reason and the partial rhs
@pytest.mark.parametrize("form", TO.FORMS)
@pytest.mark.parametrize("kind", ["missing", "zero", "negzero"])
def test_trisolve_singular(sp, form, kind):
    rng = np.random.default_rng(3)
    n = 300
    base = dominant(rng, n, 10)
    for k in (0, n - 1, n // 2 + 7):
        m = sps.lil_matrix(base)
        if kind == "missing":
            m[k, k] = 0.0
            m = sps.csr_matrix(m)
            m.eliminate_zeros()
        else:
            m = sps.csr_matrix(m)
            m.sort_indices()
            j = m.indptr[k] + np.flatnonzero(m.indices[m.indptr[k]:m.indptr[k + 1]] == k)[0]
            m.data[j] = 0.0 if kind == "zero" else -0.0
        b = rng.standard_normal(n)
        want = b.copy()
        err = TO.solve(form, *(lambda s: (s.indptr, s.indices, s.data))(as_storage(m, form)), want)
        reason = {"lsolve_csr": ZERO, "usolve_csr": NUMERIC}.get(
            form, STRUCTURAL if kind == "missing" else NUMERIC)
        assert err == (k, reason)
        run(sp, form, m, b)


# ---- 4. shapes: n = 0, n = 1, long rows, a column every row depends on
@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_small_and_long_rows(sp, form):
    rng = np.random.default_rng(4)
    run(sp, form, sps.csr_matrix((0, 0)), np.zeros(0))
    run(sp, form, sps.csr_matrix(np.array([[3.0]])), [2.0])
    run(sp, form, sps.csr_matrix(np.array([[0.0]])), [2.0])
    run(sp, form, sps.csr_matrix((1, 1)), [2.0])  # nothing stored: singular
    # rows of 33, 1025 and 3000 terms in both triangles
    n = 3200
    m = sps.lil_matrix(dominant(rng, n, 3))
    for r, cnt in ((40, 33), (1500, 1025), (3100, 3000), (100, 2500)):
        cols = rng.choice(n, cnt, replace=False)
        m[r, cols] = rng.standard_normal(cnt)
    m = sps.csr_matrix(m)
    m.setdiag(1.0 + np.asarray(abs(m).sum(axis=1)).ravel())
    run(sp, form, m, rng.standard_normal(n))
    # a column (lower: 0, upper: n-1) on which every row depends
    n = 2000
    m = sps.lil_matrix(dominant(rng, n, 4))
    m[:, 0] = rng.standard_normal((n, 1))
    m[:, n - 1] = rng.standard_normal((n, 1))
    m = sps.csr_matrix(m)
    m.setdiag(2.0 + np.asarray(abs(m).sum(axis=1)).ravel())
    run(sp, form, m, rng.standard_normal(n))


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_chain_and_diagonal_large(sp, form):
    """A bidiagonal chain of 10^5 rows (depth n) and a diagonal of 10^6 rows (depth 1)."""
    rng = np.random.default_rng(5)
    n = 100_000
    off = rng.standard_normal(n - 1) * 0.5
    k = -1 if form.startswith("l") else 1
    m = sps.diags([np.full(n, 1.0) + rng.random(n), off], [0, k], format="csr")
    run(sp, form, m, rng.standard_normal(n))
    n = 1_000_000
    run(sp, form, sps.diags(rng.standard_normal(n) + 3.0, 0, format="csr"), rng.standard_normal(n))


def test_trisolve_usolve_csc_order_differs_from_csr(sp):
    """usolve_csc subtracts the terms of a row in descending column order: on this matrix its
    bits differ from usolve_csr on the same matrix.  A kernel that summed usolve_csc in
    ascending order would return usolve_csr's bits and fail here."""
    u = sps.csr_matrix(np.array([[1., 1., 1.], [0, 1, 0], [0, 0, 1]]))
    b = [1.0, 1.0, 2.0 ** -54]
    xr = run(sp, "usolve_csr", u, b)
    xc = run(sp, "usolve_csc", u, b)
    assert xr[0] == -2.0 ** -54 and xc[0] == 0.0
    # the same on a random matrix with long rows: many rows differ
    rng = np.random.default_rng(6)
    m = dominant(rng, 3000, 60, lower=False)
    b = rng.standard_normal(3000)
    xr, xc = run(sp, "usolve_csr", m, b), run(sp, "usolve_csc", m, b)
    assert np.count_nonzero(xr != xc) > 0


# ---- 5. the plan: repeated device solves, epochs
def test_trisolve_solve_dev_back_to_back(sp):
    import torch
    from sprs_b200 import generate as G
    rng = np.random.default_rng(7)
    n = 5000
    for form in TO.FORMS:
        m = as_storage(dominant(rng, n, 12), form)
        cls = sp.CsMat.new if form.endswith("csr") else sp.CsMat.new_csc
        mat = cls((n, n), m.indptr, m.indices, m.data)
        plan = sp.linalg.TriSolvePlan(mat, lower=form.startswith("l"))
        assert plan.singular() is None
        ctx = mat.context()
        bs = [rng.standard_normal(n) for _ in range(3)]
        xs = [torch.from_numpy(b.copy()).to(G._device(ctx)) for b in bs]
        for x in xs:  # three solves enqueued back to back on one stream, one plan
            assert G.trisolve_dev(ctx, plan, x) is None
        G._sync()
        for b, x in zip(bs, xs):
            want = b.copy()
            assert TO.solve(form, m.indptr, m.indices, m.data, want) is None
            assert TO.first_difference(x.cpu().numpy(), want) is None, form
        # a host solve on the same plan after them
        x = bs[0].copy()
        plan.solve(x)
        assert TO.first_difference(x, xs[0].cpu().numpy()) is None
        plan.free()


def test_trisolve_solve_dev_singular(sp):
    import torch
    from sprs_b200 import generate as G
    m = sps.csr_matrix(np.array([[2., 0, 0], [1, 0, 0], [4, 3, 1]]))
    mat = sp.CsMat.new_csc((3, 3), *(lambda s: (s.indptr, s.indices, s.data))(as_storage(m, "csc")))
    plan = sp.linalg.TriSolvePlan(mat, lower=True)
    assert (plan.singular().index, plan.singular().reason) == (1, STRUCTURAL)
    x = torch.tensor([4., 5, 7], dtype=torch.float64, device=G._device(mat.context()))
    e = G.trisolve_dev(mat.context(), plan, x)
    G._sync()
    assert (e.index, e.reason) == (1, STRUCTURAL)
    assert x.cpu().tolist() == [2., 3, -1]


# ---- 6. the panics, in the reference's order
def test_trisolve_panics(sp):
    ts = sp.linalg.trisolve
    rect = sp.CsMat.new((2, 3), [0, 1, 2], [0, 1], [1., 1.])
    sq = sp.CsMat.new((3, 3), [0, 1, 2, 3], [0, 1, 2], [1., 1., 1.])
    for f in (ts.lsolve_csr_dense_rhs, ts.usolve_csr_dense_rhs, ts.lsolve_csc_dense_rhs,
              ts.usolve_csc_dense_rhs):
        csr = f.__name__.endswith("csr_dense_rhs")
        # square first, even with a wrong rhs length and the wrong storage
        for m in (rect, rect.transpose_view()):
            with pytest.raises(sp.SprsPanic, match="^Non square matrix passed to solver$"):
                f(m, np.zeros(7))
        wrong = sq if not csr else sq.to_other_storage()
        right = sq if csr else sq.to_other_storage()
        with pytest.raises(sp.SprsPanic, match="^Dimension mismatch$"):
            f(wrong, np.zeros(4))  # dimension before storage
        with pytest.raises(sp.SprsPanic, match="^Storage mismatch$"):
            f(wrong, np.zeros(3))
        with pytest.raises(TypeError):
            f(right, np.zeros(3, dtype=np.float32))
        x = np.ones(3)
        f(right, x)
        assert x.tolist() == [1., 1., 1.]
    with pytest.raises(sp.SprsPanic, match="^Non square matrix passed to solver$"):
        sp.linalg.TriSolvePlan(rect)
    plan = sp.linalg.TriSolvePlan(sq)
    with pytest.raises(sp.SprsPanic, match="^Dimension mismatch$"):
        plan.solve(np.zeros(2))


# ---- 7. 64-bit indptr (child process: SPRS_B200_FORCE_INDPTR64 is read once per process)
_WIDTH_CHILD = r"""
import json, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np, scipy.sparse as sps
import test_gpu_trisolve as T
import sprs_b200 as sp
rng = np.random.default_rng(8)
errs = []
for form in T.TO.FORMS:
    for m in (T.dominant(rng, 900, 14), T.dominant(rng, 900, 14, lower=form.startswith("l"))):
        try:
            T.run(sp, form, m, rng.standard_normal(900), idx=np.uint64)
        except AssertionError as e:
            errs.append(str(e))
    m = sps.lil_matrix(T.dominant(rng, 300, 6)); m[150, 150] = 0.0
    try:
        T.run(sp, form, sps.csr_matrix(m), rng.standard_normal(300), idx=np.uint64)
    except AssertionError as e:
        errs.append(str(e))
print(json.dumps(errs))
"""


def test_trisolve_indptr64_child_process(tmp_path):
    script = tmp_path / "child.py"
    script.write_text(_WIDTH_CHILD % {"root": ROOT, "tests": os.path.join(ROOT, "tests")})
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []


# ---- 8. full size (H100): both triangles of configs 2 and 5, whole x against the oracle
def _full(sp, a, lower, seed, csc=False):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    t = G.triangular(ctx, a, lower)
    mirror = t.mirror
    if csc:
        mirror, ip, ind, dat = G._with_views(ctx, t.mirror.to_other_storage())
    else:
        ip, ind, dat = t.indptr, t.indices, t.data
    form = ("lsolve_" if lower else "usolve_") + ("csc" if csc else "csr")
    plan = sp.linalg.TriSolvePlan(mirror, lower)
    b = G.normal_vector(ctx, t.rows, seed=seed)
    want = b.cpu().numpy().copy()
    assert G.trisolve_dev(ctx, plan, b) is None
    G._sync()
    got = b.cpu().numpy()
    plan.free()
    hip = ip.cpu().numpy().view(np.uint32)
    hind = ind.cpu().numpy().view(np.uint32)
    hdat = dat.cpu().numpy()
    assert TO.solve(form, hip, hind, hdat, want) is None
    d = TO.first_difference(got, want)
    assert d is None, "%s: %s" % (form, d)
    assert np.isfinite(got).all()


def test_trisolve_rand1m_full_size(sp):
    from sprs_b200 import generate as G
    a = G.rand_csr(sp.Context.default(), 1_000_000, 1_000_000, 32, seed=0x5EED0002)
    _full(sp, a, True, 0x5EED7001)
    _full(sp, a, False, 0x5EED7002)
    _full(sp, a, True, 0x5EED7003, csc=True)
    _full(sp, a, False, 0x5EED7004, csc=True)


def test_trisolve_rmat10m_full_size(sp):
    from sprs_b200 import generate as G
    a = G.rmat_csr(sp.Context.default(), 10_000_000, 100, seed=0x5EED0005)
    _full(sp, a, True, 0x5EED7005)
    _full(sp, a, False, 0x5EED7006)


# ---- 9. the C++ host mirror
def test_cpp_trisolve_kats(tmp_path):
    exe = str(tmp_path / "test_trisolve_kats")
    lib_dir = os.path.join(ROOT, "sprs_b200")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_trisolve_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK ")
