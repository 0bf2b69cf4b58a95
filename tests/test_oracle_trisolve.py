"""CPU-only: the trisolve oracle (tests/trisolve_oracle.cpp) reproduces the reference's KATs,
agrees with scipy's triangular solve to rounding, and leaves the reference's partial state
after a singular index."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sps
from scipy.sparse.linalg import spsolve_triangular

import trisolve_oracle as TO
from conftest import ROOT, rand_csr

ZERO, NUMERIC, STRUCTURAL = TO.REASONS


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "trisolve_fixtures.json")) as f:
        return json.load(f)


def test_oracle_reproduces_kats(kats):
    assert sorted(kats) == sorted(TO.FORMS)
    for form, k in kats.items():
        x = np.array(k["b"], np.float64)
        assert TO.solve(form, k["indptr"], k["indices"], k["data"], x) is None
        assert x.tolist() == k["x"], form


def _scipy(form, ip, ind, dat, n, b):
    cls = sps.csr_matrix if form.endswith("csr") else sps.csc_matrix
    m = cls((dat, ind, ip), shape=(n, n))
    lower = form.startswith("l")
    t = sps.tril(m) if lower else sps.triu(m)
    return spsolve_triangular(sps.csr_matrix(t), b, lower=lower)


@pytest.mark.parametrize("form", TO.FORMS)
def test_oracle_agrees_with_scipy(form):
    rng = np.random.default_rng(11)
    n = 300
    ip, ind, dat = rand_csr(rng, n, n, 6)
    # a full diagonal that dominates its row, with entries of the ignored triangle kept
    dense = sps.csr_matrix((dat, ind, ip), shape=(n, n)).toarray()
    dense[np.arange(n), np.arange(n)] = 1.0 + np.abs(dense).sum(axis=1)
    m = sps.csr_matrix(dense) if form.endswith("csr") else sps.csc_matrix(dense)
    m.sort_indices()
    b = rng.standard_normal(n)
    x = b.copy()
    assert TO.solve(form, m.indptr, m.indices, m.data, x) is None
    want = _scipy(form, m.indptr, m.indices, m.data, n, b)
    assert np.allclose(x, want, rtol=1e-12, atol=1e-14)


def test_oracle_partial_state_after_singular():
    # L = [[2,0,0],[1,.,0],[4,3,1]]: the diagonal of row / column 1 is missing
    lo = sps.csr_matrix(np.array([[2., 0, 0], [1, 0, 0], [4, 3, 1]]))
    x = np.array([4., 5, 7])
    assert TO.solve("lsolve_csr", lo.indptr, lo.indices, lo.data, x) == (1, ZERO)
    assert x.tolist() == [2., 5, 7]             # row 0 solved, rows 1.. untouched
    lc = lo.tocsc()
    x = np.array([4., 5, 7])
    assert TO.solve("lsolve_csc", lc.indptr, lc.indices, lc.data, x) == (1, STRUCTURAL)
    assert x.tolist() == [2., 5 - 1 * 2, 7 - 4 * 2]  # column 0 applied, nothing divided
    # U = [[1,2,3],[0,-0.0,4],[0,0,2]]: a stored -0.0 on the diagonal of row / column 1
    up = sps.csr_matrix((np.array([1., 2, 3, -0.0, 4, 2]), [0, 1, 2, 1, 2, 2], [0, 3, 5, 6]),
                        shape=(3, 3))
    x = np.array([1., 2, 4])
    assert TO.solve("usolve_csr", up.indptr, up.indices, up.data, x) == (1, NUMERIC)
    assert x.tolist() == [1., 2, 2]
    uc = up.tocsc()
    uc.sort_indices()
    x = np.array([1., 2, 4])
    assert TO.solve("usolve_csc", uc.indptr, uc.indices, uc.data, x) == (1, NUMERIC)
    assert x.tolist() == [1 - 3 * 2., 2 - 4 * 2., 2]
    # a NaN diagonal is not singular
    x = np.array([1.])
    assert TO.solve("lsolve_csr", [0, 1], [0], [np.nan], x) is None and np.isnan(x[0])
    # n = 0 is Ok
    assert TO.solve("usolve_csc", [0], [], [], np.zeros(0)) is None


def test_oracle_usolve_csc_subtracts_in_descending_column_order():
    """usolve_csc sums row r from the end; usolve_csr on the same matrix from the start.  Row 0
    of [[1, 1, 1], ...] with x = (., 1, 2^-54) gives different bits in the two orders."""
    u = sps.csr_matrix(np.array([[1., 1., 1.], [0, 1, 0], [0, 0, 1]]))
    b = np.array([1.0, 1.0, 2.0 ** -54])
    xr, xc = b.copy(), b.copy()
    assert TO.solve("usolve_csr", u.indptr, u.indices, u.data, xr) is None
    uc = u.tocsc()
    assert TO.solve("usolve_csc", uc.indptr, uc.indices, uc.data, xc) is None
    # csr: (1 - 1) - 2^-54 = -2^-54;  csc: (1 - 2^-54) - 1 = 1 - 1 = 0 (1 - 2^-54 rounds to 1)
    assert xr[0] == -2.0 ** -54
    assert xc[0] == 0.0
    assert xr[0] != xc[0]


def test_levels():
    n = 6
    chain = sps.csr_matrix(np.eye(n) + np.eye(n, k=-1))
    assert TO.levels(chain.indptr, chain.indices, upper=False) == n
    assert TO.levels(chain.indptr, chain.indices, upper=True) == 1
    c = chain.tocsc()
    assert TO.levels(c.indptr, c.indices, upper=False, csr=False) == n
    eye = sps.csr_matrix(np.eye(n))
    assert TO.levels(eye.indptr, eye.indices, upper=False) == 1
    assert TO.levels([0], [], upper=False) == 0
