"""The CPU restatement of the sprs-ldl crate (tests/ldl_oracle.cpp) against the reference's own
known answers (tests/golden/ldl_fixtures.json), bit for bit, and against scipy on random
inputs within rounding.  No GPU."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sps

import ldl_oracle as LO

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "ldl_fixtures.json")))


def f(v):
    return np.array([float(s) for s in v])


def bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def test_factor1():
    k = KATS["test_mat1"]
    fa = LO.Factor(k["indptr"], k["indices"])
    assert fa.update(f(k["data"])) is None
    cp, li, lv = fa.l()
    assert cp.tolist() == k["l_colptr"]
    assert li.tolist() == k["l_indices"]
    assert np.array_equal(bits(lv), bits(f(k["l_data"])))
    assert np.array_equal(bits(fa.diag()), bits(f(k["d"])))


def test_solve1():
    k = KATS["test_mat1"]
    x = f(k["b"])
    LO.lsolve(k["l_colptr"], k["l_indices"], f(k["l_data"]), x)
    assert np.array_equal(bits(x), bits(f(k["lsolve"])))
    LO.diag_solve(f(k["d"]), x)
    assert np.array_equal(bits(x), bits(f(k["dsolve"])))
    LO.ltsolve(k["l_colptr"], k["l_indices"], f(k["l_data"]), x)
    assert np.array_equal(bits(x), bits(f(k["x"])))


def test_factor_solve1():
    k = KATS["test_mat1"]
    fa = LO.Factor(k["indptr"], k["indices"])
    assert fa.update(f(k["data"])) is None
    assert np.array_equal(bits(fa.solve(f(k["b"]))), bits(f(k["x"])))


def test_permuted_ldl_solve():
    k = KATS["permuted_ldl_solve"]
    fa = LO.Factor(k["indptr"], k["indices"], k["perm"])
    assert fa.update(f(k["data"])) is None
    assert np.array_equal(fa.solve(f(k["b"])), f(k["x"]))


def random_spd(rng, n, density):
    m = sps.random(n, n, density=density, random_state=rng, data_rvs=rng.standard_normal)
    a = (m + m.T).tocsr()
    a = a + sps.diags(1.0 + np.asarray(abs(a).sum(axis=1)).ravel())
    a = sps.csr_matrix(a)
    a.sort_indices()
    return a


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_against_scipy(seed):
    rng = np.random.default_rng(seed)
    n = 60
    a = random_spd(rng, n, 0.08)
    perm = rng.permutation(n)
    fa = LO.Factor(a.indptr, a.indices, perm)
    assert fa.update(a.data) is None
    cp, li, lv = fa.l()
    lo = sps.csc_matrix((lv, li.astype(np.int64), cp.astype(np.int64)), shape=(n, n)).toarray()
    lo += np.eye(n)
    pm = np.eye(n)[perm]
    pap = pm @ a.toarray() @ pm.T
    assert np.allclose(lo @ np.diag(fa.diag()) @ lo.T, pap, rtol=1e-12, atol=1e-12)
    b = rng.standard_normal(n)
    assert np.allclose(fa.solve(b), np.linalg.solve(a.toarray(), b), rtol=1e-9, atol=1e-12)
    assert 1 <= fa.etree_height() <= n


def test_pattern_order_is_reverse_entry_order():
    """Row 3 of an arrow-like pattern reads columns 0, 1, 2 (three separate paths, no tree
    edges between them): the reference processes the paths in reverse stored order, so D_3 is
    reduced by the terms of columns 2, 1, 0 in that order.  Chosen so that the two orders round
    differently."""
    n = 4
    a = np.diag([1.0, 3.0, 7.0, 1.0])
    a[3, :3] = a[:3, 3] = [1.0, 1.0 / 3.0, 0.1]
    m = sps.csc_matrix(a)
    fa = LO.Factor(m.indptr, m.indices)
    assert fa.update(m.data) is None
    d3 = 1.0
    for i in (2, 1, 0):
        y = a[3, i]
        d3 = d3 - (y / a[i, i]) * y
    assert bits(fa.diag())[3] == bits([d3])[0]


def test_singular_early_return():
    a = sps.csc_matrix(np.array([[1.0, 1.0, 0.0], [1.0, 1.0, 0.0], [0.0, 0.0, 2.0]]))
    fa = LO.Factor(a.indptr, a.indices)
    assert fa.update(a.data) == 1
    # the workspaces stay consistent: another update of the same pattern succeeds
    a2 = sps.csc_matrix(np.array([[2.0, 1.0, 0.0], [1.0, 2.0, 0.0], [0.0, 0.0, 2.0]]))
    assert fa.update(a2.data) is None
    assert np.array_equal(fa.diag(), [2.0, 1.5, 2.0])


def test_negative_zero_input_becomes_positive():
    a = sps.csc_matrix(([-0.0, 1.0, 1.0], [0, 1, 1], [0, 1, 2, 3]), shape=(3, 3))
    fa = LO.Factor(a.indptr, a.indices)
    assert fa.update(a.data) == 0
    assert bits(fa.diag())[0] == bits([0.0])[0]
