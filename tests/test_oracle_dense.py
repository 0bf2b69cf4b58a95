"""The CPU oracle of the dense boundary (tests/dense_oracle.cpp) pinned to the reference's known
answers (tests/golden/dense_fixtures.json) and to a numpy model of its formulas.  No GPU."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

import dense_oracle as DO
from conftest import ROOT


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "dense_fixtures.json")) as f:
        return json.load(f)


def mat(m):
    return SimpleNamespace(storage=m["storage"], shape=tuple(m["shape"]),
                           indptr=np.array(m["indptr"]), indices=np.array(m["indices"]),
                           data=np.array(m["data"], np.float64))


def arrays_of(ip, ind, d, storage, shape):
    return SimpleNamespace(storage=storage, shape=shape, indptr=ip, indices=ind, data=d)


def test_oracle_kats(kats):
    eye = np.array(kats["eye3_dense"])
    for key in ("eye3_csr", "eye3_csc"):
        assert np.array_equal(DO.to_dense(mat(kats[key])), eye)
    assert np.array_equal(DO.to_dense(mat(kats["mat1"])), kats["to_dense_mat1"])
    assert np.array_equal(DO.to_dense(mat(kats["mat3"])), kats["to_dense_mat3"])
    fd = np.array(kats["from_dense_in"])
    for fn, key in ((DO.csr_from_dense, "csr_from_dense_out"), (DO.csc_from_dense, "csc_from_dense_out")):
        ip, ind, d = fn(fd, kats["from_dense_eps"])
        want = kats[key]
        assert ip.tolist() == want["indptr"] and ind.tolist() == want["indices"]
        assert d.tolist() == want["data"]
    out = np.zeros((5, 5))
    DO.binop_dense(mat(kats["mat1"]), DO.ADD, 1.0, 1.0, np.array(kats["mat_dense1"]), out)
    assert np.array_equal(out, kats["add_dense_out"])
    out = np.zeros((3, 3))
    DO.binop_dense(mat(kats["eye3_csr"]), DO.MUL, 1.0, 0.0, np.ones((6, 6))[::2, ::2], out)
    assert np.array_equal(out, eye)


def _model(storage, shape, rng):
    rows, cols = shape
    d = rng.standard_normal(shape)
    d[rng.random(shape) < 0.6] = 0.0
    specials = [np.inf, -np.inf, np.nan, -0.0, 5e-324, 0.5]
    m = rng.random(shape) < 0.1
    d[m] = rng.choice(specials, int(m.sum()))
    return d


@pytest.mark.parametrize("storage", ["CSR", "CSC"])
@pytest.mark.parametrize("eps", [0.0, -1.0, np.nan, 0.5, np.inf])
def test_oracle_matches_numpy(storage, eps):
    rng = np.random.default_rng(3)
    d = _model(storage, (13, 17), rng)
    view = d[::-1] if storage == "CSR" else np.asfortranarray(d)
    fn = DO.csr_from_dense if storage == "CSR" else DO.csc_from_dense
    ip, ind, data = fn(view, eps)
    e = eps if eps > 0 else 0.0
    keep = np.abs(view) > e
    if storage == "CSC":  # column-major walk: the transpose's row-major walk
        keep_o, vals = keep.T, view.T
    else:
        keep_o, vals = keep, view
    assert ip.tolist() == [0] + np.cumsum(keep_o.sum(axis=1)).tolist()
    assert ind.tolist() == np.nonzero(keep_o)[1].tolist()
    assert DO.same_bits(data, vals[keep_o])
    a = arrays_of(ip, ind, data, storage, view.shape)
    # to_dense: the kept values at their places, +0.0 elsewhere
    assert DO.same_bits(DO.to_dense(a), np.where(keep, view, 0.0))
    sentinel = np.full(view.shape, 7.0)
    DO.assign_to_dense(sentinel, a)
    assert DO.same_bits(sentinel, np.where(keep, view, 7.0))
    # the closures: x = +0.0 where A has no entry, every operation rounded on its own
    x = np.where(keep, view, 0.0)
    y = rng.standard_normal(view.shape)
    y[0, :4] = [-0.0, np.inf, np.nan, -3.0]
    y = np.asarray(y, order="C" if storage == "CSR" else "F")
    for alpha, beta in ((1.0, 1.0), (-0.5, 2.0), (np.nan, 1.0), (0.0, -0.0)):
        out = np.zeros(view.shape, order="C" if storage == "CSR" else "F")
        DO.binop_dense(a, DO.ADD, alpha, beta, y, out)
        with np.errstate(invalid="ignore"):
            assert DO.same_values(out, (alpha * x) + (beta * y))
        DO.binop_dense(a, DO.MUL, alpha, 0.0, y, out)
        with np.errstate(invalid="ignore"):
            assert DO.same_values(out, (alpha * x) * y)
    # -0.0 of D at a missing position becomes +0.0 with alpha = beta = 1
    z = arrays_of(np.zeros(view.shape[0 if storage == "CSR" else 1] + 1, np.uint64),
                  np.zeros(0, np.uint64), np.zeros(0), storage, view.shape)
    out = np.zeros(view.shape, order="C" if storage == "CSR" else "F")
    DO.binop_dense(z, DO.ADD, 1.0, 1.0, np.asarray(np.full(view.shape, -0.0), order=out.flags.c_contiguous and "C" or "F"), out)
    assert (out.view(np.uint64) == 0).all()
