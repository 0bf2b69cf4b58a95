"""CPU tests of the binop oracle (tests/binop_oracle.cpp): the restatement of
csmat_binop_same_storage_raw (binop.rs:229-271) and CsMatBase::map that the device results are
compared with.  Pinned to the reference's own KATs (tests/golden/binop_fixtures.json) at every
index width, and to two independent models on random matrices: a dense restatement of the
literal formula (every value class: explicit zeros, exact cancellations, -0.0, +-inf, NaN) and
scipy (finite values; its sparse +, - and .multiply also drop exact zeros)."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sps

import binop_oracle as BO
from conftest import ROOT

WIDTHS = [(np.uint32, np.uint32), (np.uint64, np.uint64), (np.uint32, np.uint64)]
OPS = {BO.ADD: lambda a, b: a + b, BO.SUB: lambda a, b: a - b, BO.MUL: lambda a, b: a * b}


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "sprs_fixtures.json")) as f:
        base = json.load(f)
    with open(os.path.join(ROOT, "tests", "golden", "binop_fixtures.json")) as f:
        return dict(base, **json.load(f))


def arrays(m, idx, ptr):
    return (np.array(m["indptr"], dtype=ptr), np.array(m["indices"], dtype=idx),
            np.array(m["data"], dtype=np.float64))


def assert_same(got, want):
    """structure exact, values bit for bit, NaN by class (position, not payload or sign)"""
    gi, gj, gd = got
    wi, wj, wd = want
    assert np.array_equal(np.asarray(gi, np.int64), np.asarray(wi, np.int64))
    assert np.array_equal(np.asarray(gj, np.int64), np.asarray(wj, np.int64))
    gd, wd = np.asarray(gd, np.float64), np.asarray(wd, np.float64)
    assert np.array_equal(np.isnan(gd), np.isnan(wd))
    ok = ~np.isnan(wd)
    assert np.array_equal(gd[ok].view(np.uint64), wd[ok].view(np.uint64))


@pytest.mark.parametrize("idx,ptr", WIDTHS)
@pytest.mark.parametrize("op,key", [(BO.ADD, "mat1_plus_mat2"), (BO.SUB, "mat1_minus_mat2"),
                                    (BO.MUL, "mat1_times_mat2")])
def test_oracle_binop_kats(kats, idx, ptr, op, key):
    got = BO.binop(op, arrays(kats["mat1"], idx, ptr), arrays(kats["mat2"], idx, ptr))
    assert_same(got, arrays(kats[key], idx, ptr))
    assert got[0].dtype == ptr and got[1].dtype == idx


@pytest.mark.parametrize("idx,ptr", WIDTHS)
def test_oracle_add_differing_patterns_and_scale(kats, idx, ptr):
    got = BO.binop(BO.ADD, arrays(kats["add1_lhs"], idx, ptr), arrays(kats["add1_rhs"], idx, ptr))
    assert_same(got, arrays(kats["add1_sum"], idx, ptr))
    assert_same(BO.scale(arrays(kats["mat1"], idx, ptr), 2.0), arrays(kats["mat1_times_2"], idx, ptr))


def dense_model(op, shape, a, b):
    """The literal formula on every position of the union of the two patterns (CSR)."""
    f = OPS[op]
    rows, cols = shape
    da, db = np.zeros(shape), np.zeros(shape)
    ha, hb = np.zeros(shape, bool), np.zeros(shape, bool)
    for (ip, ind, d), dense, has in ((a, da, ha), (b, db, hb)):
        for r in range(rows):
            for k in range(int(ip[r]), int(ip[r + 1])):
                dense[r, ind[k]] = d[k]
                has[r, ind[k]] = True
    with np.errstate(all="ignore"):
        v = f(da, db)
    keep = (ha | hb) & (v != 0.0)
    indptr = np.concatenate([[0], np.cumsum(keep.sum(axis=1))])
    rr, cc = np.nonzero(keep)
    return indptr, cc, v[rr, cc]


def random_pair(rng, rows, cols, specials):
    def one(lens):
        ip = np.zeros(rows + 1, np.int64)
        np.cumsum(lens, out=ip[1:])
        ind = np.concatenate([np.sort(rng.choice(cols, n, replace=False)) for n in lens] +
                             [np.zeros(0, np.int64)])
        d = rng.integers(-3, 4, ip[-1]).astype(np.float64) * 0.5
        if specials and d.size:
            k = rng.integers(0, d.size, max(1, d.size // 6))
            d[k] = rng.choice([0.0, -0.0, np.inf, -np.inf, np.nan, 1e308, -1e308], k.size)
        return ip, ind, d
    la = np.minimum(rng.choice([0, 0, 1, 2, 3, 7, cols], rows), cols)
    a = one(la)
    if rng.random() < 0.5:  # the same pattern: Both everywhere, exact cancellations under SUB
        b = (a[0].copy(), a[1].copy(), a[2].copy() if rng.random() < 0.5 else -a[2])
    else:
        b = one(np.minimum(rng.choice([0, 0, 1, 2, 3, 7, cols], rows), cols))
    return a, b


@pytest.mark.parametrize("seed", range(40))
def test_oracle_binop_dense_model(seed):
    rng = np.random.default_rng(seed)
    rows, cols = int(rng.integers(0, 12)), int(rng.integers(1, 12))
    a, b = random_pair(rng, rows, cols, specials=True)
    for op in OPS:
        want = dense_model(op, (rows, cols), a, b)
        for idx, ptr in WIDTHS:
            got = BO.binop(op, (a[0].astype(ptr), a[1].astype(idx), a[2]),
                           (b[0].astype(ptr), b[1].astype(idx), b[2]))
            assert_same(got, want)


@pytest.mark.parametrize("seed", range(10))
def test_oracle_binop_scipy(seed):
    rng = np.random.default_rng(100 + seed)
    rows, cols = int(rng.integers(1, 200)), int(rng.integers(1, 200))
    a, b = random_pair(rng, rows, cols, specials=False)
    sa = sps.csr_matrix((a[2], a[1], a[0]), shape=(rows, cols))
    sb = sps.csr_matrix((b[2], b[1], b[0]), shape=(rows, cols))
    for op, s in ((BO.ADD, sa + sb), (BO.SUB, sa - sb), (BO.MUL, sa.multiply(sb).tocsr())):
        s.sort_indices()
        got = BO.binop(op, (a[0].astype(np.uint32), a[1].astype(np.uint32), a[2]),
                       (b[0].astype(np.uint32), b[1].astype(np.uint32), b[2]))
        assert_same(got, (s.indptr, s.indices, s.data))


def test_oracle_value_classes():
    """The literal formula's edge cases: MUL Left(+-inf / NaN) -> a * 0.0 = NaN, kept; SUB
    Right(b) -> -b; ADD Left(-0.0) -> +0.0, dropped; explicit zeros disappear; A - A empty."""
    u = np.uint32
    a = (np.array([0, 4], u), np.array([0, 1, 2, 3], u), np.array([np.inf, np.nan, -0.0, 0.0]))
    b = (np.array([0, 2], u), np.array([4, 5], u), np.array([2.0, -0.0]))
    ip, ind, d = BO.binop(BO.MUL, a, b)  # Right(b): 0.0 * b = +-0.0, dropped
    assert ind.tolist() == [0, 1] and np.isnan(d).all()
    ip, ind, d = BO.binop(BO.SUB, a, b)
    assert ind.tolist() == [0, 1, 4] and d[0] == np.inf and np.isnan(d[1]) and d[2] == -2.0
    ip, ind, d = BO.binop(BO.ADD, a, b)
    assert ind.tolist() == [0, 1, 4]
    ip, ind, d = BO.binop(BO.SUB, a, a)
    assert ip.tolist() == [0, 2] and ind.tolist() == [0, 1] and np.isnan(d).all()  # inf - inf
    c = (np.array([0, 2, 2, 3], u), np.array([1, 3, 0], u), np.array([1.5, -2.0, 4.0]))
    ip, ind, d = BO.binop(BO.SUB, c, c)
    assert ip.tolist() == [0, 0, 0, 0] and ind.size == 0
    sip, sind, sd = BO.scale(c, 0.0)  # map keeps zeros
    assert sind.tolist() == [1, 3, 0] and (sd == 0.0).all() and np.signbit(sd).tolist() == [False, True, False]


@pytest.mark.parametrize("rows", [0, 1, 5])
def test_oracle_empty(rows):
    for idx, ptr in WIDTHS:
        e = (np.zeros(rows + 1, ptr), np.zeros(0, idx), np.zeros(0))
        for op in OPS:
            ip, ind, d = BO.binop(op, e, e)
            assert ip.tolist() == [0] * (rows + 1) and ind.size == 0 and d.size == 0
