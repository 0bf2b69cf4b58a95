"""CPU-only: the construction oracle (tests/construct_oracle.cpp + .py) reproduces the
reference's own known answers (tests/golden/construct_fixtures.json) -- vstack_trivial,
hstack_trivial, vstack_with_conversion, bmat_simple, bmat_complex, the panic tests and
test_kronecker_product in its four storage combinations -- and the unequal-width bmat rule of
the reference's composition."""
import json
import os

import numpy as np
import pytest

import construct_oracle as CO
from conftest import ROOT


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "sprs_fixtures.json")) as f:
        base = json.load(f)
    with open(os.path.join(ROOT, "tests", "golden", "construct_fixtures.json")) as f:
        return dict(base, **json.load(f))


def m(k):
    return CO.mat(k["storage"], k["shape"], k["indptr"], k["indices"], k["data"])


def same(got, want):
    err = CO.first_difference(got, want)
    assert err is None, err


def test_oracle_stack_kats(kats):
    a, b = m(kats["mat1"]), m(kats["mat2"])
    want = m(kats["mat1_vstack_mat2"])
    same(CO.vstack([a, b]), want)                                           # vstack_trivial
    same(CO.hstack([CO.transpose_view(a), CO.transpose_view(b)]), CO.transpose_view(want))
    same(CO.vstack([CO.to_other_storage(a), b]), want)                      # with conversion
    same(CO.same_storage_fast_stack([a, b]), want)


def test_oracle_bmat_kats(kats):
    eye = lambda n: CO.mat("CSR", (n, n), np.arange(n + 1), np.arange(n), np.ones(n))  # noqa
    same(CO.bmat([[eye(5), None], [None, eye(4)]]), m(kats["bmat_simple"]))
    a, b, d, e = (m(kats[k]) for k in ("mat1", "mat2", "mat3", "mat4"))
    same(CO.bmat([[a, b], [b, None]]), m(kats["bmat_complex_1"]))
    same(CO.bmat([[d, a], [None, e]]), m(kats["bmat_complex_2"]))


def test_oracle_panics(kats):
    for case in kats["panics"]:
        with pytest.raises(CO.Panic, match=case["message"]):
            if "stack" in case:
                CO.same_storage_fast_stack([m(kats[k]) for k in case["stack"]])
            else:
                CO.bmat([[m(kats[k]) if k else None for k in row] for row in case["blocks"]])
    # same_storage_fast_stack_fail_storage (not reachable through vstack / hstack)
    with pytest.raises(CO.Panic, match="Storage mismatch"):
        CO.same_storage_fast_stack([m(kats["mat1"]), m(kats["mat4"])])


def test_oracle_bmat_unequal_widths():
    """A block's column offset is the sum of the widths to its left in ITS block row; only the
    block rows' total widths must agree (the vstack)."""
    rng = np.random.default_rng(3)

    def dense(r, c):
        x = rng.integers(1, 9, (r, c)).astype(float) * (rng.random((r, c)) < 0.6)
        ip = np.concatenate([[0], np.cumsum((x != 0).sum(1))])
        return CO.mat("CSR", (r, c), ip, np.nonzero(x)[1], x[x != 0]), x
    (A, a), (B, b), (Cm, c), (D, d) = dense(2, 3), dense(2, 5), dense(2, 5), dense(2, 3)
    got = CO.bmat([[A, B], [Cm, D]])
    assert got.shape == (4, 8)
    assert np.array_equal(CO.to_dense(got), np.block([[a, b], [c, d]]))
    with pytest.raises(CO.Panic, match="Dimension mismatch"):
        CO.bmat([[A, None], [Cm, D]])   # widths 3 + 3 and 5 + 3
    with pytest.raises(CO.Panic, match="Dimension mismatch"):
        CO.bmat([[A, dense(3, 2)[0]]])  # heights 2 and 3 in one block row


@pytest.mark.parametrize("sa", ["CSR", "CSC"])
@pytest.mark.parametrize("sb", ["CSR", "CSC"])
def test_oracle_kron_kat(kats, sa, sb):
    a, b = m(kats["kron_a"]), m(kats["kron_b"])
    a = a if sa == "CSR" else CO.to_other_storage(a)
    b = b if sb == "CSR" else CO.to_other_storage(b)
    c = CO.kronecker_product(a, b)
    assert c.storage == sa and c.shape == (6, 6)
    want = np.zeros((6, 6))
    for i, j, v in kats["kron_entries"]:
        want[i, j] = v
    assert np.array_equal(CO.to_dense(c), want) and int(c.indptr[-1]) == 16
    assert np.array_equal(CO.to_dense(c), np.kron(CO.to_dense(a), CO.to_dense(b)))
