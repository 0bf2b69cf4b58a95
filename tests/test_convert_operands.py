"""The operands of tests/test_gpu_zzz_convert_bits.py reach the seams they claim, with the oracle
alone (no GPU): radix pass counts of `bits_for`, duplicate runs straddling the sort's warp and
block boundaries in both of its sorts, an inner index over several sort blocks, long product
rows, and -- for the fixed seeds -- another summation order that changes at least 15 % of the
entries of three or more terms, so the device tests could tell the orders apart."""
import numpy as np
import pytest

import test_gpu_zzz_convert_bits as T


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def test_bits_for_pass_seams():
    """bits_for restated from transpose.cu: 1, 2, 3 and 4 passes of 8 bits at the seams."""
    want = {1: 1, 2: 1, 256: 1, 257: 2, 65536: 2, 65537: 3, 1 << 24: 3, (1 << 24) + 1: 4}
    assert {r: T.passes(r) for r in want} == want
    assert T.bits_for(0) == 1 and T.bits_for(1) == 1 and T.bits_for(2) == 1 and T.bits_for(3) == 2


@pytest.mark.parametrize("name", T.CONVERT_CASES)
def test_convert_cases_reach_their_seams(O, name):
    rng = np.random.default_rng(T.CONVERT_CASES.index(name) + 11)
    outer, inner, ip, ind = T.convert_case(rng, name)
    s = T.convert_seams(outer, inner, ip, ind)
    if name.startswith("inner="):
        assert s["blocks"] >= 3
    if name.startswith("nnz="):
        assert s["nnz"] == int(name[4:])
        assert s["blocks"] == (1 if s["nnz"] <= T.RS_CHUNK else 2)
    if name in ("hub", "inner=1"):
        assert s["hub_blocks"] > 3
    if name.startswith("empty") or name == "no_nonzeros":
        assert s["nnz"] == 0
    # the oracle's conversion keeps every value's bits (the device test compares with it)
    d = T.plant_raw(rng, T.real_values(rng, len(ind)))
    t = O.convert_mat_storage(outer, inner, ip, ind, d)
    assert np.array_equal(np.sort(T.u64(t[2])), np.sort(T.u64(d)))


@pytest.mark.parametrize("pc", list(T.TRIPLET_SHAPES))
def test_triplet_cases_straddle_and_are_order_sensitive(O, pc):
    """Same seed and draws as test_from_triplets_duplicate_order_bits."""
    shape = T.TRIPLET_SHAPES[pc]
    rng = np.random.default_rng(pc[0] * 10 + pc[1])
    r, c, _ = T.triplet_case(rng, *shape)
    s = T.triplet_seams(r, c, *shape)
    assert s["passes"] == pc
    for k in ("col_warp", "col_block", "row_warp", "row_block"):
        assert s[k] >= 20, s
    v = T.triplet_values(rng, len(r))
    n3, share = T.triplet_sensitivity(O, rng, shape, r, c, v)
    assert n3 >= 300 and share >= T.MIN_SHARE
    lens = [len(m) for m in T.run_members(r, c, *shape)]
    assert min(lens) >= 3 and max(lens) >= 40


def test_ping_pong_parities_covered():
    """The column sort's pass count decides which buffer the row sort starts from: both
    parities occur, and so does a 4-pass sort."""
    col_passes = {pc[1] for pc in T.TRIPLET_SHAPES}
    assert {p % 2 for p in col_passes} == {0, 1} and 4 in col_passes


@pytest.mark.parametrize("k", [8, 33, 64, 66, 129])
def test_product_operands_are_order_sensitive(O, k):
    """Same seed and draws as test_csc_mulacc_dense_rowmaj_bits: rows of > 100 non-zeros, and a
    column permutation changes >= 15 % of the >= 3-term outputs."""
    rng = np.random.default_rng(300 + k)
    rows, cols = 600, 900
    csr = T.product_operand(rng, rows, cols)
    b = T.real_values(rng, cols * k).reshape(cols, k)
    c0 = T.real_values(rng, rows * k).reshape(rows, k)
    T.assert_product_sensitivity(O, rng, rows, cols, csr, b, c0)


def test_dot_dense_reference_sign_of_zero():
    """The restated reference sums: dot_dense folds from -0.0, dot_acc from +0.0."""
    i = np.array([1, 4])
    assert np.signbit(T.ref_dot_dense([], [], np.ones(5)))
    assert np.signbit(T.ref_dot_dense(i, np.array([-1.0, -2.0]), np.zeros(5)))
    assert not np.signbit(T.ref_dot_dense(i, np.array([1.0, -2.0]), np.zeros(5)))
    assert not np.signbit(T.ref_dot_dense_acc(i, np.array([-1.0, -2.0]), np.zeros(5)))
