"""GPU parity tests for SpGEMM (smmp.rs) and the CSC side of the dispatch tables
(csmat.rs:1895-1949, 2009-2046), through the C ABI.  SpGEMM indptr / indices and every value
must be bit-exact: every numeric bin adds A's non-zeros in storage order, like the reference."""
import numpy as np
import pytest
import scipy.sparse as sp_

import exact
from conftest import mat_arrays, rand_csr

pytestmark = pytest.mark.gpu
RTOL = 1e-6


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def csmat(sp, m, idx=np.uint64):
    ip, ind, d = mat_arrays(m, idx)
    ctor = sp.CsMat.new if m["storage"] == "CSR" else sp.CsMat.new_csc
    return ctor(tuple(m["shape"]), ip, ind, d)


def expect(sp, fixtures, name):
    return csmat(sp, fixtures[name])


# ------------------------------------------------------------------ reference KATs
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_mul_csr_csr(sp, fixtures, idx):
    """prod.rs:426-437 mul_csr_csr / smmp.rs:468-473: assert_eq! on the whole CsMat."""
    a = csmat(sp, fixtures["mat1"], idx)
    b = csmat(sp, fixtures["mat2"], idx)
    res = a * a
    e = fixtures["mat1_self_matprod"]
    assert res.indptr.tolist() == e["indptr"] and res.indices.tolist() == e["indices"]
    assert res.data.tolist() == e["data"]
    assert res.indices.dtype == idx and res.is_csr() and res.shape == (5, 5)
    res = a * b
    assert res == expect(sp, fixtures, "mat1_matprod_mat2")
    assert sp.smmp.mul_csr_csr(a, a) == expect(sp, fixtures, "mat1_self_matprod")


def test_mul_csc_csc(sp, fixtures):
    """prod.rs:439-446 mul_csc_csc -> CSC result (csmat.rs:1944-1947)."""
    res = csmat(sp, fixtures["mat1_csc"]) * csmat(sp, fixtures["mat4"])
    assert res == expect(sp, fixtures, "mat1_csc_matprod_mat4")
    assert res.is_csc()


def test_mul_csc_csr(sp, fixtures):
    """prod.rs:448-458 mul_csc_csr: mixed storage converts (csmat.rs:1935-1943)."""
    a, a_ = csmat(sp, fixtures["mat1"]), csmat(sp, fixtures["mat1_csc"])
    exp = expect(sp, fixtures, "mat1_self_matprod")
    assert a * a_ == exp
    assert (a_ * a).to_other_storage() == exp


def test_csr_to_csc(sp, fixtures):
    """csmat.rs:2571 csr_to_csc (to_other_storage, csmat.rs:1405-1426)."""
    assert csmat(sp, fixtures["mat1"]).to_other_storage() == csmat(sp, fixtures["mat1_csc"])
    assert csmat(sp, fixtures["mat1_csc"]).to_other_storage() == csmat(sp, fixtures["mat1"])


def test_mul_zero_rows_and_issue_99(sp):
    """smmp.rs:476-489 mul_zero_rows (gh#239); csmat.rs:3047-3052 issue_99."""
    a = sp.CsMat.new((0, 11), [0], [], [])
    b = sp.CsMat.new((11, 11), [0] * 12, [], [])
    c = a * b
    assert c.rows() == 0 and c.cols() == 11 and c.nnz() == 0
    c = sp.CsMat.zero((10, 1)) * sp.CsMat.zero((1, 9))
    assert c.shape == (10, 9) and c.nnz() == 0 and c.indptr.tolist() == [0] * 11


def test_spgemm_dimension_panic(sp, fixtures):
    """smmp.rs:207 assert_eq!(lhs.cols(), rhs.rows())."""
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.smmp.mul_csr_csr(csmat(sp, fixtures["mat5"]), csmat(sp, fixtures["mat1"]))
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        csmat(sp, fixtures["mat5"]) * csmat(sp, fixtures["mat1"])


def test_structural_zeros_kept(sp):
    """SURVEY F12 / smmp.rs:109-129: cancellation keeps the structural entry."""
    a = sp.CsMat.new((1, 2), [0, 2], [0, 1], [1., 1.])
    b = sp.CsMat.new((2, 1), [0, 1, 2], [0, 0], [1., -1.])
    c = a * b
    assert c.indptr.tolist() == [0, 1] and c.indices.tolist() == [0] and c.data.tolist() == [0.0]


def test_csvec_products(sp, fixtures):
    """prod.rs:476-500 mul_csvec_csr / mul_csc_csvec / mul_csvec_csc."""
    k = fixtures["kat_csvec"]
    v = sp.CsVec(5, k["v"]["indices"], k["v"]["data"])
    exp_va = sp.CsVec(5, k["v_times_mat1"]["indices"], k["v_times_mat1"]["data"])
    exp_av = sp.CsVec(5, k["mat1_times_v"]["indices"], k["mat1_times_v"]["data"])
    assert v * csmat(sp, fixtures["mat1"]) == exp_va
    assert csmat(sp, fixtures["mat1_csc"]) * v == exp_av
    assert v * csmat(sp, fixtures["mat1_csc"]) == exp_va


def test_csc_dense_kats(sp, fixtures):
    """prod.rs:326-373 mul_csc_vec; :545-578 mul_csc_dense_rowmaj / colmaj + operators."""
    k = fixtures["kat_mul_csc_vec"]
    mat = csmat(sp, k["mat"])
    res = np.zeros(5)
    sp.prod.mul_acc_mat_vec_csc(mat, np.array(k["x"]), res)
    assert np.all(np.abs(res - np.array(k["expected"])) < k["epsilon"])
    a = csmat(sp, fixtures["mat1_csc"])
    b = np.array(fixtures["mat_dense1"])
    res = np.zeros((5, 5))
    sp.prod.csc_mulacc_dense_rowmaj(a, b, res)
    assert np.array_equal(res, np.array(fixtures["kat_mat1_x_dense1"]))
    assert np.array_equal(a * b, np.array(fixtures["kat_mat1_x_dense1"]))
    bf = np.asfortranarray(b)
    res = np.zeros((5, 5), order="F")
    sp.prod.csc_mulacc_dense_colmaj(a, bf, res)
    assert np.array_equal(res, np.array(fixtures["kat_mat1_x_dense1"]))


def test_sparse_dot_dense_all_storages(sp, fixtures):
    """prod.rs:618-692 test_sparse_dot_dense + test_dense_dot_sparse: all 6 sparse
    operands (CSR, CSC, transposed) x 5 dense layouts, rtol 1e-7 atol 1e-12."""
    tol = fixtures["assert_close"]
    m2 = csmat(sp, fixtures["mat2"])
    sparse = [csmat(sp, fixtures["mat1"]), csmat(sp, fixtures["mat1_csc"]), m2,
              m2.transpose_into(), csmat(sp, fixtures["mat4"]), csmat(sp, fixtures["mat5"])]
    d1, d2 = np.array(fixtures["mat_dense1"]), np.array(fixtures["mat_dense2"])
    dense = [d1, np.asfortranarray(d1), d1.T, d2, d2.T]
    n = 0
    for s in sparse:
        for dn in dense:
            if dn.shape[0] >= s.cols():
                dv = dn[:s.cols(), :]
                truth = s.to_dense().dot(dv)
                assert np.all(np.abs(s.dot(dv) - truth) <= np.abs(truth) * tol["rtol"] + tol["atol"])
                n += 1
            if dn.shape[1] >= s.rows():
                dv = dn[:, :s.rows()]
                truth = dv.dot(s.to_dense())
                test = dv @ s  # dense.dot(&sparse), csmat.rs:2050-2099
                assert np.all(np.abs(test - truth) <= np.abs(truth) * tol["rtol"] + tol["atol"])
                n += 1
    assert n >= 40


# ------------------------------------------------------------------ oracle parity, random
def check_spgemm(sp, O, a, b, shape_a, shape_b):
    A = sp.CsMat.new(shape_a, *a)
    B = sp.CsMat.new(shape_b, *b)
    C = A * B
    rip, rind, rd = O.mul_csr_csr(shape_a, a, shape_b, b, threads=1)
    assert np.array_equal(C.indptr, rip), "indptr differs"
    assert np.array_equal(C.indices, rind), "indices differ"
    exact.assert_same_class(C.data, rd, "spgemm values")
    return C


@pytest.mark.parametrize("case", [
    dict(n=1, m=1, p=1, da=1, db=1),
    dict(n=300, m=200, p=250, da=6, db=5, empty=0.2),
    dict(n=2000, m=1500, p=1800, da=12, db=10),                 # mostly warp-per-row bins
    dict(n=400, m=3000, p=20000, da=60, db=40),                 # CTA hash bins (n_prod ~2400)
    dict(n=60, m=4000, p=30000, da=900, db=60),                 # large rows: shared-memory column panels
    dict(n=3000, m=3000, p=3000, da=20, db=20, skew=True),      # power-law mix of all bins
])
def test_spgemm_vs_oracle(sp, O, case):
    rng = np.random.default_rng(case["n"] * 31 + case["p"])
    a = rand_csr(rng, case["n"], case["m"], case["da"], skew=case.get("skew", False),
                 empty_frac=case.get("empty", 0.0))
    b = rand_csr(rng, case["m"], case["p"], case["db"], skew=case.get("skew", False))
    check_spgemm(sp, O, a, b, (case["n"], case["m"]), (case["m"], case["p"]))


def test_spgemm_wide_bitmap_spill(sp, O):
    """B.cols beyond the shared-memory bitmap (1.6M columns): the large-row path spills
    its bitmap and dense accumulator to global memory."""
    rng = np.random.default_rng(77)
    n, m, p = 40, 3000, 2_000_000
    a = rand_csr(rng, n, m, 500)
    b = rand_csr(rng, m, p, 30)
    check_spgemm(sp, O, a, b, (n, m), (m, p))


def test_spgemm_matches_scipy_pattern(sp):
    rng = np.random.default_rng(9)
    a = rand_csr(rng, 500, 400, 8)
    b = rand_csr(rng, 400, 600, 7)
    C = sp.CsMat.new((500, 400), *a) * sp.CsMat.new((400, 600), *b)
    S = sp_.csr_matrix((a[2], a[1], a[0]), shape=(500, 400)) @ \
        sp_.csr_matrix((b[2], b[1], b[0]), shape=(400, 600))
    S.sort_indices()
    assert np.array_equal(C.indptr, S.indptr) and np.array_equal(C.indices, S.indices)


@pytest.mark.parametrize("shape", [(1, 1), (37, 501), (5000, 3000), (300, 70000)])
def test_to_other_storage_vs_oracle(sp, O, shape):
    """convert_mat_storage (csmat.rs:1782-1829): device stable radix sort vs the oracle's
    counting sort -- all three arrays bit-exact, including value order inside a bucket."""
    rng = np.random.default_rng(shape[0] + shape[1])
    ip, ind, d = rand_csr(rng, shape[0], shape[1], min(9, shape[1]), empty_frac=0.1)
    a = sp.CsMat.new(shape, ip, ind, d)
    t = a.to_other_storage()
    oip, oind, od = O.convert_mat_storage(shape[0], shape[1], ip, ind, d)
    assert t.is_csc() and t.shape == shape
    assert np.array_equal(t.indptr, oip) and np.array_equal(t.indices, oind)
    assert np.array_equal(t.data, od)
    assert t.to_other_storage() == a  # idempotent round trip


def test_csc_spmv_matches_csr(sp, O):
    """mul_acc_mat_vec_csc == the CSR kernel on the converted mirror (same summation
    order: ascending column), checked against the oracle's scatter loop (prod.rs:74-99)."""
    rng = np.random.default_rng(21)
    ip, ind, d = rand_csr(rng, 3000, 2000, 15)   # CSR of A^T == CSC of A (2000 x 3000)
    a = sp.CsMat.new_csc((2000, 3000), ip, ind, d)
    x = rng.standard_normal(3000)
    ref, bound = np.zeros(2000), np.zeros(2000)
    O.mul_acc_mat_vec_csc(ip, ind, d, x, ref)
    O.mul_acc_mat_vec_csc(ip, ind, np.abs(d), np.abs(x), bound)
    got = a * x
    assert np.all(np.abs(got - ref) <= RTOL * bound + 1e-300)


def test_spgemm_rmat_properties_full_size(sp):
    """BASELINE config 4 shape (two 500k x 500k R-MAT, ~16 nnz/row) on the device:
    structural properties that hold at any size -- sorted unique columns per row,
    monotone indptr, nnz(C_i) <= n_prod_i, and C x = A (B x) within tolerance."""
    import ctypes as C_
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 500_000
    A = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    B = G.rmat_csr(ctx, n, 16, seed=0x5EED1004)
    plan, nnz_c = C_.c_void_p(), C_.c_uint64()
    ctx.check(ctx.lib.sprs_b200_spgemm_symbolic(ctx.h, A.mirror.h, B.mirror.h, C_.byref(plan),
                                                C_.byref(nnz_c)))
    cm = C_.c_void_p()
    ctx.check(ctx.lib.sprs_b200_spgemm_numeric_dev(ctx.h, plan, C_.byref(cm)))
    nprod = ctx.lib.sprs_b200_spgemm_nprod(plan)
    ctx.lib.sprs_b200_spgemm_free(plan)
    Cm = sp.DeviceCsMat(ctx, cm)
    assert Cm.nnz == nnz_c.value and 0 < Cm.nnz <= nprod
    x = G.normal_vector(ctx, n, 5)
    y1, y2, t = (torch.empty(n, device=x.device, dtype=torch.float64) for _ in range(3))
    G.spmv(ctx, Cm, x, y1)
    G.spmv(ctx, B, x, t)
    G.spmv(ctx, A, t, y2)
    absA = G.DeviceCsr(ctx, n, n, A.indptr, A.indices, A.data.abs())
    absB = G.DeviceCsr(ctx, n, n, B.indptr, B.indices, B.data.abs())
    bound = torch.empty_like(y1)
    G.spmv(ctx, absB, x.abs(), t)
    G.spmv(ctx, absA, t, bound)
    torch.cuda.synchronize()
    assert bool(((y1 - y2).abs() <= 1e-9 * bound + 1e-300).all())
    # sprs invariants of C (monotone indptr, ascending unique in-range columns), on device
    bad = C_.c_uint64(1)
    ctx.check(ctx.lib.sprs_b200_csmat_check_structure(ctx.h, cm, C_.byref(bad)))
    assert bad.value == 0


@pytest.mark.parametrize("shape,n", [((1, 1), 1), ((50, 70), 400), ((3000, 2000), 60000),
                                     ((200000, 300000), 500000), ((10, 10), 0)])
def test_from_triplets_vs_scipy(sp, shape, n):
    """TriMat -> CSR (triplet_iter.rs:127-224): unsorted COO with duplicates -> sorted unique
    columns per row, duplicates summed.  Structure exact vs scipy's coo->csr, values to
    rounding (the summation order of duplicates is unspecified in the reference too)."""
    rng = np.random.default_rng(shape[0] + n)
    r = rng.integers(0, shape[0], n)
    c = rng.integers(0, shape[1], n)
    if n > 10:  # force duplicates
        r[: n // 5] = r[n // 5: 2 * (n // 5)]
        c[: n // 5] = c[n // 5: 2 * (n // 5)]
    d = rng.standard_normal(n)
    m = sp.CsMat.from_triplets(shape, r, c, d)
    ref = sp_.coo_matrix((d, (r, c)), shape=shape).tocsr()
    ref.sum_duplicates()
    ref.sort_indices()
    assert np.array_equal(m.indptr, ref.indptr) and np.array_equal(m.indices, ref.indices)
    absref = sp_.coo_matrix((np.abs(d), (r, c)), shape=shape).tocsr()
    absref.sum_duplicates()
    absref.sort_indices()
    assert np.all(np.abs(m.data - ref.data) <= 1e-12 * absref.data + 1e-300)
    if n:
        x = rng.standard_normal(shape[1])
        assert np.allclose(m * x, ref @ x, rtol=1e-9, atol=1e-9)
