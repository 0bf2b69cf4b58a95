// test_reference_kats.cpp -- the reference's own product tests, replayed through the C++
// host mirror (include/sprs_b200.hpp) on the GPU.  Each function names the sprs test it
// follows; fixtures are the data of sprs/src/test_data.rs:6-123.  Run by
// tests/test_gpu_cpp_host.py (needs a GPU); exits non-zero on the first failure.
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "../../include/sprs_b200.hpp"

using namespace sprs;
static int g_checks = 0;
#define CHECK(cond)                                                             \
    do {                                                                        \
        ++g_checks;                                                             \
        if (!(cond)) {                                                          \
            fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);    \
            exit(1);                                                            \
        }                                                                       \
    } while (0)

// ---- sprs/src/test_data.rs
static CsMat mat1() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static CsMat mat1_csc() { return CsMat::new_csc({5, 5}, {0, 0, 1, 3, 6, 7}, {3, 0, 2, 0, 1, 4, 1}, {8., 3., 5., 4., 2., 7., 5.}); }
static CsMat mat2() { return CsMat::new_({5, 5}, {0, 4, 6, 6, 8, 10}, {0, 1, 2, 4, 0, 3, 2, 3, 1, 2}, {6., 7., 3., 3., 8., 9., 2., 4., 4., 4.}); }
static CsMat mat4() { return CsMat::new_csc({5, 5}, {0, 4, 6, 6, 8, 10}, {0, 1, 2, 4, 0, 3, 2, 3, 1, 2}, {6., 7., 3., 3., 8., 9., 2., 4., 4., 4.}); }
static CsMat mat5() {
    return CsMat::new_({5, 15}, {0, 5, 11, 14, 20, 22},
                       {1, 2, 6, 7, 13, 3, 4, 6, 8, 13, 14, 7, 11, 13, 3, 8, 9, 10, 11, 14, 4, 12},
                       {4.8, 2., 3.7, 5.9, 6., 1.6, 0.3, 9.2, 9.9, 4.8, 6.1, 4.4, 6., 0.1, 7.2, 1., 1.4, 6.4, 2.8, 3.4, 5.5, 3.5});
}
static CsMat mat1_self_matprod() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 7, 8}, {1, 2, 1, 3, 2, 3, 4, 1}, {32., 15., 16., 35., 25., 16., 40., 56.}); }
static CsMat mat1_matprod_mat2() { return CsMat::new_({5, 5}, {0, 2, 5, 5, 7, 9}, {2, 3, 1, 2, 3, 0, 3, 2, 3}, {8., 16., 20., 24., 8., 64., 72., 14., 28.}); }
static CsMat mat1_csc_matprod_mat4() {
    return CsMat::new_csc({5, 5}, {0, 4, 7, 7, 11, 14}, {0, 1, 2, 3, 0, 1, 4, 0, 1, 2, 4, 0, 2, 3},
                          {9., 15., 15., 56., 36., 18., 63., 22., 8., 10., 28., 12., 20., 32.});
}
static Array2 mat_dense1() { return Array2::from_rows({{0., 1., 2., 3., 4.}, {5., 6., 5., 4., 3.}, {4., 5., 4., 3., 2.}, {3., 4., 3., 2., 1.}, {1., 2., 1., 1., 0.}}); }
static Array2 mat_dense2() {
    return Array2::from_rows({{8.2, 1.8, 0.9, 2.6, 6.7, 7.6, 8.3}, {8.7, 9.4, 2.6, 6.4, 3.5, 1.2, 4.7}, {5.3, 9., 8.7, 9.8, 4.6, 2.5, 4.6},
                              {4.7, 6.2, 3.7, 5.6, 4.7, 8.3, 3.}, {3.5, 6.4, 2.3, 7.3, 4.2, 3.3, 8.9}, {3.6, 6.2, 7.3, 3.1, 1.5, 4.1, 0.8},
                              {8.8, 8.7, 1.6, 6.1, 5.6, 0.1, 8.5}, {4.8, 4.1, 8.1, 0., 0.4, 3., 5.1}, {6.6, 3.4, 1.7, 3.9, 2.2, 5.5, 6.8},
                              {4.8, 3.7, 9.2, 7.4, 3.5, 1.5, 5.8}, {4.3, 6.9, 6.5, 5.7, 7.6, 9.5, 5.8}, {5.7, 6.9, 8.5, 0.1, 5.8, 9.6, 4.9},
                              {6.9, 5.4, 0., 1.2, 4.8, 1.5, 7.9}, {2.8, 5.1, 0.6, 3., 8.4, 8.6, 1.}, {8.1, 1.9, 6.3, 0.2, 0.3, 5.9, 0.}});
}
static Array2 expected_mat1_dense1() {
    return Array2::from_rows({{24., 31., 24., 17., 10.}, {11., 18., 11., 9., 2.}, {20., 25., 20., 15., 10.}, {40., 48., 40., 32., 24.}, {21., 28., 21., 14., 7.}});
}

// prod.rs:376-398 mul_csr_vec
static void mul_csr_vec() {
    auto mat = CsMat::new_({5, 5}, {0, 3, 3, 5, 6, 7}, {1, 2, 3, 2, 3, 4, 4},
                           {0.75672424, 0.1649078, 0.30140296, 0.10358244, 0.6283315, 0.39244208, 0.57202407});
    Array1 vector = {0.1, 0.2, -0.1, 0.3, 0.9}, res_vec(5, 0.0);
    prod::mul_acc_mat_vec_csr(mat, vector, res_vec);
    const double expected[] = {0.22527496, 0., 0.17814121, 0.35319787, 0.51482166};
    for (int i = 0; i < 5; ++i) CHECK(std::fabs(res_vec[i] - expected[i]) < 1e-7);
    Array1 y = mat * vector;  // operator form, csmat.rs:2119-2160
    for (int i = 0; i < 5; ++i) CHECK(std::fabs(y[i] - expected[i]) < 1e-7);
}
// prod.rs:326-349 mul_csc_vec
static void mul_csc_vec() {
    auto mat = CsMat::new_csc({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3},
                              {0.35310881, 0.42380633, 0.28035896, 0.58082095, 0.53350123, 0.88132896, 0.72527863});
    Array1 vector = {0.1, 0.2, -0.1, 0.3, 0.9}, res_vec(5, 0.0);
    prod::mul_acc_mat_vec_csc(mat, vector, res_vec);
    const double expected[] = {0., 0.26439869, -0.01803924, 0.75120319, 0.11616419};
    for (int i = 0; i < 5; ++i) CHECK(std::fabs(res_vec[i] - expected[i]) < 1e-7);
}
// prod.rs:426-458 mul_csr_csr / mul_csc_csc / mul_csc_csr ; smmp.rs:468-473
static void mul_csr_csr_family() {
    auto a = mat1();
    CHECK(a * a == mat1_self_matprod());
    CHECK(a * mat2() == mat1_matprod_mat2());
    CHECK(smmp::mul_csr_csr(a, a) == mat1_self_matprod());
    CHECK(mat1_csc() * mat4() == mat1_csc_matprod_mat4());
    auto a_ = mat1_csc();
    CHECK(a * a_ == mat1_self_matprod());
    CHECK((a_ * a).to_other_storage() == mat1_self_matprod());
    CHECK(a.to_other_storage() == a_);  // csmat.rs:2571 csr_to_csc
}
// smmp.rs:476-489 mul_zero_rows ; csmat.rs:3047-3052 issue_99
static void edge_cases() {
    auto a = CsMat::new_({0, 11}, {0}, {}, {});
    auto b = CsMat::new_({11, 11}, std::vector<size_t>(12, 0), {}, {});
    auto c = a * b;
    CHECK(c.rows() == 0 && c.cols() == 11 && c.nnz() == 0);
    auto d = CsMat::zero({10, 1}) * CsMat::zero({1, 9});
    CHECK(d.rows() == 10 && d.cols() == 9 && d.nnz() == 0);
    bool panicked = false;
    try { (void)(mat5() * mat1()); } catch (const Panic& p) { panicked = std::string(p.what()) == "Dimension mismatch"; }
    CHECK(panicked);
    panicked = false;
    Array1 x(5, 0.0), y(5, 0.0);
    try { prod::mul_acc_mat_vec_csc(mat1(), x, y); } catch (const Panic& p) { panicked = std::string(p.what()) == "Storage mismatch"; }
    CHECK(panicked);
}
// prod.rs:461-500 CsVec products ; lib.rs:54-60 README example
static void csvec_products() {
    CsVec v(5, {0, 2, 4}, {1., 1., 1.});
    CHECK(mat1() * v == CsVec(5, {0, 1, 2}, {3., 5., 5.}));
    CHECK(v * mat1() == CsVec(5, {2, 3}, {8., 11.}));
    CHECK(mat1_csc() * v == CsVec(5, {0, 1, 2}, {3., 5., 5.}));
    CHECK(v * mat1_csc() == CsVec(5, {2, 3}, {8., 11.}));
    CsVec x(5, {0, 2, 4}, {1., 2., 3.});
    CHECK(CsMat::eye(5) * x == x);
    CsVec zero(0, {}, {});
    CHECK(mat1() * zero == zero);
    // prod.rs:312-323 test_csvec_dot_by_binary_search
    CsVec v1(8, {0, 2, 4, 6}, {1., 1., 1., 1.}), v2(8, {1, 3, 5, 7}, {2., 2., 2., 2.}),
        v3(8, {1, 2, 5, 6}, {3., 3., 3., 3.});
    CHECK(prod::csvec_dot_by_binary_search(v1, v2) == 0.);
    CHECK(prod::csvec_dot_by_binary_search(v1, v1) == 4.);
    CHECK(prod::csvec_dot_by_binary_search(v2, v2) == 16.);
    CHECK(prod::csvec_dot_by_binary_search(v1, v3) == 6.);
    CHECK(prod::csvec_dot_by_binary_search(v2, v3) == 12.);
    // vec.rs:1649-1689 dot_product (+ the two panics)
    CHECK(dot(v1, v2) == 0. && dot(v1, v1) == 4. && dot(v2, v2) == 16. && dot(v1, v3) == 6. &&
          dot(v2, v3) == 12.);
    Array1 dense(8);
    for (size_t i = 0; i < 8; ++i) dense[i] = (double)(i + 1);
    CHECK(dot_dense(v1, dense) == 16.);
    bool p1 = false, p2 = false;
    try { dot(v1, CsVec(9, {1, 3, 5, 7}, {2., 2., 2., 2.})); } catch (const Panic&) { p1 = true; }
    try { dot_dense(v1, Array1(9, 1.0)); } catch (const Panic&) { p2 = true; }
    CHECK(p1 && p2);
    // dot_dense sums with `Iterator::sum`, whose f64 fold starts from -0.0 (std since
    // rust-lang/rust#129321, inside the reference's rust-version 1.88; pinned from the std
    // source, not from a run): an empty vector and all -0.0 products give -0.0.  dot with a
    // dense rhs is dot_acc, which starts from +0.0.
    Array1 zeros(8, 0.0);
    CsVec empty8(8, {}, {}), neg(8, {1, 4, 6}, {-1., -2.5, -0.0});
    CHECK(std::signbit(dot_dense(empty8, dense)) && dot_dense(empty8, dense) == 0.);
    CHECK(std::signbit(dot_dense(neg, zeros)));                  // -1*0, -2.5*0, -0*0: all -0.0
    CHECK(!std::signbit(dot_dense(v1, zeros)));                  // +0.0 products
    CsVec mixed(8, {1, 4}, {-0.0, 2.});
    CHECK(dot_dense(mixed, dense) == 10.);                       // -0.0 + 10
    CHECK(!std::signbit(dot(neg, CsVec(8, {1, 4, 6}, {0., 0., 0.}))));  // dot_acc: +0.0 + -0.0
    CHECK(!std::signbit(dot(empty8, v1)));
}
// prod.rs:503-595 dense products
static void dense_products() {
    auto e = CsMat::eye(3);
    Array2 a = Array2::from_rows({{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}), res = Array2::zeros(3, 3);
    prod::csr_mulacc_dense_rowmaj(e, a, res);
    CHECK(res == a);
    auto b = mat_dense1();
    res = Array2::zeros(5, 5);
    prod::csr_mulacc_dense_rowmaj(mat1(), b, res);
    CHECK(res == expected_mat1_dense1());
    CHECK(mat1() * b == expected_mat1_dense1());
    res = Array2::zeros(5, 7);
    prod::csr_mulacc_dense_rowmaj(mat5(), mat_dense2(), res);
    auto exp = Array2::from_rows({{130.04, 150.1, 87.19, 90.89, 99.48, 80.43, 99.3}, {217.72, 161.61, 79.47, 121.5, 124.23, 146.91, 157.79},
                                  {55.6, 59.95, 86.7, 0.9, 37.4, 71.66, 51.94}, {118.18, 123.16, 128.04, 92.02, 106.84, 175.1, 87.36},
                                  {43.4, 54.1, 12.65, 44.35, 39.9, 23.4, 76.6}});
    for (size_t i = 0; i < 5; ++i)
        for (size_t j = 0; j < 7; ++j) CHECK(std::fabs(res(i, j) - exp(i, j)) <= 1e-8);
    res = Array2::zeros(5, 5);
    prod::csc_mulacc_dense_rowmaj(mat1_csc(), b, res);
    CHECK(res == expected_mat1_dense1());
    CHECK(mat1_csc() * b == expected_mat1_dense1());
    auto bf = b.to_f_order();
    res = Array2::zeros_f(5, 5);
    prod::csc_mulacc_dense_colmaj(mat1_csc(), bf, res);
    CHECK(res == expected_mat1_dense1());
    res = Array2::zeros_f(5, 5);
    prod::csr_mulacc_dense_colmaj(mat1(), bf, res);
    CHECK(res == expected_mat1_dense1());
    Array2 c = mat1() * bf;  // 5 columns < 8 -> F-order result (csmat.rs:2009)
    CHECK(c.rs == 1 && c == expected_mat1_dense1());
}
// prod.rs:618-651 test_sparse_dot_dense (rtol 1e-7, atol 1e-12)
static void sparse_dot_dense() {
    std::vector<CsMat> sparse;
    sparse.push_back(mat1()); sparse.push_back(mat1_csc()); sparse.push_back(mat2());
    sparse.push_back(mat2().transpose_into()); sparse.push_back(mat4()); sparse.push_back(mat5());
    std::vector<Array2> dense = {mat_dense1(), mat_dense1().to_f_order(), mat_dense1().reversed_axes(),
                                 mat_dense2(), mat_dense2().reversed_axes()};
    int n = 0;
    for (auto& s : sparse)
        for (auto& d : dense) {
            if (d.rows < s.cols()) continue;
            Array2 dv = d;  // slice(s![0..s.cols(), ..]): same strides, fewer rows
            dv.rows = s.cols();
            Array2 test = s.dot(dv);
            for (size_t i = 0; i < s.rows(); ++i)
                for (size_t j = 0; j < dv.cols; ++j) {
                    double truth = 0.0;
                    for (size_t k = 0; k < s.cols(); ++k) truth += s.to_dense_at(i, k) * dv(k, j);
                    CHECK(std::fabs(test(i, j) - truth) <= std::fabs(truth) * 1e-7 + 1e-12);
                }
            ++n;
        }
    CHECK(n >= 20);
}
// CsMatI<u32> (the BASELINE index width) and sliced views
static void u32_and_slices() {
    using M = CsMatI<uint32_t, uint32_t>;
    auto a = M::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.});
    auto c = a * a;
    CHECK((c.indptr() == std::vector<uint32_t>{0, 2, 4, 5, 7, 8}));
    CHECK((c.indices() == std::vector<uint32_t>{1, 2, 1, 3, 2, 3, 4, 1}));
    CHECK((c.data() == std::vector<double>{32., 15., 16., 35., 25., 16., 40., 56.}));
    Array1 x = {1., 2., 3., 4., 5.};
    Array1 full = mat1() * x;
    Array1 part = mat1().slice_outer(2, 5) * x;  // non-zero-based indptr view (indptr.rs:122-124)
    for (int i = 0; i < 3; ++i) CHECK(part[i] == full[2 + i]);
}

int main() {
    try {
        mul_csr_vec();
        mul_csc_vec();
        mul_csr_csr_family();
        edge_cases();
        csvec_products();
        dense_products();
        sparse_dot_dense();
        u32_and_slices();
    } catch (const std::exception& e) {
        fprintf(stderr, "EXCEPTION: %s\n", e.what());
        return 2;
    }
    printf("OK %d checks\n", g_checks);
    return 0;
}
