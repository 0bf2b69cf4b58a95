// test_dense_kats.cpp -- the reference's dense-boundary tests (to_dense.rs:56-92,
// csmat.rs:2493-2539, binop.rs:600-718) replayed through the C++ host mirror
// (include/sprs_b200.hpp) on the GPU.  Built and run by
// tests/test_gpu_dense.py::test_cpp_dense_kats; exits non-zero on the first failure.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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

static CsMat mat1() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static CsMat mat3() { return CsMat::new_({5, 4}, {0, 2, 4, 5, 6, 7}, {2, 3, 2, 3, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static Array2 eye3() { return Array2::from_rows({{1., 0., 0.}, {0., 1., 0.}, {0., 0., 1.}}); }
static CsMat eye_csc(size_t n) { return CsMat::eye(n).transpose_into(); }  // eye is symmetric

template <class F>
static bool panics_with(F f, const char* msg) {
    try {
        f();
    } catch (const Panic& p) {
        return std::string(p.what()).find(msg) != std::string::npos;
    }
    return false;
}

static bool same_bits(const Array2& a, const Array2& b) {
    if (a.rows != b.rows || a.cols != b.cols) return false;
    for (size_t i = 0; i < a.rows; ++i)
        for (size_t j = 0; j < a.cols; ++j) {
            const double x = a(i, j), y = b(i, j);
            if (std::memcmp(&x, &y, 8) != 0) return false;
        }
    return true;
}

// a strided view: every other column of a C-order array with twice the columns
static Array2 every_other_col(size_t r, size_t c, double v, bool f_order) {
    Array2 a = f_order ? Array2::zeros_f(r, 2 * c) : Array2::zeros(r, 2 * c);
    for (auto& x : a.data) x = v;
    a.cols = c;
    a.cs *= 2;
    return a;
}

int main() {
    // to_dense.rs:56-92
    for (const CsMat& e : {CsMat::eye(3), eye_csc(3)}) {
        Array2 d = Array2::zeros(3, 3);
        assign_to_dense(d, e);
        CHECK(d == eye3());
        CHECK(e.to_dense() == eye3());
    }
    CHECK(mat1().to_dense() == Array2::from_rows({{0., 0., 3., 4., 0.}, {0., 0., 0., 2., 5.},
                                                   {0., 0., 5., 0., 0.}, {0., 8., 0., 0., 0.},
                                                   {0., 0., 0., 7., 0.}}));
    CHECK(mat3().to_dense() == Array2::from_rows({{0., 0., 3., 4.}, {0., 0., 2., 5.}, {0., 0., 5., 0.},
                                                   {0., 8., 0., 0.}, {0., 0., 0., 7.}}));
    // csmat.rs:2493-2539
    CHECK(CsMat::csr_from_dense(eye3(), 0.) == CsMat::eye(3));
    CHECK(CsMat::csc_from_dense(eye3(), 0.) == eye_csc(3));
    const Array2 m = Array2::from_rows({{1., 0., 2., 1e-7, 1.}, {0., 0., 0., 1., 0.}, {3., 0., 1., 0., 0.}});
    CHECK(CsMat::csr_from_dense(m, 1e-5) ==
          CsMat::new_({3, 5}, {0, 3, 4, 6}, {0, 2, 4, 3, 0, 2}, {1., 2., 1., 1., 3., 1.}));
    CHECK(CsMat::csc_from_dense(m, 1e-5) ==
          CsMat::new_csc({3, 5}, {0, 2, 2, 4, 5, 6}, {0, 2, 0, 2, 1, 0}, {1., 3., 2., 1., 1., 1.}));
    CHECK(CsMat::csr_from_dense(m.to_f_order(), 1e-5) == CsMat::csr_from_dense(m, 1e-5));
    // binop.rs:600-718: csr_add_dense_rowmaj, csr_mul_dense_rowmaj, mul_dense_strided
    CHECK(binop::add_dense_mat_same_ordering(CsMat::eye(3), Array2::zeros(3, 3), 1., 1.) == eye3());
    const Array2 dense1 = Array2::from_rows({{0., 1., 2., 3., 4.}, {5., 6., 5., 4., 3.}, {4., 5., 4., 3., 2.},
                                             {3., 4., 3., 2., 1.}, {1., 2., 1., 1., 0.}});
    const Array2 expect = Array2::from_rows({{0., 1., 5., 7., 4.}, {5., 6., 5., 6., 8.}, {4., 5., 9., 3., 2.},
                                             {3., 12., 3., 2., 1.}, {1., 2., 1., 8., 0.}});
    CHECK(binop::add_dense_mat_same_ordering(mat1(), dense1, 1., 1.) == expect);
    CHECK(mat1() + dense1 == expect);
    const Array2 sum_f = mat1() + dense1.to_f_order();     // CSR + F-like D: A converted first
    CHECK(sum_f == expect && !sum_f.is_standard_layout());
    Array2 ones = Array2::zeros(3, 3);
    for (auto& x : ones.data) x = 1.;
    CHECK(binop::mul_dense_mat_same_ordering(CsMat::eye(3), ones, 1.) == eye3());
    const Array2 c = binop::mul_dense_mat_same_ordering(CsMat::eye(3), every_other_col(3, 3, 1., false), 1.);
    CHECK(c.is_standard_layout() && c == eye3());
    const Array2 cf = binop::mul_dense_mat_same_ordering(eye_csc(3), every_other_col(3, 3, 1., true), 1.);
    CHECK(cf.reversed_axes().is_standard_layout() && cf == eye3());
    // the panics: shapes first, then the layout
    CHECK(panics_with([] { binop::add_dense_mat_same_ordering(mat1(), Array2::zeros_f(5, 4), 1., 1.); },
                      "Dimension mismatch"));
    CHECK(panics_with([&] { binop::add_dense_mat_same_ordering(mat1(), dense1.to_f_order(), 1., 1.); },
                      "Storage mismatch"));
    CHECK(panics_with([] { Array2 d = Array2::zeros(4, 5); assign_to_dense(d, mat1()); }, "Dimension mismatch"));
    // the value rules of the closures
    const CsMat e = CsMat::new_({1, 3}, {0, 1}, {0}, {2.});
    const Array2 nz = Array2::from_rows({{1., -0., -5.}});
    const Array2 s = binop::add_dense_mat_same_ordering(e, nz, 1., 1.);
    CHECK(same_bits(s, Array2::from_rows({{3., 0., -5.}})));            // -0.0 became +0.0
    const Array2 p = binop::mul_dense_mat_same_ordering(e, nz, 1.);
    CHECK(same_bits(p, Array2::from_rows({{2., -0., -0.}})));           // (1 * 0) * -5 = -0.0
    printf("OK %d checks\n", g_checks);
    return 0;
}
