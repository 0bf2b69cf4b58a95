// test_binop_kats.cpp -- the reference's binop tests (sprs/src/sparse/binop.rs:488-531,
// test_data.rs:55-60) replayed through the C++ host mirror (include/sprs_b200.hpp) on the GPU.
// Built and run by tests/test_gpu_binop.py::test_cpp_binop_kats (and on the emulator by
// tests/test_emu_binop.py); exits non-zero on the first failure.
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

static CsMat mat1() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static CsMat mat2() { return CsMat::new_({5, 5}, {0, 4, 6, 6, 8, 10}, {0, 1, 2, 4, 0, 3, 2, 3, 1, 2}, {6., 7., 3., 3., 8., 9., 2., 4., 4., 4.}); }
static CsMat mat1_plus_mat2() {
    return CsMat::new_({5, 5}, {0, 5, 8, 9, 12, 15}, {0, 1, 2, 3, 4, 0, 3, 4, 2, 1, 2, 3, 1, 2, 3},
                       {6., 7., 6., 4., 3., 8., 11., 5., 5., 8., 2., 4., 4., 4., 7.});
}
static CsMat mat1_minus_mat2() {
    return CsMat::new_({5, 5}, {0, 4, 7, 8, 11, 14}, {0, 1, 3, 4, 0, 3, 4, 2, 1, 2, 3, 1, 2, 3},
                       {-6., -7., 4., -3., -8., -7., 5., 5., 8., -2., -4., -4., -4., 7.});
}
static CsMat mat1_times_mat2() { return CsMat::new_({5, 5}, {0, 1, 2, 2, 2, 2}, {2, 3}, {9., 18.}); }
static CsMat mat1_times_2() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {6., 8., 4., 10., 10., 16., 14.}); }

template <class F>
static bool panics_with(F f, const char* msg) {
    try {
        f();
    } catch (const Panic& p) {
        return std::string(p.what()).find(msg) != std::string::npos;
    }
    return false;
}

int main() {
    // binop.rs:512-531 test_add1
    CHECK(mat1() + mat2() == mat1_plus_mat2());
    const CsMat a = CsMat::new_({3, 3}, {0, 1, 1, 2}, {0, 2}, {1., 1.});
    const CsMat b = CsMat::new_({3, 3}, {0, 1, 2, 2}, {0, 1}, {1., 1.});
    CHECK(a + b == CsMat::new_({3, 3}, {0, 1, 2, 3}, {0, 1, 2}, {2., 1., 1.}));
    // test_sub1, test_mul1 (mul_mat_same_storage), the scalar product
    CHECK(mat1() - mat2() == mat1_minus_mat2());
    CHECK(binop::mul_mat_same_storage(mat1(), mat2()) == mat1_times_mat2());
    CHECK(mat1() * 2.0 == mat1_times_2());
    // mixed storage: rhs converted, the result in lhs storage
    CHECK(mat1() + mat2().to_other_storage() == mat1_plus_mat2());
    const CsMat d = mat1().to_other_storage() - mat2();
    CHECK(d.is_csc() && d.to_other_storage() == mat1_minus_mat2());
    // A - A: all entries cancel, the full indptr stays
    const CsMat z = mat1() - mat1();
    CHECK(z.nnz() == 0 && z.indptr() == std::vector<size_t>(6, 0));
    // the panics: shape before storage; Hadamard product refuses mixed storage
    const CsMat wide = CsMat::new_({5, 6}, {0, 0, 0, 0, 0, 0}, {}, {});
    CHECK(panics_with([&] { (void)(mat1() + wide.to_other_storage()); }, "Dimension mismatch"));
    CHECK(panics_with([&] { (void)binop::mul_mat_same_storage(mat1(), wide.to_other_storage()); },
                      "Dimension mismatch"));
    CHECK(panics_with([&] { (void)binop::mul_mat_same_storage(mat1(), mat2().to_other_storage()); },
                      "Storage mismatch"));
    printf("OK %d checks\n", g_checks);
    return 0;
}
