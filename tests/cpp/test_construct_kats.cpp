// test_construct_kats.cpp -- the reference's construction tests (sprs/src/sparse/construct.rs
// mod test, kronecker.rs test_kronecker_product) replayed through the C++ host mirror
// (include/sprs_b200.hpp) on the GPU.  Built and run by
// tests/test_gpu_construct.py::test_cpp_construct_kats (and on the emulator by
// tests/test_emu_construct.py); exits non-zero on the first failure.
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "../../include/sprs_b200.hpp"

using namespace sprs;
static int g_checks = 0;
#define CHECK(...)                                                              \
    do {                                                                        \
        ++g_checks;                                                             \
        if (!(__VA_ARGS__)) {                                                   \
            fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #__VA_ARGS__); \
            exit(1);                                                            \
        }                                                                       \
    } while (0)

static CsMat mat1() { return CsMat::new_({5, 5}, {0, 2, 4, 5, 6, 7}, {2, 3, 3, 4, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static CsMat mat2() { return CsMat::new_({5, 5}, {0, 4, 6, 6, 8, 10}, {0, 1, 2, 4, 0, 3, 2, 3, 1, 2}, {6., 7., 3., 3., 8., 9., 2., 4., 4., 4.}); }
static CsMat mat3() { return CsMat::new_({5, 4}, {0, 2, 4, 5, 6, 7}, {2, 3, 2, 3, 2, 1, 3}, {3., 4., 2., 5., 5., 8., 7.}); }
static CsMat mat4() { return CsMat::new_csc({5, 5}, {0, 4, 6, 6, 8, 10}, {0, 1, 2, 4, 0, 3, 2, 3, 1, 2}, {6., 7., 3., 3., 8., 9., 2., 4., 4., 4.}); }
static CsMat mat1_vstack_mat2() {
    return CsMat::new_({10, 5}, {0, 2, 4, 5, 6, 7, 11, 13, 13, 15, 17},
                       {2, 3, 3, 4, 2, 1, 3, 0, 1, 2, 4, 0, 3, 2, 3, 1, 2},
                       {3., 4., 2., 5., 5., 8., 7., 6., 7., 3., 3., 8., 9., 2., 4., 4., 4.});
}

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
    const CsMat a = mat1(), b = mat2(), c = mat3(), d = mat4();
    // vstack_trivial, hstack_trivial, vstack_with_conversion
    CHECK(vstack<size_t, size_t>({a, b}) == mat1_vstack_mat2());
    const CsMat h = hstack<size_t, size_t>({a.transpose_into(), b.transpose_into()});
    CHECK(h.is_csc() && h == mat1_vstack_mat2().transpose_into());
    CHECK(vstack<size_t, size_t>({a.to_csc(), b}) == mat1_vstack_mat2());
    // bmat_simple
    const CsMat e5 = CsMat::eye(5), e4 = CsMat::eye(4);
    std::vector<size_t> ip9(10), ind9(9);
    for (size_t i = 0; i < 10; ++i) ip9[i] = i;
    for (size_t i = 0; i < 9; ++i) ind9[i] = i;
    CHECK(bmat<size_t, size_t>({{&e5, nullptr}, {nullptr, &e4}}) ==
          CsMat::new_({9, 9}, ip9, ind9, std::vector<double>(9, 1.)));
    // bmat_complex, both halves
    CHECK(bmat<size_t, size_t>({{&a, &b}, {&b, nullptr}}) ==
          CsMat::new_({10, 10}, {0, 6, 10, 11, 14, 17, 21, 23, 23, 25, 27},
                      {2, 3, 5, 6, 7, 9, 3, 4, 5, 8, 2, 1, 7, 8, 3, 6, 7, 0, 1, 2, 4, 0, 3, 2, 3, 1, 2},
                      {3., 4., 6., 7., 3., 3., 2., 5., 8., 9., 5., 8., 2., 4., 7., 4., 4., 6., 7.,
                       3., 3., 8., 9., 2., 4., 4., 4.}));
    CHECK(bmat<size_t, size_t>({{&c, &a}, {nullptr, &d}}) ==
          CsMat::new_({10, 9}, {0, 4, 8, 10, 12, 14, 16, 18, 21, 23, 24},
                      {2, 3, 6, 7, 2, 3, 7, 8, 2, 6, 1, 5, 3, 7, 4, 5, 4, 8, 4, 7, 8, 5, 7, 4},
                      {3., 4., 3., 4., 2., 5., 2., 5., 5., 5., 8., 8., 7., 7., 6., 8., 7., 4., 3.,
                       2., 4., 9., 4., 3.}));
    // the panic tests
    CHECK(panics_with([&] { (void)vstack<size_t, size_t>({}); }, "Empty stacking list"));
    CHECK(panics_with([&] { (void)vstack<size_t, size_t>({a, c}); }, "Dimension mismatch"));
    CHECK(panics_with([&] { (void)bmat<size_t, size_t>({{nullptr, nullptr}, {nullptr}}); },
                      "Dimension mismatch"));
    CHECK(panics_with([&] { (void)bmat<size_t, size_t>({{}}); }, "Empty stacking list"));
    CHECK(panics_with([&] { (void)bmat<size_t, size_t>({{nullptr, nullptr}, {&a, &c}}); },
                      "Empty bmat row"));
    CHECK(panics_with([&] { (void)bmat<size_t, size_t>({{&c, nullptr}, {&a, nullptr}}); },
                      "Empty bmat col"));
    // test_kronecker_product in its four storage combinations
    const CsMat ka = CsMat::new_({2, 3}, {0, 2, 4}, {1, 2, 0, 2}, {2., 3., 6., 8.});
    const CsMat kb = CsMat::new_({3, 2}, {0, 1, 2, 4}, {0, 0, 0, 1}, {1., 2., 3., -3.});
    const double want[][3] = {{0, 2, 2},   {0, 4, 3},  {1, 2, 4},   {1, 4, 6},  {2, 2, 6},   {2, 3, -6},
                              {2, 4, 9},   {2, 5, -9}, {3, 0, 6},   {3, 4, 8},  {4, 0, 12},  {4, 4, 16},
                              {5, 0, 18},  {5, 1, -18}, {5, 4, 24}, {5, 5, -24}};
    for (int sa = 0; sa < 2; ++sa)
        for (int sb = 0; sb < 2; ++sb) {
            const CsMat x = sa ? ka.to_csc() : ka, y = sb ? kb.to_csc() : kb;
            const CsMat k = kronecker_product(x, y);
            CHECK(k.storage() == x.storage() && k.rows() == 6 && k.cols() == 6 && k.nnz() == 16);
            for (const auto& w : want) CHECK(k.to_dense_at((size_t)w[0], (size_t)w[1]) == w[2]);
        }
    // an index that does not fit the index type: the reference's unwrap panic
    using CsMat32 = CsMatI<int32_t, int32_t>;
    const CsMat32 wide = CsMat32::new_({1, 50000}, {0, 1}, {49999}, {2.});
    CHECK(panics_with([&] { (void)kronecker_product(wide, wide); }, "Option::unwrap()"));
    printf("OK %d checks\n", g_checks);
    return 0;
}
